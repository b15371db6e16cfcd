"""Quatro correspondences and max-clique inliers of every loop attempt (b200reg_ctx_set_quatro_matches /
b200reg_quatro_matches, b200reg_batch_set_quatro_matches / b200reg_batch_quatro_matches): the correspondences equal
b200reg_quatro_align_ex's on all three solve paths, the inliers equal the solve tap's and the oracle's clique, the points
are the matched clouds' floats; rows in caller order on the keyframe path; nothing changes and nothing is launched with
recording off; driver jobs return the bytes of the synchronous call; and a C++ client that reads them through the ABI
alone."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc")
CLIENT_SRC = os.path.join(REPO, "tests", "cpp", "quatro_matches_client.cpp")
EINVAL, ESTATE = -1, -4
SOURCE, TARGET = 1, 2
QUERIES = [137, 139, 20, 118]  # 20 has no candidate; the others close loops at the start of the lap
NKF = 140  # keyframes of the sequence; 140 and 141 are the structureless far pair
MAXC, ADV_CAP = 512, 8192
KEYS = ("corr", "inlier", "src_xyz", "dst_xyz")


def _build_client(tmp):
    from b200reg.build import build_native
    build_native()
    exe = os.path.join(tmp, "quatro_matches_client")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-pthread", "-I" + os.path.join(REPO, "include"),
                           "-o", exe, CLIENT_SRC, "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    return exe


def test_quatro_matches_client_compiles(tmp_path):
    """The ABI alone is enough to read a loop attempt's matches from a context and from a driver job (no GPU needed)."""
    assert os.path.exists(_build_client(str(tmp_path)))


def _blobs():
    rng = np.random.default_rng(0)  # no structure at FPFH radii: Quatro finds no valid solution
    return rng.normal(0, 20, (300, 4)).astype(np.float32), rng.normal(0, 20, (280, 4)).astype(np.float32)


def _sparse():
    """Points 50 m apart: no neighbour within the normal radius, so no descriptor and no match at all."""
    g = np.stack(np.meshgrid(np.arange(6), np.arange(6), np.arange(2)), -1).reshape(-1, 3) * 50.0
    return np.c_[g, np.zeros(len(g))].astype(np.float32)


def _cfg(**kv):
    import b200reg
    cfg = b200reg.default_loop_config()
    for k, v in kv.items():
        setattr(cfg, k, v)
    return cfg


def _opt(native, max_corres):
    prm = native.default_quatro_params()
    prm.max_corres = max_corres
    return prm


def _adv(native):
    prm = native.default_quatro_params()
    prm.use_optimized_matching = 0
    return prm


def _recorded(ctx, call):
    """call() on the session context with recording on -> (its return value, the matches)."""
    ctx.set_quatro_matches(True)
    try:
        out = call()
        return out, ctx.quatro_matches()
    finally:
        ctx.set_quatro_matches(False)


def _rows_equal(a, b):
    return len(a) == len(b) and all(all(x[k].shape == y[k].shape and x[k].tobytes() == y[k].tobytes() for k in KEYS)
                                    for x, y in zip(a, b))


def _tap_path(n, advanced):
    if not advanced:
        return "shared" if n <= MAXC else "global"
    return "global" if n <= ADV_CAP else "wide"


def _check_pair(ctx, oracle, row, info, spts, dpts, advanced, prm):
    """One pair's row against quatro_align_ex's info, the solve tap on the path the call used, the oracle and the points."""
    corr = info["corr"]
    assert np.array_equal(row["corr"], corr)
    assert row["inlier"].shape == (len(corr),) and set(np.unique(row["inlier"])) <= {0, 1}
    assert int(row["inlier"].sum()) == info["clique_size"]
    S, D = spts[corr[:, 0]], dpts[corr[:, 1]]
    assert row["src_xyz"].tobytes() == np.ascontiguousarray(S).tobytes()
    assert row["dst_xyz"].tobytes() == np.ascontiguousarray(D).tobytes()
    if len(corr) == 0:
        return
    inl = np.flatnonzero(row["inlier"])
    tap = ctx.quatro_solve_tap(S, D, params=prm, path=_tap_path(len(corr), advanced))
    assert np.array_equal(inl, tap["clique"]) and tap["clique_size"] == info["clique_size"]
    assert tap["T"].tobytes() == info["T"].tobytes()
    o = oracle.quatro_solve(S, D, np.repeat(np.arange(len(corr), dtype=np.int32)[:, None], 2, 1))
    assert np.array_equal(inl, o["clique"])


# ---------------------------------------------------------------------------------------------------------------------
# raw-buffer calls: all three solve paths
@pytest.fixture(scope="module")
def opt_pairs(synth):
    """A valid pair, the structureless pair (nothing kept: invalid), a pair without a single descriptor, a 50k pair whose
    set passes 512 at max_corres 1000."""
    a, b = _blobs()
    sp = _sparse()
    good = synth.make_pair(2005, 3000, 2500, mode="quatro")[:2]
    big = synth.make_pair(2004, 50000, 50000, mode="quatro")[:2]
    return [good[0], a, sp, big[0]], [good[1], b, sp.copy(), big[1]]


@pytest.mark.gpu
@pytest.mark.parametrize("max_corres", [200, 1000])
def test_optimized_matching_rows(ctx, native, oracle, opt_pairs, max_corres):
    prm = _opt(native, max_corres)
    cl = ctx.create_clouds(opt_pairs[0] + opt_pairs[1])
    cs, cd = cl[:4], cl[4:]
    try:
        infos, rows = _recorded(ctx, lambda: ctx.quatro_align(cs, cd, params=prm, want_corr=True))
        pts = [ctx.cloud_points(c) for c in cl]
    finally:
        for c in cl:
            c.destroy()
    n = [i["n_corr"] for i in infos]
    assert infos[0]["valid"] and not infos[1]["valid"] and n[0] > 0 and n[2] == 0
    assert (n[3] > MAXC) == (max_corres == 1000)
    assert len(rows) == 4
    for i in range(4):
        _check_pair(ctx, oracle, rows[i], infos[i], pts[i], pts[4 + i], False, prm)


@pytest.mark.gpu
def test_invalid_solve_with_a_clique_of_at_most_one(ctx, native, oracle, opt_pairs):
    """A noise bound far below the pair's noise leaves the consistency graph without edges: the solve is invalid with a
    clique of one, and exactly that one row is an inlier."""
    prm = _opt(native, 200)
    prm.noise_bound = 1e-9
    cl = ctx.create_clouds([opt_pairs[0][0], opt_pairs[1][0]])
    try:
        (info,), rows = _recorded(ctx, lambda: ctx.quatro_align(cl[:1], cl[1:], params=prm, want_corr=True))
        pts = [ctx.cloud_points(c) for c in cl]
    finally:
        for c in cl:
            c.destroy()
    assert info["n_corr"] > 0 and not info["valid"] and info["clique_size"] <= 1
    corr = info["corr"]
    S, D = pts[0][corr[:, 0]], pts[1][corr[:, 1]]
    tap = ctx.quatro_solve_tap(S, D, params=prm, path="shared")
    assert np.array_equal(np.flatnonzero(rows[0]["inlier"]), tap["clique"]) and len(tap["clique"]) == info["clique_size"]


@pytest.fixture(scope="module")
def wide_pair():
    from test_gpu_quatro_big import make_submap_pair
    return make_submap_pair()[:2]


@pytest.mark.gpu
def test_advanced_matching_rows_with_a_wide_pair(ctx, native, oracle, synth, wide_pair):
    """advancedMatching: a pair beyond 8192 correspondences (the one-pair wide chain) between a batched valid pair and the
    structureless pair, and the wide pair again swapped, so that the shared workspace is reused."""
    a, b = _blobs()
    good = synth.make_pair(2010, 30000, 30000, mode="quatro", voxel=0.3)[:2]
    srcs = [good[0], wide_pair[0], a, wide_pair[1]]
    dsts = [good[1], wide_pair[1], b, wide_pair[0]]
    prm = _adv(native)
    cl = ctx.create_clouds(srcs + dsts)
    try:
        infos, rows = _recorded(ctx, lambda: ctx.quatro_align(cl[:4], cl[4:], params=prm, want_corr=True))
        pts = [ctx.cloud_points(c) for c in cl]
    finally:
        for c in cl:
            c.destroy()
    assert infos[1]["n_corr"] > ADV_CAP and infos[3]["n_corr"] > ADV_CAP and infos[0]["n_corr"] <= ADV_CAP
    assert infos[0]["valid"] and infos[1]["valid"] and not infos[2]["valid"]
    for i in range(4):
        _check_pair(ctx, oracle, rows[i], infos[i], pts[i], pts[4 + i], True, prm)


@pytest.mark.gpu
def test_recording_changes_nothing_and_off_launches_nothing(ctx, native, opt_pairs):
    """quatro_align_ex and loop_closure with recording off, on and off: identical bytes; off launches what off launched,
    on adds exactly the capture launch; LM traces and loop clouds are unchanged by it."""
    prm = _opt(native, 1000)
    cl = ctx.create_clouds(opt_pairs[0] + opt_pairs[1])
    ctx.fpfh(cl)  # computed once per cloud: the calls below launch only the match and solve
    try:
        def align(on):
            ctx.set_quatro_matches(on)
            l0 = ctx.launch_count
            out = ctx.quatro_align(cl[:4], cl[4:], params=prm, want_corr=True)
            ctx.set_quatro_matches(False)
            return [(o["T"].tobytes(), o["corr"].tobytes(), o["valid"], o["n_corr"], o["clique_size"]) for o in out], ctx.launch_count - l0
        off, n_off = align(False)
        on, n_on = align(True)
        off2, n_off2 = align(False)
        assert off == on == off2 and n_off == n_off2 and n_on == n_off + 1
    finally:
        for c in cl:
            c.destroy()

    def lc(on):
        ctx.set_quatro_matches(on)
        ctx.set_lm_trace(True)
        ctx.set_loop_clouds(15)
        try:
            l0 = ctx.launch_count
            res, qi = ctx.loop_closure(opt_pairs[0], opt_pairs[1], qparams=prm)
            n = ctx.launch_count - l0
            tr = ctx.lm_trace()
            clouds = [ctx.loop_clouds(k) for k in (4, 8)]
        finally:
            ctx.set_quatro_matches(False)
            ctx.set_lm_trace(False)
            ctx.set_loop_clouds(0)
        key = ([(r["T"].tobytes(), r["converged"]) for r in res], [(q["T"].tobytes(), q["clique_size"]) for q in qi],
               b"".join(t.tobytes() for t in tr), [b"".join(r.tobytes() for r in k) for k in clouds])
        return key, n
    lc(False)  # the LM arena and graph at this batch size
    k_off, n_off = lc(False)
    k_on, n_on = lc(True)
    assert k_off == k_on and n_on == n_off + 1


@pytest.mark.gpu
def test_loop_closure_rows_equal_quatro_align(ctx, native, opt_pairs):
    """b200reg_loop_closure records once, over the caller's pairs: the rows of quatro_align on the same clouds."""
    prm = _opt(native, 1000)
    (_, qi), rows = _recorded(ctx, lambda: ctx.loop_closure(opt_pairs[0], opt_pairs[1], qparams=prm))
    cl = ctx.create_clouds(opt_pairs[0] + opt_pairs[1])
    try:
        _, want = _recorded(ctx, lambda: ctx.quatro_align(cl[:4], cl[4:], params=prm))
    finally:
        for c in cl:
            c.destroy()
    assert _rows_equal(rows, want)
    assert [int(r["inlier"].sum()) for r in rows] == [q["clique_size"] for q in qi]


# ---------------------------------------------------------------------------------------------------------------------
# the keyframe path
@pytest.fixture(scope="module")
def seq(synth):
    """The loop-capable sequence plus two structureless keyframes far away (140, 141) whose pair fails the coarse stage."""
    s = synth.make_sequence(7, NKF, pts_per_keyframe=6000, spacing=3.0, speed=8.0)
    far = synth.se3(t=(5000.0, 0.0, 0.0))
    return list(s["clouds"]) + list(_blobs()), list(s["poses"]) + [far, far], list(s["stamps"]) + [1000.0, 1001.0]


@pytest.fixture(scope="module")
def store(ctx, seq):
    kf = ctx.keyframes()
    for c, T, t in zip(*seq):
        kf.add(c, T, t)
    yield kf
    kf.destroy()


def _queries(store):
    q = np.array(QUERIES + [141], np.int32)
    closest = np.append(store.fetch_closest(np.array(QUERIES, np.int32)), 140).astype(np.int32)
    return q, closest


@pytest.mark.gpu
def test_keyframe_path_rows_in_caller_order(ctx, store, native):
    """Quatro mode: a query without a candidate has an empty row; every other row is quatro_align_ex's answer on the
    assembled clouds, its points are rows of the SOURCE and TARGET loop clouds of the same call, its inliers number the
    pair's clique_size.  GICP-only mode: every row is empty."""
    q, closest = _queries(store)
    cfg = _cfg()
    ctx.set_loop_clouds(SOURCE | TARGET)
    try:
        (_, qi), rows = _recorded(ctx, lambda: store.perform_loop_closure(q, closest, cfg))
        src_rows, tgt_rows = ctx.loop_clouds(SOURCE), ctx.loop_clouds(TARGET)
    finally:
        ctx.set_loop_clouds(0)
    assert len(rows) == len(q) and closest[2] == -1 and len(rows[2]["corr"]) == 0
    assert not qi[4]["valid"] and any(x["valid"] for x in qi[:2])
    has = [i for i in range(len(q)) if closest[i] >= 0]
    cs, cd = store.assemble(q[has], closest[has], cfg, n_keyframes=q[has] + 1)  # the sub-maps perform_loop_closure builds
    try:
        want = ctx.quatro_align(cs, cd, params=cfg.quatro, want_corr=True)
    finally:
        for c in cs + cd:
            c.destroy()
    for k, i in enumerate(has):
        r = rows[i]
        assert np.array_equal(r["corr"], want[k]["corr"]), i
        assert int(r["inlier"].sum()) == qi[i]["clique_size"] == want[k]["clique_size"], i
        assert r["src_xyz"].tobytes() == np.ascontiguousarray(src_rows[i][r["corr"][:, 0], :3]).tobytes(), i
        assert r["dst_xyz"].tobytes() == np.ascontiguousarray(tgt_rows[i][r["corr"][:, 1], :3]).tobytes(), i
    _, none = _recorded(ctx, lambda: store.perform_loop_closure(q, closest, _cfg(enable_quatro=0)))
    assert len(none) == len(q) and all(len(r["corr"]) == 0 for r in none)
    _, none = _recorded(ctx, lambda: store.perform_loop_closure(np.array([20], np.int32), np.array([-1], np.int32), cfg))
    assert len(none) == 1 and len(none[0]["corr"]) == 0


@pytest.mark.gpu
def test_getter_state_and_capacity_rules(ctx, store, native, opt_pairs):
    import b200reg
    lib = native.lib()
    q, closest = _queries(store)

    def rc(c, off=None, cap=0, bufs=(None, None, None, None)):
        p = [None if b is None else b.ctypes.data_as(C.c_void_p) for b in bufs]
        return lib.b200reg_quatro_matches(c.h, None if off is None else off.ctypes.data_as(C.c_void_p), C.c_size_t(cap), *p)

    fresh = b200reg.Context(0)
    try:
        assert rc(fresh) == ESTATE  # before any recording call
    finally:
        fresh.close()
    assert lib.b200reg_ctx_set_quatro_matches(None, 1) == EINVAL
    _, rows = _recorded(ctx, lambda: store.perform_loop_closure(q, closest))
    total = sum(len(r["corr"]) for r in rows)
    # the capacity rule: offsets only; any output may be NULL
    off = np.full(len(q) + 1, -7, np.int64)
    bufs = (np.full((total, 2), -7, np.int32), np.full(total, -7, np.int32), np.full((total, 3), -7, np.float32),
            np.full((total, 3), -7, np.float32))
    assert rc(ctx, off, total - 1, bufs) == ESTATE
    assert off.tolist() == np.cumsum([0] + [len(r["corr"]) for r in rows]).tolist() and all((b == -7).all() for b in bufs)
    assert rc(ctx) == len(q)
    for k in range(4):
        part = tuple(b if j == k else None for j, b in enumerate(bufs))
        assert rc(ctx, off, total, part) == 0
        assert bufs[k].tobytes() == b"".join(r[KEYS[k]].tobytes() for r in rows)
    # the tap and the calls without a Quatro stage leave them; a failing call and a call with recording off drop them
    ctx.set_quatro_matches(True)
    try:
        r = next(r for r in rows if len(r["corr"]))
        ctx.quatro_solve_tap(r["src_xyz"], r["dst_xyz"], path="shared")
        ctx.icp_alignment([opt_pairs[0][0]], [opt_pairs[1][0]])
        assert _rows_equal(ctx.quatro_matches(), rows)
        bad = _cfg()
        bad.quatro.estimate_scale = 1
        with pytest.raises(native.B200RegError):
            store.perform_loop_closure(q, closest, bad)
        assert rc(ctx) == ESTATE and "failed" in lib.b200reg_last_error().decode()
        store.perform_loop_closure(q, closest)
        assert _rows_equal(ctx.quatro_matches(), rows)
    finally:
        ctx.set_quatro_matches(False)
    store.perform_loop_closure(q, closest)
    assert rc(ctx) == ESTATE


# ---------------------------------------------------------------------------------------------------------------------
# batch-driver jobs
class Spec:
    def __init__(self, name, ctx_call, submit):
        self.name, self.ctx_call, self.submit = name, ctx_call, submit


@pytest.fixture(scope="module")
def jobs(ctx, store, opt_pairs):
    """Every recording job kind with what the context returns after the synchronous call."""
    q, closest = _queries(store)
    srcs = [np.ascontiguousarray(a, np.float32) for a in opt_pairs[0]]
    dsts = [np.ascontiguousarray(a, np.float32) for a in opt_pairs[1]]
    args = ([a.ctypes.data for a in srcs], [len(a) for a in srcs], [a.ctypes.data for a in dsts], [len(a) for a in dsts], 16, 0)
    specs = [Spec("loop_closure", lambda: ctx.loop_closure_ptrs(*args), lambda b: b.submit_loop_closure(*args))]
    specs[0].buffers = (srcs, dsts)
    for mode, kv in (("quatro", {}), ("gicp_only", {"enable_quatro": 0})):
        cfg = _cfg(**kv)
        specs.append(Spec("perform/%s/explicit" % mode, lambda c=cfg: store.perform_loop_closure(q, closest, c, raw=True),
                          lambda b, c=cfg: b.submit_perform_loop_closure(store, q, closest, c)))

        def searched(c=cfg):  # what a job with closest NULL runs: the candidate search, then the attempt
            return store.perform_loop_closure(q, store.fetch_closest(q, c.loop_detection_radius, c.loop_detection_timediff_threshold),
                                              c, raw=True)
        specs.append(Spec("perform/%s/searched" % mode, searched, lambda b, c=cfg: b.submit_perform_loop_closure(store, q, None, c)))
    return [(s, _recorded(ctx, s.ctx_call)) for s in specs]


def _same_records(got, want):
    return bytes(got[0]) == bytes(want[0]) and bytes(got[1]) == bytes(want[1])


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 3, 6])
def test_jobs_return_the_bytes_of_the_synchronous_call(jobs, depth):
    import b200reg
    batch = b200reg.Batch(0, depth=depth)
    try:
        batch.set_quatro_matches(True)
        tickets = [s.submit(batch) for s, _ in jobs]
        for (s, (out, rows)), t in reversed(list(zip(jobs, tickets))):
            assert _same_records(batch.wait(t, want_quatro=True), out), (s.name, depth)
            assert _rows_equal(batch.quatro_matches(t), rows), (s.name, depth)
            batch.release(t)
    finally:
        batch.close()


@pytest.mark.gpu
def test_mixed_settings_and_settings_taken_at_submit(jobs, native):
    """Settings alternate over a burst, so each worker runs recording and non-recording jobs back to back, and the setting
    changes right after each submit; jobs are waited for out of order.  Each job returns its own matches or none."""
    import b200reg
    lib = native.lib()
    batch = b200reg.Batch(0, depth=3)
    try:
        sub = []
        for rnd in range(2):
            for i, (s, want) in enumerate(jobs):
                on = (i + rnd) % 2 == 0
                batch.set_quatro_matches(on)
                t = s.submit(batch)
                batch.set_quatro_matches(not on)  # changed after submit: does not reach the job
                sub.append((s, want, on, t))
        order = list(range(len(sub)))
        for k in order[1::2] + order[0::2][::-1]:
            s, (out, rows), on, t = sub[k]
            assert _same_records(batch.wait(t, want_quatro=True), out), s.name
            if on:
                assert _rows_equal(batch.quatro_matches(t), rows), s.name
            else:
                assert lib.b200reg_batch_quatro_matches(batch.h, C.c_int64(t), None, C.c_size_t(0), None, None, None, None) == ESTATE
                assert "did not record" in lib.b200reg_last_error().decode()
    finally:
        batch.close()


@pytest.mark.gpu
def test_job_lifetime_and_errors(ctx, store, jobs, opt_pairs, native):
    import b200reg
    lib = native.lib()
    spec, (_, want) = next((s, w) for s, w in jobs if s.name == "perform/quatro/explicit")

    def rc(b, t):
        return lib.b200reg_batch_quatro_matches(b.h, C.c_int64(t), None, C.c_size_t(0), None, None, None, None)

    def message():
        return lib.b200reg_last_error().decode()

    batch = b200reg.Batch(0, depth=1)
    try:
        batch.set_quatro_matches(True)
        t = [spec.submit(batch) for _ in range(2)]
        assert rc(batch, t[1]) == ESTATE and "not been waited for" in message()
        for bad in (-1, t[1] + 1, 10 ** 9):
            assert rc(batch, bad) == EINVAL
        batch.wait(t[0])
        assert rc(batch, t[0]) == len(QUERIES) + 1
        assert _rows_equal(batch.quatro_matches(t[0]), want)
        assert lib.b200reg_batch_release(batch.h, C.c_int64(t[0])) == 0
        assert rc(batch, t[0]) == ESTATE and "released" in message()
        # an icpAlignment job has no Quatro stage
        src = np.ascontiguousarray(opt_pairs[0][0], np.float32)
        dst = np.ascontiguousarray(opt_pairs[1][0], np.float32)
        t_icp = batch.submit_icp([src.ctypes.data], [len(src)], [dst.ctypes.data], [len(dst)], 16, 0)
        batch.wait(t_icp)
        assert rc(batch, t_icp) == ESTATE and "did not record" in message()
        # a job refused inside its worker keeps nothing
        bad = _cfg()
        bad.quatro.estimate_scale = 1
        q, closest = _queries(store)
        t_bad = batch.submit_perform_loop_closure(store, q, closest, bad)
        with pytest.raises(b200reg.B200RegError):
            batch.wait(t_bad)
        assert rc(batch, t_bad) == ESTATE and "failed" in message()
        # destroyed with t[1] still held
        batch.wait(t[1])
        assert _rows_equal(batch.quatro_matches(t[1]), want)
    finally:
        batch.close()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_client_matches_binding(tmp_path, ctx, seq, store):
    exe = _build_client(str(tmp_path))
    clouds, poses, stamps = seq
    clouds, poses, stamps = clouds[:NKF], poses[:NKF], stamps[:NKF]
    path = str(tmp_path / "keyframes.bin")
    with open(path, "wb") as f:
        f.write(np.int32(len(clouds)).tobytes())
        for cl, T, t in zip(clouds, poses, stamps):
            cl = np.ascontiguousarray(cl, np.float32)
            f.write(np.int64(len(cl)).tobytes() + np.ascontiguousarray(T, np.float64).tobytes() + np.float64(t).tobytes() + cl.tobytes())
    prefix = str(tmp_path / "out")
    got = json.loads(subprocess.check_output([exe, path, prefix] + [str(x) for x in QUERIES], timeout=600).decode())
    q = np.array(QUERIES, np.int32)
    closest = store.fetch_closest(q)
    (_, qi), rows = _recorded(ctx, lambda: store.perform_loop_closure(q, closest))
    assert got["closest"] == closest.tolist() and got["clique_size"] == [x["clique_size"] for x in qi]
    offsets = np.cumsum([0] + [len(r["corr"]) for r in rows]).tolist()
    blob = b"".join(b"".join(r[k].tobytes() for r in rows) for k in KEYS)
    for who in ("ctx", "job"):
        assert got[who] == offsets
        with open("%s_%s.bin" % (prefix, who), "rb") as f:
            assert f.read() == blob, who
    assert got["released"] == 0 and got["after_release"] == ESTATE
