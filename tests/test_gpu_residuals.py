"""Per-point residuals of the fitness pass (b200reg_ctx_set_residuals / b200reg_residuals, b200reg_batch_set_residuals /
b200reg_batch_residuals, NanoGICP::getFitnessScore(max_range)): each source point's nearest target point and fp32 squared
distance at the final pose equal an exact 1-NN of the oracle, bit for bit; rows follow the caller's pairs with empty rows
where no fine stage ran, and address the SOURCE / TARGET loop clouds on the keyframe path; nothing changes and nothing is
launched with recording off; driver jobs return the bytes of the synchronous call; and the facade's
getFitnessScore(max_range) equals PCL's rule summed over the oracle's distances."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(REPO, "fast-lio-sam-qn_b200", "host")
CSRC = os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc")
CLIENT_SRC = os.path.join(REPO, "tests", "cpp", "residuals_client.cpp")
MOCK_PCL = os.path.join(REPO, "tests", "cpp", "mock_pcl")
EINVAL, ESTATE = -1, -4
SOURCE, TARGET, COARSE, FINAL = 1, 2, 4, 8
QUERIES = [137, 139, 20, 118]  # 20 has no candidate; the others close loops at the start of the lap
NKF = 140  # keyframes of the sequence; 140 and 141 are the structureless far pair
DBL_MAX = sys.float_info.max


def _build_client(tmp, pcl_config=False):
    from b200reg.build import build_native
    build_native()
    exe = os.path.join(tmp, "residuals_client_pcl" if pcl_config else "residuals_client")
    extra = ["-I" + MOCK_PCL, "-DB200REG_EXPECT_PCL"] if pcl_config else []
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-I" + HOST] + extra + ["-o", exe, CLIENT_SRC,
                           "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    return exe


@pytest.mark.parametrize("pcl_config", [False, True])
def test_residuals_client_compiles(tmp_path, pcl_config):
    """getFitnessScore(max_range) / lastResiduals through the facade compile as C++14 in both type configurations (no GPU
    needed)."""
    assert os.path.exists(_build_client(str(tmp_path), pcl_config))


def _pcl_score(d2, max_range):
    """pcl::Registration::getFitnessScore(max_range), restated: keep d2 <= max_range, float64 sum in point order."""
    s, nr = 0.0, 0
    for v in np.asarray(d2, np.float32):
        if float(v) <= max_range:
            s += float(v)
            nr += 1
    return s / nr if nr else DBL_MAX


def test_fitness_score_helper():
    from b200reg import fitness_score
    d2 = np.array([0.5, 2.0, 0.25, 3.0, 0.0], np.float32)
    for r in (0.0, -1.0, 0.25, 0.5, 2.0, 1.5, float("inf"), float("nan"), DBL_MAX):
        assert fitness_score(d2, r) == _pcl_score(d2, r), r
    assert fitness_score(d2, 0.5) == 0.75 / 3 and fitness_score(d2, -1.0) == DBL_MAX and fitness_score(d2, float("nan")) == DBL_MAX
    assert fitness_score(np.zeros(0, np.float32), 1.0) == DBL_MAX


# ---------------------------------------------------------------------------------------------------------------------
# GPU
def _recorded(ctx, call):
    """call() on the context with recording on -> (its return value, the rows)."""
    ctx.set_residuals(True)
    try:
        out = call()
        return out, ctx.residuals()
    finally:
        ctx.set_residuals(False)


def _rows_equal(a, b):
    return len(a) == len(b) and all(x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() and len(x[0]) == len(y[0])
                                    for x, y in zip(a, b))


def _check_rows(oracle, nn, d2, tgt_xyz, q_xyz):
    """The rows of one pair against the oracle's exact 1-NN of the final-pose source points q_xyz in the target."""
    oi, od = oracle.knn(np.ascontiguousarray(tgt_xyz, np.float32), np.ascontiguousarray(q_xyz, np.float32), 1)
    assert nn.dtype == np.int32 and d2.dtype == np.float32 and len(nn) == len(q_xyz)
    assert np.array_equal(nn, oi[:, 0])
    assert d2.tobytes() == od[:, 0].tobytes()


@pytest.fixture(scope="module")
def icp_pairs(synth):
    """A 20k pair and a 100k pair."""
    a = synth.make_pair(1000, 20000)
    b = synth.make_pair(1003, 100000, 100000)
    return [a[0], b[0]], [a[1], b[1]]


@pytest.mark.gpu
def test_icp_alignment_rows_equal_the_oracle(ctx, oracle, icp_pairs):
    srcs, dsts = icp_pairs
    res, rows = _recorded(ctx, lambda: ctx.icp_alignment(srcs, dsts))
    assert len(rows) == 2
    for i in range(2):
        nn, d2 = rows[i]
        _check_rows(oracle, nn, d2, dsts[i][:, :3], oracle.transform_output(res[i]["Tf"], srcs[i]))
        fit = res[i]["fitness"]
        assert abs(np.sum(d2.astype(np.float64)) / len(d2) - fit) <= 1e-12 * abs(fit), i


@pytest.mark.gpu
def test_gicp_align_with_guesses(ctx, native, oracle, synth, icp_pairs):
    """b200reg_gicp_align records: with guesses against the oracle at the result's pose; without, the bytes of
    icp_alignment on the same buffers."""
    srcs, dsts = [p[:8000] for p in icp_pairs[0][:1]] * 2, [p for p in icp_pairs[1][:1]] * 2
    guesses = np.stack([np.eye(4), synth.se3(yaw=0.05, t=(0.3, -0.2, 0.0))])
    cl = ctx.create_clouds(srcs + dsts)
    try:
        res, rows = _recorded(ctx, lambda: ctx.gicp_align(cl[:2], cl[2:], guesses=guesses))
        res0, rows0 = _recorded(ctx, lambda: ctx.gicp_align(cl[:2], cl[2:]))
    finally:
        for c in cl:
            c.destroy()
    for i in range(2):
        _check_rows(oracle, rows[i][0], rows[i][1], dsts[i][:, :3], oracle.transform_output(res[i]["Tf"], srcs[i]))
    _, want = _recorded(ctx, lambda: ctx.icp_alignment(srcs, dsts))
    assert _rows_equal(rows0, want)


def _blobs():
    rng = np.random.default_rng(0)  # no structure at FPFH radii: Quatro finds no valid solution
    return rng.normal(0, 20, (300, 4)).astype(np.float32), rng.normal(0, 20, (280, 4)).astype(np.float32)


@pytest.fixture(scope="module")
def lc_pairs(synth):
    """Voxelised loop-closure pairs: two valid ones around the structureless pair (an invalid Quatro solve)."""
    a, b = _blobs()
    p1 = synth.make_pair(2000, 30000, 30000, mode="quatro", voxel=0.3)[:2]
    p2 = synth.make_pair(2005, 3000, 2500, mode="quatro")[:2]
    return [p1[0], a, p2[0]], [p1[1], b, p2[1]]


@pytest.mark.gpu
def test_loop_closure_rows(ctx, oracle, lc_pairs):
    """Empty rows where the coarse stage is invalid; elsewhere the oracle's 1-NN of the FINAL loop cloud (the fine stage's
    output cloud, rows of the caller's source) in the caller's target."""
    srcs, dsts = lc_pairs
    ctx.set_loop_clouds(FINAL)
    try:
        (res, qi), rows = _recorded(ctx, lambda: ctx.loop_closure(srcs, dsts))
        final = ctx.loop_clouds(FINAL)
    finally:
        ctx.set_loop_clouds(0)
    assert [q["valid"] for q in qi] == [True, False, True]
    assert len(rows) == 3 and len(rows[1][0]) == 0 and len(rows[1][1]) == 0
    for i in (0, 2):
        assert len(rows[i][0]) == len(srcs[i])
        _check_rows(oracle, rows[i][0], rows[i][1], dsts[i][:, :3], final[i][:, :3])
        assert abs(np.sum(rows[i][1].astype(np.float64)) / len(srcs[i]) - res[i]["fitness"]) <= 1e-12 * res[i]["fitness"]


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


def _cfg(**kv):
    import b200reg
    cfg = b200reg.default_loop_config()
    for k, v in kv.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["quatro", "gicp_only"])
def test_keyframe_path_rows_address_the_loop_clouds(ctx, oracle, store, mode):
    """Rows in caller order: empty for the query without a candidate and (Quatro mode) for the invalid coarse stage;
    every other row is a row of the SOURCE loop cloud, its nn a row of the TARGET loop cloud, and the pair is the
    oracle's 1-NN of the FINAL loop cloud (the same rows as SOURCE) in TARGET."""
    q, closest = _queries(store)
    cfg = _cfg() if mode == "quatro" else _cfg(enable_quatro=0)
    ctx.set_loop_clouds(SOURCE | TARGET | FINAL)
    try:
        (res, qi), rows = _recorded(ctx, lambda: store.perform_loop_closure(q, closest, cfg))
        clouds = {k: ctx.loop_clouds(k) for k in (SOURCE, TARGET, FINAL)}
    finally:
        ctx.set_loop_clouds(0)
    assert len(rows) == len(q) and closest[2] == -1
    ran = [closest[i] >= 0 and (mode == "gicp_only" or qi[i]["valid"]) for i in range(len(q))]
    if mode == "quatro":
        assert not qi[4]["valid"] and not ran[4]
    assert sum(ran) >= 2
    for i in range(len(q)):
        nn, d2 = rows[i]
        if not ran[i]:
            assert len(nn) == 0 and len(d2) == 0, i
            continue
        assert len(nn) == len(clouds[SOURCE][i]) == len(clouds[FINAL][i]), i
        _check_rows(oracle, nn, d2, clouds[TARGET][i][:, :3], clouds[FINAL][i][:, :3])
        assert abs(np.sum(d2.astype(np.float64)) / len(d2) - res[i]["fitness"]) <= 1e-12 * res[i]["fitness"], i
    _, none = _recorded(ctx, lambda: store.perform_loop_closure(np.array([20], np.int32), np.array([-1], np.int32), cfg))
    assert len(none) == 1 and len(none[0][0]) == 0


@pytest.mark.gpu
def test_recording_changes_nothing_and_off_launches_nothing(ctx, native, icp_pairs, lc_pairs, store):
    """Every recording call with recording off launches what the same call launches on a context that never recorded;
    on adds exactly the capture launch; results, LM traces, loop clouds and Quatro matches keep their bytes."""
    import b200reg
    q, closest = _queries(store)
    fresh = b200reg.Context(0)
    try:
        calls = {
            "icp": lambda c, kf: c.icp_alignment(icp_pairs[0][:1], icp_pairs[1][:1], raw=True),
            "loop_closure": lambda c, kf: c.loop_closure(*lc_pairs),
            "perform": lambda c, kf: kf.perform_loop_closure(q, closest, raw=True),
        }

        def run(c, kf, name, on):
            c.set_residuals(on)
            c.set_lm_trace(True)
            c.set_quatro_matches(True)
            c.set_loop_clouds(15)
            try:
                l0 = c.launch_count
                out = calls[name](c, kf)
                n = c.launch_count - l0
                tr = c.lm_trace()
                qm = c.quatro_matches() if name != "icp" else []
                clouds = [c.loop_clouds(k) for k in (SOURCE, TARGET, COARSE, FINAL)] if name != "icp" else [c.loop_clouds(FINAL)]
            finally:
                c.set_residuals(False)
                c.set_lm_trace(False)
                c.set_quatro_matches(False)
                c.set_loop_clouds(0)
            if name == "loop_closure":
                res = [(r["T"].tobytes(), r["Tf"].tobytes(), r["fitness"], r["converged"], r["valid"]) for r in out[0]]
                res.append([(x["T"].tobytes(), x["clique_size"]) for x in out[1]])
            elif name == "perform":
                res = [bytes(out[0]), bytes(out[1])]
            else:
                res = [bytes(out)]
            key = (res, b"".join(t.tobytes() for t in tr), [b"".join(r.tobytes() for r in k) for k in clouds],
                   [b"".join(m[k].tobytes() for k in ("corr", "inlier", "src_xyz", "dst_xyz")) for m in qm])
            return key, n

        for name in calls:
            kf = store if name == "perform" else None
            run(ctx, kf, name, False)  # the LM arena and graph at this batch size
            k_off, n_off = run(ctx, kf, name, False)
            k_on, n_on = run(ctx, kf, name, True)
            assert k_off == k_on, name
            assert n_on == n_off + 1, name
            if name != "perform":  # the keyframe path runs the same solve code on its assembled clouds
                fresh.set_lm_trace(True)
                fresh.set_quatro_matches(True)
                fresh.set_loop_clouds(15)
                try:
                    l0 = fresh.launch_count
                    calls[name](fresh, None)
                    assert fresh.launch_count - l0 == n_off, name
                finally:
                    fresh.set_lm_trace(False)
                    fresh.set_quatro_matches(False)
                    fresh.set_loop_clouds(0)
    finally:
        fresh.close()


@pytest.mark.gpu
def test_getter_state_and_capacity_rules(ctx, native, icp_pairs, store):
    import b200reg
    lib = native.lib()
    srcs, dsts = [icp_pairs[0][0][:5000], icp_pairs[0][0][:3000]], [icp_pairs[1][0], icp_pairs[1][0]]

    def rc(c, off=None, cap=0, nn=None, d2=None):
        p = [None if b is None else b.ctypes.data_as(C.c_void_p) for b in (off, nn, d2)]
        return lib.b200reg_residuals(c.h if c is not None else None, p[0], C.c_size_t(cap), p[1], p[2])

    fresh = b200reg.Context(0)
    try:
        assert rc(fresh) == ESTATE  # before any recording call
    finally:
        fresh.close()
    assert rc(None) == EINVAL and lib.b200reg_ctx_set_residuals(None, 1) == EINVAL
    assert lib.b200reg_batch_set_residuals(None, 1) == EINVAL
    assert lib.b200reg_batch_residuals(None, C.c_int64(0), None, C.c_size_t(0), None, None) == EINVAL
    _, rows = _recorded(ctx, lambda: ctx.icp_alignment(srcs, dsts))
    total = sum(len(r[0]) for r in rows)
    assert total == 8000
    off = np.full(3, -7, np.int64)
    nn, d2 = np.full(total, -7, np.int32), np.full(total, -7, np.float32)
    assert rc(ctx, off, total - 1, nn, d2) == ESTATE  # capacity: offsets only
    assert off.tolist() == [0, 5000, 8000] and (nn == -7).all() and (d2 == -7).all()
    assert rc(ctx) == 2
    assert rc(ctx, off, total, nn, None) == 0 and nn.tobytes() == b"".join(r[0].tobytes() for r in rows) and (d2 == -7).all()
    assert rc(ctx, off, total, None, d2) == 0 and d2.tobytes() == b"".join(r[1].tobytes() for r in rows)
    # Quatro alone and the taps leave them; a failing call and a call with recording off drop them
    ctx.set_residuals(True)
    try:
        cl = ctx.create_clouds([srcs[0], dsts[0]])
        try:
            ctx.quatro_align(cl[:1], cl[1:])
            ctx.knn(cl[1], srcs[0][:100], 1)
            ctx.covariances(cl, 15)
            ctx.linearize(cl[0], cl[1], np.eye(4))
        finally:
            for c in cl:
                c.destroy()
        assert _rows_equal(ctx.residuals(), rows)
        q, closest = _queries(store)
        bad = _cfg()
        bad.quatro.estimate_scale = 1
        with pytest.raises(native.B200RegError):
            store.perform_loop_closure(q, closest, bad)
        assert rc(ctx) == ESTATE and "failed" in lib.b200reg_last_error().decode()
        ctx.icp_alignment(srcs, dsts)
        assert _rows_equal(ctx.residuals(), rows)
        bad_prm = b200reg.default_params()
        with pytest.raises(native.B200RegError):  # refused: an empty cloud
            ctx.icp_alignment_ptrs([0], [0], [0], [0], 16, 0, bad_prm)
        assert rc(ctx) == ESTATE
    finally:
        ctx.set_residuals(False)
    _recorded(ctx, lambda: ctx.icp_alignment(srcs, dsts))
    ctx.icp_alignment(srcs, dsts)
    assert rc(ctx) == ESTATE


# ---------------------------------------------------------------------------------------------------------------------
# batch-driver jobs
class Spec:
    def __init__(self, name, ctx_call, submit):
        self.name, self.ctx_call, self.submit = name, ctx_call, submit


@pytest.fixture(scope="module")
def jobs(ctx, store, icp_pairs, lc_pairs):
    """Every job kind with what the context returns after the synchronous call."""
    q, closest = _queries(store)
    isrc = [np.ascontiguousarray(icp_pairs[0][0][:6000], np.float32), np.ascontiguousarray(icp_pairs[0][0][:4000], np.float32)]
    idst = [np.ascontiguousarray(icp_pairs[1][0], np.float32)] * 2
    iargs = ([a.ctypes.data for a in isrc], [len(a) for a in isrc], [a.ctypes.data for a in idst], [len(a) for a in idst], 16, 0)
    srcs = [np.ascontiguousarray(a, np.float32) for a in lc_pairs[0]]
    dsts = [np.ascontiguousarray(a, np.float32) for a in lc_pairs[1]]
    args = ([a.ctypes.data for a in srcs], [len(a) for a in srcs], [a.ctypes.data for a in dsts], [len(a) for a in dsts], 16, 0)
    specs = [Spec("icp", lambda: ctx.icp_alignment_ptrs(*iargs), lambda b: b.submit_icp(*iargs)),
             Spec("loop_closure", lambda: ctx.loop_closure_ptrs(*args), lambda b: b.submit_loop_closure(*args))]
    specs[0].buffers = (isrc, idst)
    specs[1].buffers = (srcs, dsts)
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
    if isinstance(want, tuple):
        return bytes(got[0]) == bytes(want[0]) and bytes(got[1]) == bytes(want[1])
    return bytes(got) == bytes(want)


def _wait(batch, s, t):
    return batch.wait(t) if s.name == "icp" else batch.wait(t, want_quatro=True)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 3, 6])
def test_jobs_return_the_bytes_of_the_synchronous_call(jobs, depth):
    import b200reg
    batch = b200reg.Batch(0, depth=depth)
    try:
        batch.set_residuals(True)
        tickets = [s.submit(batch) for s, _ in jobs]
        for (s, (out, rows)), t in reversed(list(zip(jobs, tickets))):
            assert _same_records(_wait(batch, s, t), out), (s.name, depth)
            assert _rows_equal(batch.residuals(t), rows), (s.name, depth)
            batch.release(t)
    finally:
        batch.close()


@pytest.mark.gpu
def test_mixed_settings_and_settings_taken_at_submit(jobs, native):
    """Settings alternate over a burst, so each worker runs recording and non-recording jobs back to back, and the setting
    changes right after each submit; jobs are waited for out of order.  Each job returns its own rows or none."""
    import b200reg
    lib = native.lib()
    batch = b200reg.Batch(0, depth=3)
    try:
        sub = []
        for rnd in range(2):
            for i, (s, want) in enumerate(jobs):
                on = (i + rnd) % 2 == 0
                batch.set_residuals(on)
                t = s.submit(batch)
                batch.set_residuals(not on)  # changed after submit: does not reach the job
                sub.append((s, want, on, t))
        order = list(range(len(sub)))
        for k in order[1::2] + order[0::2][::-1]:
            s, (out, rows), on, t = sub[k]
            assert _same_records(_wait(batch, s, t), out), s.name
            if on:
                assert _rows_equal(batch.residuals(t), rows), s.name
            else:
                assert lib.b200reg_batch_residuals(batch.h, C.c_int64(t), None, C.c_size_t(0), None, None) == ESTATE
                assert "did not record" in lib.b200reg_last_error().decode()
    finally:
        batch.close()


@pytest.mark.gpu
def test_job_lifetime_and_errors(store, jobs, native):
    import b200reg
    lib = native.lib()
    spec, (_, want) = next((s, w) for s, w in jobs if s.name == "perform/quatro/explicit")

    def rc(b, t):
        return lib.b200reg_batch_residuals(b.h, C.c_int64(t), None, C.c_size_t(0), None, None)

    def message():
        return lib.b200reg_last_error().decode()

    batch = b200reg.Batch(0, depth=1)
    try:
        batch.set_residuals(True)
        t = [spec.submit(batch) for _ in range(2)]
        assert rc(batch, t[1]) == ESTATE and "not been waited for" in message()
        for bad in (-1, t[1] + 1, 10 ** 9):
            assert rc(batch, bad) == EINVAL
        batch.wait(t[0])
        assert rc(batch, t[0]) == len(QUERIES) + 1
        assert _rows_equal(batch.residuals(t[0]), want)
        assert lib.b200reg_batch_release(batch.h, C.c_int64(t[0])) == 0
        assert rc(batch, t[0]) == ESTATE and "released" in message()
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
        assert _rows_equal(batch.residuals(t[1]), want)
    finally:
        batch.close()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_facade_fitness_score_at_ranges(tmp_path, oracle, icp_pairs):
    """NanoGICP::align then getFitnessScore(r) for r in {0, below the smallest d2, the median d2, 1.5, +inf, NaN}: each
    equals PCL's rule summed in float64 over the oracle's d2 at the facade's final pose, bit for bit; DBL_MAX returns the
    result's fitness."""
    exe = _build_client(str(tmp_path))
    src, dst = icp_pairs[0][0], icp_pairs[1][0]
    paths = []
    for name, a in (("src", src), ("dst", dst)):
        p = str(tmp_path / (name + ".bin"))
        np.ascontiguousarray(a, np.float32).tofile(p)
        paths.append(p)
    # the ranges the client is given first, those that depend on the distances after the facade's pose is known
    got = json.loads(subprocess.check_output([exe] + paths + ["0"], timeout=600).decode())
    Tf = np.array(got["Tf"], np.float32).reshape(4, 4)
    _, od = oracle.knn(np.ascontiguousarray(dst[:, :3]), oracle.transform_output(Tf, src), 1)
    d2 = od[:, 0]
    ranges = [0.0, float(np.nextafter(np.float64(d2.min()), -np.inf)), float(np.median(d2.astype(np.float64))), 1.5,
              float("inf"), float("nan"), DBL_MAX]
    got = json.loads(subprocess.check_output([exe] + paths + [repr(r) for r in ranges], timeout=600).decode())
    assert np.array(got["Tf"], np.float32).reshape(4, 4).tobytes() == Tf.tobytes()
    assert got["rows"] == got["nn_rows"] == len(src)
    want = [_pcl_score(d2, r) for r in ranges[:-1]]
    assert got["scores"][:-1] == want
    assert got["scores"][1] == DBL_MAX and got["scores"][5] == DBL_MAX and got["scores"][4] != DBL_MAX
    assert got["scores"][-1] == got["fitness"]
    assert abs(got["scores"][4] - got["fitness"]) <= 1e-12 * got["fitness"]
