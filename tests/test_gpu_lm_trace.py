"""The LM trace of the device solve (b200reg_ctx_set_lm_trace / b200reg_lm_trace, NanoGICP::setDebugPrint): one record per
trial of step_lm (lsq_registration_impl.hpp:170-205).  Tracing changes no result; the records agree with the result
counters, with the reference's lambda / nu rules and with the CPU oracle's trials (tests/lm_trials.py)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import lm_trials

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(REPO, "fast-lio-sam-qn_b200", "host")
CSRC = os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc")
CLIENT_SRC = os.path.join(REPO, "tests", "cpp", "lm_trace_client.cpp")
MOCK_PCL = os.path.join(REPO, "tests", "cpp", "mock_pcl")
ESTATE = -4

# one parameter set for both solvers: the deployment's (loop_closure.cpp:10-14, lsq_registration_impl.hpp:53-59)
DEFAULTS = dict(k_correspondences=15, max_iterations=32, max_corr_dist=52.5, transformation_eps=0.01, rotation_eps=2e-3,
                lm_max_iterations=10, lm_init_lambda_factor=1e-9)
# variants that reach every decision: lm_max_iterations 1 fails on the first rejection (3); with huge epsilons a rejected
# step already counts as converged (2)
VARIANTS = {"default": {}, "one_trial": dict(lm_max_iterations=1), "wide_eps": dict(transformation_eps=10.0, rotation_eps=10.0)}


def _params(**kv):
    import b200reg
    from oracle.oracle import GicpParams
    p, o = b200reg.default_params(), GicpParams.default()
    for k, v in dict(DEFAULTS, **kv).items():
        setattr(p, k, v)
        setattr(o, k, v)
    return p, o


def _build_client(tmp, pcl_config=False):
    from b200reg.build import build_native
    build_native()
    exe = os.path.join(tmp, "lm_client_pcl" if pcl_config else "lm_client")
    extra = ["-I" + MOCK_PCL, "-DB200REG_EXPECT_PCL"] if pcl_config else []
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-I" + HOST] + extra + ["-o", exe, CLIENT_SRC,
                           "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    return exe


@pytest.mark.parametrize("pcl_config", [False, True])
def test_lm_trace_client_compiles(tmp_path, pcl_config):
    """setDebugPrint / lastLmTrace through the facade compile as C++14 in both type configurations (no GPU needed)."""
    assert os.path.exists(_build_client(str(tmp_path), pcl_config))


def test_lm_trial_struct_size(native):
    assert native.lib().b200reg_struct_size(6) == C.sizeof(native.LmTrial) == native.LM_TRIAL_DTYPE.itemsize == 200


# ---------------------------------------------------------------------------------------------------------------------
# GPU
@pytest.fixture(scope="module")
def batch(synth):
    """8 pairs of 4k-20k points: the 32-iteration divergent pair of the batch test, pairs that stop after 2 to 16 outer
    iterations, and one started 0.8 rad off (rejected trials).  -> (srcs, dsts, guesses)"""
    specs = [((1104, 6000, 3800), None), ((1000, 20000), None), ((1001, 5000, 6000), None), ((1100, 4000, 5000), None),
             ((1101, 4500, 4700), None), ((1104, 5000, 5000), synth.se3(yaw=0.8, t=(1.0, 0.0, 0.0))),
             ((1102, 8000, 9000), synth.se3(yaw=0.3, t=(1.0, 0.0, 0.0))), ((1103, 12000, 11000), None)]
    pairs = [synth.make_pair(*a) for a, _ in specs]
    guesses = np.stack([np.eye(4) if g is None else g for _, g in specs])
    return [p[0] for p in pairs], [p[1] for p in pairs], guesses


def _solve(ctx, batch, prm, trace, profiling=False):
    """-> (raw Result bytes, launches, trace or None)"""
    from b200reg import native
    srcs, dsts, guesses = batch
    clouds = ctx.create_clouds(srcs + dsts)
    cs, ct = clouds[:len(srcs)], clouds[len(srcs):]
    ctx.covariances(clouds, 15)
    ctx.set_lm_trace(trace)
    ctx.set_profiling(profiling)
    n = len(cs)
    res = (native.Result * n)()
    g = np.ascontiguousarray(guesses, np.float64)
    l0 = ctx.launch_count
    try:
        native._check(native.lib().b200reg_gicp_align(ctx.h, n, (C.c_void_p * n)(*[c.h for c in cs]), (C.c_void_p * n)(*[c.h for c in ct]),
                                                      g.ctypes.data_as(C.c_void_p), C.byref(prm), res))
        launches = ctx.launch_count - l0
        tr = ctx.lm_trace() if trace else None
    finally:
        ctx.set_lm_trace(False)
        ctx.set_profiling(False)
        for c in clouds:
            c.destroy()
    return bytes(res), launches, tr, [r.as_dict() for r in res]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_tracing_changes_nothing(ctx, native, batch, variant):
    prm, _ = _params(**VARIANTS[variant])
    off_bytes, off_launches, _, _ = _solve(ctx, batch, prm, False)
    on_bytes, on_launches, tr, _ = _solve(ctx, batch, prm, True)
    assert on_bytes == off_bytes and on_launches == off_launches
    # an untraced solve discards the stored trace
    _solve(ctx, batch, prm, False)
    with pytest.raises(native.B200RegError):
        ctx.lm_trace()
    # the host-polled launch mode writes the same records
    prof_bytes, _, tr_prof, _ = _solve(ctx, batch, prm, True, profiling=True)
    assert prof_bytes == off_bytes
    assert len(tr) == len(tr_prof) and all(a.tobytes() == b.tobytes() for a, b in zip(tr, tr_prof))


@pytest.mark.gpu
def test_trace_agrees_with_result(ctx, batch):
    seen = set()
    for variant in sorted(VARIANTS):
        prm, _ = _params(**VARIANTS[variant])
        _, _, tr, res = _solve(ctx, batch, prm, True)
        for t, r in zip(tr, res):
            assert len(t) == r["n_error"] > 0
            assert len(np.unique(t["outer"])) == r["n_linearize"] and t["outer"].max() == r["iterations"]
            assert (np.diff(t["outer"]) >= 0).all() and (t["reserved"] == 0).all()
            last = t[-1]
            if r["converged"]:
                assert last["decision"] == 2 or (last["decision"] == 1 and lm_trials.is_converged(_delta(last), prm.rotation_eps, prm.transformation_eps))
            assert (last["decision"] == 3) == r["lm_failed"]
            assert (t["decision"][:-1] != 3).all() and (t["decision"][:-1] != 2).all()
            assert np.array_equal(last["T"], r["T"][:3]), "the pose of the last record is the result, bit for bit"
            _check_lambda_nu(t, prm)
            seen.update(t["decision"].tolist())
    assert seen == {0, 1, 2, 3}


def _delta(rec):
    D = np.eye(4)
    D[:3, :3] = lm_trials.so3_exp(rec["d"][:3])
    D[:3, 3] = rec["d"][3:]
    return D


def _check_lambda_nu(t, prm):
    """Replays the reference's lambda / nu updates (lsq_registration_impl.hpp:165-167, 196-204) from record to record."""
    for k in range(len(t)):
        r = t[k]
        if k == 0 or r["outer"] != t[k - 1]["outer"]:
            assert r["trial"] == 0 and r["nu"] == 2.0
        else:
            assert r["trial"] == t[k - 1]["trial"] + 1
        if k == 0:
            continue
        p = t[k - 1]
        if p["decision"] == 1:
            x = 2 * p["rho"] - 1
            want = p["lambda"] * max(1.0 / 3.0, 1 - x * x * x)
        else:
            want = p["nu"] * p["lambda"]
            assert r["nu"] == 2 * p["nu"]
        assert abs(r["lambda"] - want) <= 1e-15 * want


def _compare_with_oracle(g, o_recs):
    assert [(int(r["outer"]), int(r["trial"]), int(r["decision"])) for r in g] == [(r["outer"], r["trial"], r["decision"]) for r in o_recs]
    for a, b in zip(g, o_recs):
        assert abs(a["y0"] - b["y0"]) <= 1e-9 * abs(b["y0"]) and abs(a["yi"] - b["yi"]) <= 1e-9 * abs(b["yi"])
        nb = np.linalg.norm(b["d"])
        assert abs(np.linalg.norm(a["d"]) - nb) <= 1e-6 * nb
        if abs(b["y0"] - b["yi"]) > 1e-6 * b["y0"]:  # rho cancels near convergence
            assert abs(a["rho"] - b["rho"]) <= 1e-3 * abs(b["rho"])
        assert abs(a["lambda"] - b["lambda"]) <= 1e-6 * b["lambda"]
        assert np.abs(a["T"] - b["T"]).max() < 1e-6


@pytest.mark.gpu
def test_trace_agrees_with_oracle(ctx, oracle, synth, pair20k, pair5k):
    cases = [(pair20k[0], pair20k[1], None, {}), (pair5k[0], pair5k[1], None, {})]
    s, d, _ = synth.make_pair(1104, 5000, 5000)
    guess = synth.se3(yaw=0.8, t=(1.0, 0.0, 0.0))  # rejections far from convergence, where rho is large
    cases += [(s, d, guess, kv) for kv in VARIANTS.values()]
    big = synth.make_pair(1000, 100000)
    cases.append((big[0], big[1], None, {}))
    for src, dst, g, kv in cases:
        prm, oprm = _params(**kv)
        cs, ct = ctx.create_clouds([src, dst])
        ctx.set_lm_trace(True)
        try:
            ctx.gicp_align([cs], [ct], params=prm, guesses=None if g is None else [g])
            tr = ctx.lm_trace()[0]
        finally:
            ctx.set_lm_trace(False)
            cs.destroy(); ct.destroy()
        o_recs, _ = lm_trials.replay(oracle, src, dst, params=oprm, guess=g)
        _compare_with_oracle(tr, o_recs)


@pytest.mark.gpu
def test_trace_agrees_with_golden_oracle_trace(ctx):
    g = np.load(os.path.join(REPO, "tests", "golden", "gicp_oracle_3k.npz"))
    cs, ct = ctx.create_clouds([g["src"], g["dst"]])
    ctx.set_lm_trace(True)
    try:
        ctx.gicp_align([cs], [ct])
        t = ctx.lm_trace()[0]
    finally:
        ctx.set_lm_trace(False)
        cs.destroy(); ct.destroy()
    golden = g["trace"]
    firsts = np.flatnonzero(t["trial"] == 0)
    assert len(firsts) == len(golden) == int(g["n_linearize"]) and len(t) == int(g["n_error"])
    for k, i in enumerate(firsts):
        assert abs(t["y0"][i] - golden[k, 58]) <= 1e-9 * golden[k, 58]
        # the pose at linearization: the guess for the first outer iteration, then x0 after the previous trial
        pose = np.eye(4)[:3] if i == 0 else t["T"][i - 1]
        assert np.abs(pose - golden[k, :16].reshape(4, 4)[:3]).max() < 1e-6


def _rows_equal(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


@pytest.mark.gpu
def test_entry_points_give_caller_indexed_traces(ctx, synth):
    pairs = [synth.make_pair(1100 + i, 4000 + 500 * i, 5000 - 300 * i) for i in range(3)]
    srcs, dsts = [p[0] for p in pairs], [p[1] for p in pairs]
    ctx.set_lm_trace(True)
    try:
        res = ctx.icp_alignment(srcs, dsts)
        tr = ctx.lm_trace()
        singles = []
        for i in range(3):
            ctx.icp_alignment([srcs[i]], [dsts[i]])
            singles.append(ctx.lm_trace()[0])
        assert _rows_equal(tr, singles) and [len(t) for t in tr] == [r["n_error"] for r in res]
        # loop_closure: the fine stage runs on the pairs with a valid coarse stage only
        qpairs = [synth.make_pair(2100 + i, 5000 + 400 * i, 6000 - 300 * i, mode="quatro") for i in range(2)]
        rng = np.random.default_rng(0)
        blob_a = rng.normal(0, 20, (300, 4)).astype(np.float32)
        blob_b = rng.normal(0, 20, (280, 4)).astype(np.float32)
        qs, qd = [qpairs[0][0], blob_a, qpairs[1][0]], [qpairs[0][1], blob_b, qpairs[1][1]]
        res, qi = ctx.loop_closure(qs, qd)
        tr = ctx.lm_trace()
        assert [q["valid"] for q in qi] == [True, False, True]
        assert len(tr) == 3 and len(tr[1]) == 0 and [len(tr[0]), len(tr[2])] == [res[0]["n_error"], res[2]["n_error"]] and len(tr[0]) > 0
        for i in (0, 2):
            ctx.loop_closure([qs[i]], [qd[i]])
            assert _rows_equal([tr[i]], ctx.lm_trace())
        # only invalid coarse stages: no solve runs, every row is empty
        ctx.loop_closure([blob_a], [blob_b])
        assert [len(t) for t in ctx.lm_trace()] == [0]
    finally:
        ctx.set_lm_trace(False)


@pytest.mark.gpu
def test_perform_loop_closure_trace_rows(ctx, synth):
    seq = synth.make_sequence(7, 140, pts_per_keyframe=6000, spacing=3.0, speed=8.0)
    kf = ctx.keyframes()
    try:
        for c, T, t in zip(seq["clouds"], seq["poses"], seq["stamps"]):
            kf.add(c, T, t)
        queries = np.array([137, 139, 20, 118], np.int32)
        closest = kf.fetch_closest(queries)
        assert closest[2] == -1 and (closest[[0, 1, 3]] >= 0).all()
        import b200reg
        ctx.set_lm_trace(True)
        for quatro in (1, 0):
            cfg = b200reg.default_loop_config()
            cfg.enable_quatro = quatro
            res, qi = kf.perform_loop_closure(queries, closest, cfg)
            tr = ctx.lm_trace()
            assert len(tr) == 4 and len(tr[2]) == 0
            for k in (0, 1, 3):
                ran = not quatro or qi[k]["valid"]
                assert len(tr[k]) == (res[k]["n_error"] if ran else 0)
                kf.perform_loop_closure(queries[k:k + 1], closest[k:k + 1], cfg)
                assert _rows_equal([tr[k]], ctx.lm_trace())
            assert sum(len(t) > 0 for t in tr) >= 1
        kf.perform_loop_closure(queries[2:3], closest[2:3])  # no candidate: no solve, one empty row
        assert [len(t) for t in ctx.lm_trace()] == [0]
    finally:
        ctx.set_lm_trace(False)
        kf.destroy()


@pytest.mark.gpu
def test_abi_contract(synth):
    import b200reg
    from b200reg import native
    lib = native.lib()
    c = b200reg.Context(0)
    try:
        offsets = np.full(8, -7, np.int64)
        assert lib.b200reg_lm_trace(c.h, offsets.ctypes.data_as(C.c_void_p), C.c_size_t(100), None) == ESTATE  # before any traced solve
        assert (offsets == -7).all()
        src, dst, _ = synth.make_pair(1104, 5000, 5000)
        s2, d2, _ = synth.make_pair(1100, 4000, 5000)
        clouds = c.create_clouds([src, s2, dst, d2])
        c.set_lm_trace(True)
        c.gicp_align(clouds[:2], clouds[2:], guesses=[synth.se3(yaw=0.8, t=(1.0, 0.0, 0.0)), np.eye(4)])
        for cl in clouds:
            cl.destroy()
        assert lib.b200reg_lm_trace(c.h, None, C.c_size_t(0), None) == 2
        rows = c.lm_trace()
        total = sum(len(r) for r in rows)
        sentinel = np.frombuffer(bytes(range(256)) * (total * 200 // 256 + 1), np.uint8)[:total * 200].copy()
        buf = sentinel.copy()
        off = np.full(3, -7, np.int64)
        rc = lib.b200reg_lm_trace(c.h, off.ctypes.data_as(C.c_void_p), C.c_size_t(total - 1), buf.ctypes.data_as(C.c_void_p))
        assert rc == ESTATE and off.tolist() == [0, len(rows[0]), total] and np.array_equal(buf, sentinel)
        rc = lib.b200reg_lm_trace(c.h, off.ctypes.data_as(C.c_void_p), C.c_size_t(total), buf.ctypes.data_as(C.c_void_p))
        assert rc == 0 and buf.tobytes() == b"".join(r.tobytes() for r in rows)
        # a refused call and a call that fails in a stage both discard the trace
        with pytest.raises(native.B200RegError):  # an empty source cloud
            c.icp_alignment_ptrs([src.ctypes.data], [0], [dst.ctypes.data], [len(dst)], 16, False)
        assert lib.b200reg_lm_trace(c.h, None, C.c_size_t(0), None) == ESTATE
        kf = c.keyframes()
        try:
            kf.add(src, np.eye(4), 0.0)
            kf.add(dst, np.eye(4), 1.0)
            c.icp_alignment([src], [dst])
            assert lib.b200reg_lm_trace(c.h, None, C.c_size_t(0), None) == 1
            cfg = b200reg.default_loop_config()
            cfg.quatro.estimate_scale = 1  # refused by the Quatro stage, after sub-map assembly
            with pytest.raises(native.B200RegError):
                kf.perform_loop_closure([1], [0], cfg)
            assert lib.b200reg_lm_trace(c.h, None, C.c_size_t(0), None) == ESTATE
        finally:
            kf.destroy()
    finally:
        c.close()


@pytest.mark.gpu
def test_facade_prints_the_reference_table(tmp_path, ctx, synth):
    exe = _build_client(str(tmp_path))
    src, dst, _ = synth.make_pair(1104, 6000, 3800)
    sp, dp = str(tmp_path / "s.bin"), str(tmp_path / "d.bin")
    src.tofile(sp)
    dst.tofile(dp)
    out = subprocess.check_output([exe, sp, dp]).decode().splitlines()
    ctx.set_lm_trace(True)
    try:
        r = ctx.icp_alignment([src], [dst])[0]
        t = ctx.lm_trace()[0]
    finally:
        ctx.set_lm_trace(False)
    banner = "*" * 44
    assert out[:3] == [banner, "***************** optimize *****************", banner]
    header = "%5s %15s %15s %15s %15s %15s %5s" % ("i", "y0", "yi", "rho", "lambda", "|delta|", "dec")
    rows, k = [], 3
    while k < len(out) and not out[k].startswith("records "):
        if out[k] == "--- LM optimization ---":
            assert out[k + 1] == header
            rows.append("H")
            k += 2
            continue
        rows.append(out[k])
        k += 1
    assert out[k] == "records %d iterations %d lm_failed %d" % (len(t), r["iterations"], int(r["lm_failed"]))
    assert sum(x == "H" for x in rows) == r["n_linearize"]
    data = [x for x in rows if x != "H"]
    assert len(data) == len(t) == r["n_error"]
    j = 0
    for x in rows:  # one header per outer iteration, right before its trial 0
        if x == "H":
            assert t["trial"][j] == 0
            continue
        rec = t[j]
        m = re.fullmatch(r"(.{5}) (.{15}) (.{15}) (.{15}) (.{15}) (.{15}) (.{5})", x)
        assert m, x
        vals = [rec["y0"], rec["yi"], rec["rho"], rec["lambda"], np.sqrt(sum(float(v) * float(v) for v in rec["d"]))]
        assert int(m.group(1)) == rec["trial"]
        for got, want in zip(m.groups()[1:6], vals):
            assert got == "%15g" % want
        assert m.group(7) == "%5c" % ("x" if rec["rho"] > 0 else " ")
        j += 1
