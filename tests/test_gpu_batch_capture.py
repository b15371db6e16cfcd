"""Loop clouds and LM traces of batch-driver jobs (b200reg_batch_set_loop_clouds / _set_lm_trace, b200reg_batch_loop_clouds /
_lm_trace, b200reg_batch_release): byte identity with what a context returns after the synchronous call, for all three job
kinds at depths 1, 3 and 6; results unchanged by capture and launches unchanged with it off; jobs of mixed settings on one
worker; the settings and the store copied at submit; the lifetime and error rules; and a C++ client that publishes
loopTimerFunc's debug topics from driver jobs through the ABI alone."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc")
CLIENT_SRC = os.path.join(REPO, "tests", "cpp", "batch_capture_client.cpp")
EINVAL, ESTATE = -1, -4
SOURCE, TARGET, COARSE, FINAL = 1, 2, 4, 8
KINDS = (SOURCE, TARGET, COARSE, FINAL)
QUERIES = [137, 139, 20, 118]  # 20 has no candidate; the others close loops at the start of the lap
NKF = 140  # keyframes of the sequence; 140 and 141 are the structureless far pair


def _build_client(tmp):
    exe = os.path.join(tmp, "batch_capture_client")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-pthread", "-o", exe, CLIENT_SRC,
                           "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    return exe


def test_batch_capture_client_compiles(tmp_path):
    """The ABI alone is enough to publish the four clouds and the trace from driver jobs (no GPU needed to build)."""
    from b200reg.build import build_native
    build_native()
    assert os.path.exists(_build_client(str(tmp_path)))


def _records(x4, stride):
    """(n, 4) x, y, z, intensity -> packed xyzi (16 bytes) or pcl::PointXYZI records (32 bytes: x, y, z, 1, i, pad)."""
    if stride == 16:
        return np.ascontiguousarray(x4, np.float32)
    r = np.zeros((len(x4), 8), np.float32)
    r[:, :3], r[:, 3], r[:, 4] = x4[:, :3], 1.0, x4[:, 3]
    return r


def _blobs():
    rng = np.random.default_rng(0)  # no structure at FPFH radii: Quatro finds no valid solution
    return rng.normal(0, 20, (300, 4)).astype(np.float32), rng.normal(0, 20, (280, 4)).astype(np.float32)


def _cfg(**kv):
    import b200reg
    cfg = b200reg.default_loop_config()
    for k, v in kv.items():
        setattr(cfg, k, v)
    return cfg


CFGS = {"quatro": {}, "gicp_only": {"enable_quatro": 0}, "submap": {"enable_submap_matching": 1}}


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


@pytest.fixture(scope="module")
def raw(synth):
    """Raw-buffer pairs: three icpAlignment pairs, and two coarse-to-fine pairs around a structureless one."""
    icp = [synth.make_pair(1100 + i, 4000 + 500 * i, 5000 - 300 * i) for i in range(3)]
    qp = [synth.make_pair(2100 + i, 5000 + 400 * i, 6000 - 300 * i, mode="quatro") for i in range(2)]
    a, b = _blobs()
    return dict(icp=([p[0] for p in icp], [p[1] for p in icp]), lc=([qp[0][0], a, qp[1][0]], [qp[0][1], b, qp[1][1]]))


class Spec:
    """One job: how to run it on a context and how to submit it to a driver.  Keeps its raw buffers alive."""

    def __init__(self, name, ctx_call, submit):
        self.name, self.ctx_call, self.submit = name, ctx_call, submit


def _specs(ctx, store, raw):
    q = np.array(QUERIES + [141], np.int32)
    closest = np.append(store.fetch_closest(np.array(QUERIES, np.int32)), 140).astype(np.int32)
    specs = []
    for stride in (16, 32):
        for kind, key in (("icp", "icp"), ("loop_closure", "lc")):
            srcs = [_records(x, stride) for x in raw[key][0]]
            dsts = [_records(x, stride) for x in raw[key][1]]
            args = ([a.ctypes.data for a in srcs], [len(a) for a in srcs], [a.ctypes.data for a in dsts], [len(a) for a in dsts], stride, 0)
            if kind == "icp":
                ctx_call = lambda a=args: (ctx.icp_alignment_ptrs(*a), None)
                submit = lambda b, a=args: b.submit_icp(*a)
            else:
                ctx_call = lambda a=args: ctx.loop_closure_ptrs(*a)
                submit = lambda b, a=args: b.submit_loop_closure(*a)
            s = Spec("%s/%d" % (kind, stride), ctx_call, submit)
            s.buffers = (srcs, dsts)
            specs.append(s)
    for mode, kv in CFGS.items():
        cfg = _cfg(**kv)
        specs.append(Spec("perform/%s/explicit" % mode, lambda c=cfg: store.perform_loop_closure(q, closest, c, raw=True),
                          lambda b, c=cfg: b.submit_perform_loop_closure(store, q, closest, c)))

        def searched(c=cfg):  # what a job with closest NULL runs: the candidate search, then the attempt
            cl = store.fetch_closest(q, c.loop_detection_radius, c.loop_detection_timediff_threshold)
            return store.perform_loop_closure(q, cl, c, raw=True)
        specs.append(Spec("perform/%s/searched" % mode, searched, lambda b, c=cfg: b.submit_perform_loop_closure(store, q, None, c)))
    return specs


def _outputs(res_qi, clouds, trace):
    res, qi = res_qi
    return dict(res=bytes(res), qi=None if qi is None else bytes(qi), qi_records=qi, clouds=clouds, trace=trace)


def _sync(ctx, spec, mask=15, trace=True):
    """The synchronous call on the session context with the given settings -> what its getters return."""
    ctx.set_loop_clouds(mask)
    ctx.set_lm_trace(trace)
    try:
        out = spec.ctx_call()
        clouds = {k: ctx.loop_clouds(k) for k in KINDS if mask & k}
        tr = ctx.lm_trace() if trace else None
    finally:
        ctx.set_loop_clouds(0)
        ctx.set_lm_trace(False)
    return _outputs(out, clouds, tr)


def _job(batch, t, mask=15, trace=True):
    """A waited-for job's records and what the driver's getters return for it."""
    res = batch.wait(t, want_quatro=True)
    clouds = {k: batch.loop_clouds(t, k) for k in KINDS if mask & k}
    tr = batch.lm_trace(t) if trace else None
    return _outputs(res, clouds, tr)


def _rows_equal(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _assert_same(got, want, name, qi=True):
    assert got["res"] == want["res"], name
    if qi and want["qi"] is not None:
        assert got["qi"] == want["qi"], name
    assert set(got["clouds"]) == set(want["clouds"]), name
    for k in want["clouds"]:
        assert _rows_equal(got["clouds"][k], want["clouds"][k]), (name, k)
    assert (got["trace"] is None) == (want["trace"] is None), name
    if want["trace"] is not None:
        assert _rows_equal(got["trace"], want["trace"]), name


@pytest.fixture(scope="module")
def jobs(ctx, store, raw):
    """Every job spec with what the synchronous call returns with all four kinds and tracing on."""
    specs = _specs(ctx, store, raw)
    return [(s, _sync(ctx, s)) for s in specs]


# ---------------------------------------------------------------------------------------------------------------------
# GPU
@pytest.mark.gpu
def test_workload_has_every_row_shape(jobs):
    """The perform jobs hold a query without a candidate, a pair whose Quatro stage is invalid and a valid one; the raw
    coarse-to-fine jobs an invalid coarse stage; the icpAlignment jobs empty SOURCE / TARGET / COARSE rows."""
    want = dict((s.name, w) for s, w in jobs)
    p = want["perform/quatro/explicit"]
    sizes = [len(r) for r in p["clouds"][SOURCE]]
    assert sizes[2] == 0 and all(n > 0 for i, n in enumerate(sizes) if i != 2)
    valid = [x.valid for x in (p["qi_records"])]
    finals = [len(r) for r in p["clouds"][FINAL]]
    assert not valid[4] and finals[4] == 0  # the structureless pair: no fine stage
    assert any(valid[i] and finals[i] > 0 for i in (0, 1, 3))
    assert [len(r) > 0 for r in want["loop_closure/16"]["clouds"][COARSE]] == [True, False, True]
    for k in (SOURCE, TARGET, COARSE):
        assert [len(r) for r in want["icp/32"]["clouds"][k]] == [0, 0, 0]
    assert all(len(t) > 0 for t in want["icp/16"]["trace"])


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 3, 6])
def test_jobs_return_the_bytes_of_the_synchronous_call(jobs, depth):
    import b200reg
    batch = b200reg.Batch(0, depth=depth)
    try:
        batch.set_loop_clouds(15)
        batch.set_lm_trace(True)
        tickets = [s.submit(batch) for s, _ in jobs]
        for (s, want), t in reversed(list(zip(jobs, tickets))):
            _assert_same(_job(batch, t), want, (s.name, depth))
            batch.release(t)
    finally:
        batch.close()


@pytest.mark.gpu
def test_capture_changes_no_record_and_off_adds_no_launch(ctx, jobs):
    """The job list with capture off, on and off again: identical result and Quatro bytes; with it off the driver launches
    what the synchronous calls launch on a context, and keeps nothing."""
    import b200reg
    from b200reg import native
    lib = native.lib()
    l0 = ctx.launch_count
    for s, _ in jobs:
        s.ctx_call()
    sync_launches = ctx.launch_count - l0
    batch = b200reg.Batch(0, depth=3)
    try:
        def run(on):
            batch.set_loop_clouds(15 if on else 0)
            batch.set_lm_trace(on)
            l0 = batch.launch_count
            tickets = [s.submit(batch) for s, _ in jobs]
            out = [batch.wait(t, want_quatro=True) for t in tickets]
            return [(bytes(r), None if q is None else bytes(q)) for r, q in out], batch.launch_count - l0, tickets
        off, n_off, t_off = run(False)
        on, n_on, _ = run(True)
        off2, n_off2, _ = run(False)
        assert off == on == off2
        assert n_off == n_off2 == sync_launches and n_on > n_off
        for t in t_off:
            assert lib.b200reg_batch_loop_clouds(batch.h, C.c_int64(t), FINAL, None, C.c_size_t(0), None) == ESTATE
            assert "did not capture" in lib.b200reg_last_error().decode()
            assert lib.b200reg_batch_lm_trace(batch.h, C.c_int64(t), None, C.c_size_t(0), None) == ESTATE
            assert "not traced" in lib.b200reg_last_error().decode()
            assert lib.b200reg_batch_release(batch.h, C.c_int64(t)) == 0
    finally:
        batch.wait_all()
        batch.close()


@pytest.mark.gpu
def test_mixed_settings_back_to_back(ctx, jobs, native):
    """One burst whose settings alternate (all kinds + trace, off, FINAL only, trace only) over the perform jobs, so that
    each worker runs mixed settings back to back; waited for out of order.  Each job returns exactly its own kinds and
    trace, equal to the synchronous call with the same settings; everything else is B200REG_ESTATE."""
    import b200reg
    lib = native.lib()
    settings = [(15, True), (0, False), (FINAL, False), (0, True)]
    perform = [(s, w) for s, w in jobs if s.name.startswith("perform/")]
    batch = b200reg.Batch(0, depth=3)
    try:
        sub = []
        for rnd in range(2):
            for i, (s, want) in enumerate(perform):
                mask, trace = settings[(i + rnd) % len(settings)]
                batch.set_loop_clouds(mask)
                batch.set_lm_trace(trace)
                sub.append((s, want, mask, trace, s.submit(batch)))
        order = list(range(len(sub)))
        order = order[1::2] + order[0::2][::-1]
        for k in order:
            s, want, mask, trace, t = sub[k]
            got = _job(batch, t, mask, trace)
            expect = dict(want, clouds={c: want["clouds"][c] for c in KINDS if mask & c}, trace=want["trace"] if trace else None)
            _assert_same(got, expect, (s.name, mask, trace))
            for c in KINDS:
                if not mask & c:
                    assert lib.b200reg_batch_loop_clouds(batch.h, C.c_int64(t), c, None, C.c_size_t(0), None) == ESTATE
            if not trace:
                assert lib.b200reg_batch_lm_trace(batch.h, C.c_int64(t), None, C.c_size_t(0), None) == ESTATE
    finally:
        batch.close()  # with every output still held


@pytest.mark.gpu
def test_settings_and_poses_are_taken_at_submit(ctx, store, seq, jobs, synth, native):
    """Poses rewritten and capture switched off after the submit: the job's SOURCE / TARGET rows are those of the
    synchronous call at the old poses, and it still captures; a job submitted after the switch captures nothing."""
    import b200reg
    lib = native.lib()
    spec, want = next((s, w) for s, w in jobs if s.name == "perform/quatro/explicit")
    poses = seq[1]
    batch = b200reg.Batch(0, depth=3)
    try:
        batch.set_loop_clouds(15)
        batch.set_lm_trace(True)
        t = spec.submit(batch)
        batch.set_loop_clouds(0)
        batch.set_lm_trace(False)
        for i in range(len(poses)):  # a drift correction that grows along the trajectory
            store.set_pose(i, synth.se3(yaw=2e-4 * i, t=(0.01 * i, -0.005 * i, 0.0)) @ poses[i])
        t_after = spec.submit(batch)
        _assert_same(_job(batch, t), want, "snapshot")
        moved = _sync(ctx, spec)
        assert not _rows_equal(moved["clouds"][SOURCE], want["clouds"][SOURCE]), "the rewritten poses move the clouds"
        batch.wait(t_after)
        for c in KINDS:
            assert lib.b200reg_batch_loop_clouds(batch.h, C.c_int64(t_after), c, None, C.c_size_t(0), None) == ESTATE
        assert lib.b200reg_batch_lm_trace(batch.h, C.c_int64(t_after), None, C.c_size_t(0), None) == ESTATE
    finally:
        for i in range(len(poses)):
            store.set_pose(i, poses[i])
        batch.wait_all()
        batch.close()


@pytest.mark.gpu
def test_lifetime_and_errors(ctx, store, jobs, native):
    import b200reg
    lib = native.lib()
    spec, want = next((s, w) for s, w in jobs if s.name == "perform/quatro/explicit")

    def clouds_rc(b, t, kind=FINAL, off=None, cap=0, buf=None):
        return lib.b200reg_batch_loop_clouds(b.h, C.c_int64(t), kind, None if off is None else off.ctypes.data_as(C.c_void_p),
                                             C.c_size_t(cap), None if buf is None else buf.ctypes.data_as(C.c_void_p))

    def trace_rc(b, t):
        return lib.b200reg_batch_lm_trace(b.h, C.c_int64(t), None, C.c_size_t(0), None)

    def release_rc(b, t):
        return lib.b200reg_batch_release(b.h, C.c_int64(t))

    def message():
        return lib.b200reg_last_error().decode()

    batch = b200reg.Batch(0, depth=1)
    try:
        batch.set_loop_clouds(15)
        batch.set_lm_trace(True)
        t = [spec.submit(batch) for _ in range(3)]
        # before the wait
        assert clouds_rc(batch, t[2]) == ESTATE and "not been waited for" in message()
        assert trace_rc(batch, t[2]) == ESTATE and "not been waited for" in message()
        assert release_rc(batch, t[2]) == ESTATE
        # tickets never handed out
        for bad in (-1, t[2] + 1, 10 ** 9):
            assert clouds_rc(batch, bad) == EINVAL and trace_rc(batch, bad) == EINVAL and release_rc(batch, bad) == EINVAL
        _assert_same(_job(batch, t[0]), want, "first")
        # kinds that are not one bit
        for bad in (0, 3, 16, -1):
            assert clouds_rc(batch, t[0], bad) == EINVAL
        assert lib.b200reg_batch_set_loop_clouds(batch.h, 16) == EINVAL
        # the capacity rule: offsets only
        total = sum(len(r) for r in want["clouds"][SOURCE])
        off = np.full(len(QUERIES) + 2, -7, np.int64)
        buf = np.full((total, 4), -7, np.float32)
        assert clouds_rc(batch, t[0], SOURCE, off, total - 1, buf) == ESTATE
        assert off.tolist() == np.cumsum([0] + [len(r) for r in want["clouds"][SOURCE]]).tolist() and (buf == -7).all()
        assert clouds_rc(batch, t[0], SOURCE, off, total, buf) == 0
        assert buf.tobytes() == b"".join(r.tobytes() for r in want["clouds"][SOURCE])
        assert clouds_rc(batch, t[0], SOURCE) == len(QUERIES) + 1  # offsets_out NULL: the pair count
        # release, twice
        assert release_rc(batch, t[0]) == 0 and release_rc(batch, t[0]) == 0
        assert clouds_rc(batch, t[0]) == ESTATE and "released" in message()
        assert trace_rc(batch, t[0]) == ESTATE and "released" in message()
        # b200reg_batch_wait_all keeps the outputs; Batch.wait_all releases what it drops
        assert lib.b200reg_batch_wait_all(batch.h) == 0
        _assert_same(_outputs((batch._keep[t[1]][0], batch._keep[t[1]][1]), {k: batch.loop_clouds(t[1], k) for k in KINDS},
                              batch.lm_trace(t[1])), want, "wait_all")
        t4 = spec.submit(batch)
        batch.wait_all()
        assert clouds_rc(batch, t4) == ESTATE and "released" in message()
        # a job refused inside its worker keeps nothing; its wait carries the message
        bad = _cfg()
        bad.quatro.estimate_scale = 1
        q = np.array(QUERIES, np.int32)
        t_bad = batch.submit_perform_loop_closure(store, q, store.fetch_closest(q), bad)
        with pytest.raises(b200reg.B200RegError) as e:
            batch.wait(t_bad)
        assert "estimate_scale" in str(e.value)
        assert clouds_rc(batch, t_bad) == ESTATE and "failed" in message()
        assert trace_rc(batch, t_bad) == ESTATE and "failed" in message()
        assert release_rc(batch, t_bad) == 0
        # the driver keeps working; its last outputs stay unreleased when it is destroyed
        t5 = spec.submit(batch)
        _assert_same(_job(batch, t5), want, "after the failure")
    finally:
        batch.close()
    assert batch.h is None


@pytest.mark.gpu
def test_client_matches_binding(tmp_path, ctx, seq, store):
    """The C++ client's loopTimerFunc on the driver publishes, per tick, what the synchronous call on a context returns."""
    exe = _build_client(str(tmp_path))
    clouds, poses, stamps = seq
    queries = np.array([137, 139, 20, 118, 130, 135], np.int32)
    nk, per_tick = int(queries.max()) + 1, 2
    np.ascontiguousarray(np.stack(clouds[:nk]), np.float32).tofile(str(tmp_path / "clouds.bin"))
    np.ascontiguousarray(poses[:nk], np.float64).tofile(str(tmp_path / "poses.bin"))
    np.ascontiguousarray(stamps[:nk], np.float64).tofile(str(tmp_path / "stamps.bin"))
    queries.tofile(str(tmp_path / "queries.bin"))
    txt = subprocess.check_output([exe, str(tmp_path), str(nk), str(len(clouds[0])), str(len(queries)), str(per_tick), "3"],
                                  timeout=600).decode()
    out = json.loads([ln for ln in txt.splitlines() if ln.startswith("{")][-1])
    assert out["status"] == 0 and len(out["ticks"]) == len(queries) // per_tick
    for k, tick in enumerate(out["ticks"]):
        q = queries[per_tick * k:per_tick * (k + 1)]
        spec = Spec("tick", lambda q=q: store.perform_loop_closure(q, store.fetch_closest(q), raw=True), None)
        want = _sync(ctx, spec)
        assert tick["tick"] == k and tick["status"] == 0 and tick["released"] == 0 and tick["after_release"] == ESTATE
        assert bytes.fromhex(tick["results"]) == want["res"] and bytes.fromhex(tick["quatro"]) == want["qi"]
        for c in KINDS:
            rows = want["clouds"][c]
            assert tick["offsets"][str(c)] == np.cumsum([0] + [len(r) for r in rows]).tolist()
            assert (tmp_path / ("tick%d_%d.bin" % (k, c))).read_bytes() == b"".join(r.tobytes() for r in rows)
        assert tick["trace_offsets"] == np.cumsum([0] + [len(r) for r in want["trace"]]).tolist()
        assert (tmp_path / ("tick%d_trace.bin" % k)).read_bytes() == b"".join(r.tobytes() for r in want["trace"])
