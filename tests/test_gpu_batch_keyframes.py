"""Loop-closure attempts over the device keyframe store as jobs of the batch driver
(b200reg_batch_submit_perform_loop_closure): byte identity with b200reg_perform_loop_closure at every depth, the snapshot
taken at submit (pose rewrites, adds, interleaved ingest), the store's lifetime while jobs are in flight, the refusals at
submit, and a C++ client that uses the ABI alone."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc")
B = 16
NKF = 260  # spacing 2 m: the second pass of the street starts at ~150, about 100 keyframes have a loop candidate
MODES = {"quatro": (1, 0), "gicp_only": (0, 0), "submap": (1, 1)}  # (enable_quatro, enable_submap_matching)


@pytest.fixture(scope="module")
def seq(synth):
    return synth.make_sequence(5, NKF, pts_per_keyframe=30000, spacing=2.0, threads=max(1, min(8, os.cpu_count() or 1)))


def _store(ctx, seq, n, records=None):
    kf = ctx.keyframes()
    for i in range(n):
        kf.add(seq["clouds"][i] if records is None else records(i), seq["poses"][i], seq["stamps"][i])
    return kf


@pytest.fixture(scope="module")
def store(ctx, seq):
    kf = _store(ctx, seq, NKF)
    yield kf
    kf.destroy()


def _cfg(mode="quatro"):
    import b200reg
    cfg = b200reg.default_loop_config()
    cfg.enable_quatro, cfg.enable_submap_matching = MODES[mode]
    return cfg


def _candidates(kf, cfg):
    allq = np.arange(len(kf), dtype=np.int32)
    closest = kf.fetch_closest(allq, cfg.loop_detection_radius, cfg.loop_detection_timediff_threshold)
    return allq[closest >= 0], closest


def _bytes(res_qi):
    return bytes(res_qi[0]), bytes(res_qi[1])


@pytest.mark.parametrize("mode", list(MODES))
def test_jobs_return_the_bytes_of_the_synchronous_call(store, mode):
    """Every query with a candidate, in batches of 16, at depth 1, 3 and 6, with the candidates given and with the job
    searching them itself: the records equal b200reg_perform_loop_closure's byte for byte.  One more batch mixes in
    queries without a candidate (dummy invalid outputs)."""
    import b200reg
    cfg = _cfg(mode)
    cand, closest = _candidates(store, cfg)
    assert len(cand) >= 64
    batches = [cand[i:i + B] for i in range(0, len(cand), B)]
    batches.append(np.arange(3, NKF, 17, dtype=np.int32)[:B])
    assert (closest[batches[-1]] < 0).any() and (closest[batches[-1]] >= 0).any()
    sync = [store.perform_loop_closure(q, closest[q], cfg, raw=True) for q in batches]
    assert sum(r.valid for res, _ in sync for r in res) > 0, "the workload closes loops"
    want = [_bytes(o) for o in sync]
    for depth in (1, 3, 6):
        batch = b200reg.Batch(0, depth=depth)
        for explicit in (True, False):
            tickets = [batch.submit_perform_loop_closure(store, q, closest[q] if explicit else None, cfg) for q in batches]
            for k, t in enumerate(tickets):
                got = _bytes(batch.wait(t, want_quatro=True))
                assert got == want[k], (mode, depth, explicit, k)
        batch.close()


def test_job_sees_the_poses_at_submit(ctx, store, seq):
    """The iSAM2 write-back (fast_lio_sam_qn.cpp:180-188) arriving while attempts are in flight: every pose rewritten right
    after the submit leaves the job's answer at the old poses."""
    import b200reg
    from b200reg import synth
    cfg = _cfg()
    cand, closest = _candidates(store, cfg)
    q = cand[:B]
    want = _bytes(store.perform_loop_closure(q, closest[q], cfg, raw=True))
    batch = b200reg.Batch(0, depth=3)
    try:
        tickets = [batch.submit_perform_loop_closure(store, q, None, cfg), batch.submit_perform_loop_closure(store, q, closest[q], cfg)]
        for i in range(NKF):  # a drift correction that grows along the trajectory
            store.set_pose(i, synth.se3(yaw=2e-4 * i, t=(0.01 * i, -0.005 * i, 0.0)) @ seq["poses"][i])
        got = [_bytes(batch.wait(t, want_quatro=True)) for t in tickets]
        moved = _bytes(store.perform_loop_closure(q, closest[q], cfg, raw=True))
    finally:
        for i in range(NKF):
            store.set_pose(i, seq["poses"][i])
        batch.close()
    assert moved != want, "the rewritten poses change the synchronous answer"
    assert got == [want, want]


def test_job_ignores_keyframes_added_after_submit(ctx, seq):
    import b200reg
    cfg = _cfg("submap")
    n0 = 210
    kf = _store(ctx, seq, n0)
    batch = b200reg.Batch(0, depth=3)
    try:
        cand, closest = _candidates(kf, cfg)
        q = cand[-B:]
        want = _bytes(kf.perform_loop_closure(q, closest[q], cfg, raw=True))
        tickets = [batch.submit_perform_loop_closure(kf, q, None, cfg), batch.submit_perform_loop_closure(kf, q, closest[q], cfg)]
        for i in range(n0, NKF):
            kf.add(seq["clouds"][i], seq["poses"][i], seq["stamps"][i])
        assert [_bytes(batch.wait(t, want_quatro=True)) for t in tickets] == [want, want]
        assert len(kf) == NKF
    finally:
        batch.wait_all()
        batch.close()
        kf.destroy()


def test_interleaved_ingest_and_submits(ctx, seq):
    """One keyframe added and one job submitted per tick, no synchronisation in between: each job reads the keyframe its
    tick just uploaded, so its reads are ordered after the upload by the ingest event alone.  Every other tick arrives in
    the pcl::PointXYZI layout (32-byte records repacked by a kernel on the ingesting stream).  Each job equals the
    synchronous call at its tick (a query's answer depends on the keyframes up to it only)."""
    import b200reg
    cfg = _cfg()

    def records(i):
        c = seq["clouds"][i]
        if i % 2 == 0:
            return c
        r = np.zeros((len(c), 8), np.float32)
        r[:, :3], r[:, 3], r[:, 4] = c[:, :3], 1.0, c[:, 3]
        return r

    n0 = 180
    kf = _store(ctx, seq, n0)
    kf.reserve(30000 * (NKF - n0))
    batch = b200reg.Batch(0, depth=3)
    try:
        ticks = []
        for k in range(n0, n0 + 24):
            kf.add(records(k), seq["poses"][k], seq["stamps"][k])
            q = np.array([k - 2, k - 1, k], np.int32)
            ticks.append((q, batch.submit_perform_loop_closure(kf, q, None, cfg)))
        got = [_bytes(batch.wait(t, want_quatro=True)) for _, t in ticks]
        ctx.synchronize()
        tested = 0
        for (q, _), g in zip(ticks, got):
            closest = kf.fetch_closest(q, cfg.loop_detection_radius, cfg.loop_detection_timediff_threshold)
            tested += int((closest >= 0).sum())
            assert g == _bytes(kf.perform_loop_closure(q, closest, cfg, raw=True)), q
        assert tested >= 24, "the ticks run real attempts"
    finally:
        batch.wait_all()
        batch.close()
        kf.destroy()


def test_destroy_waits_for_jobs_and_bad_arguments_are_refused(ctx, seq):
    import b200reg
    from b200reg import native
    lib = native.lib()
    cfg = _cfg()
    kf = _store(ctx, seq, NKF)
    cand, closest = _candidates(kf, cfg)
    batch = b200reg.Batch(0, depth=1)
    try:
        for i in range(4):  # one context: the later jobs wait in its queue
            batch.submit_perform_loop_closure(kf, cand[B * i:B * (i + 1)], None, cfg)
        assert lib.b200reg_keyframes_destroy(ctx.h, kf.h) == native.ESTATE
        assert "in flight" in lib.b200reg_last_error().decode()
        with pytest.raises(b200reg.B200RegError):
            kf.destroy()
        assert kf.h and len(kf) == NKF  # nothing was freed
        batch.wait_all()

        def refused(q, cl=None, c=cfg, count=None):
            qa = np.ascontiguousarray(q, np.int32)
            ca = None if cl is None else np.ascontiguousarray(cl, np.int32)
            res, qi = (native.Result * max(len(qa), 1))(), (native.QuatroInfo * max(len(qa), 1))()
            return lib.b200reg_batch_submit_perform_loop_closure(batch.h, kf.h, len(qa) if count is None else count,
                                                                 qa.ctypes.data_as(C.c_void_p),
                                                                 None if ca is None else ca.ctypes.data_as(C.c_void_p), C.byref(c), res, qi)

        EINVAL = -1
        q0 = int(cand[0])
        assert refused([NKF]) == EINVAL and "query index" in lib.b200reg_last_error().decode()
        assert refused([-1]) == EINVAL
        assert refused([q0], [q0 + 1]) == EINVAL  # a candidate above its query
        assert refused([NKF], [3]) == EINVAL
        assert refused([-5], [3]) == EINVAL
        assert refused([q0], count=0) == EINVAL  # count 0 is refused, as the synchronous call refuses it
        bad = _cfg()
        bad.voxel_res = 0.0
        assert refused([q0], c=bad) == EINVAL and "voxel_res" in lib.b200reg_last_error().decode()
        bad = _cfg()
        bad.num_submap_keyframes = 1000
        assert refused([q0], c=bad) == EINVAL
        with pytest.raises(b200reg.B200RegError):
            batch.submit_perform_loop_closure(kf, [NKF])
        # a query outside the store without a candidate is no error for the synchronous call, nor for a job
        t = batch.submit_perform_loop_closure(kf, [NKF + 5, q0], [-1, closest[q0]], cfg)
        res, _ = batch.wait(t, want_quatro=True)
        assert not res[0].valid and bytes(res[1]) == bytes(kf.perform_loop_closure([q0], closest[[q0]], cfg, raw=True)[0][0])
        # a refusal further down (Quatro's parameters) comes back from wait with its message; the driver keeps working
        bad = _cfg()
        bad.quatro.estimate_scale = 1
        t_bad = batch.submit_perform_loop_closure(kf, [q0], None, bad)
        t_ok = batch.submit_perform_loop_closure(kf, [q0], None, cfg)
        with pytest.raises(b200reg.B200RegError) as e:
            batch.wait(t_bad)
        assert "estimate_scale" in str(e.value)
        assert bytes(batch.wait(t_ok)) == bytes(kf.perform_loop_closure([q0], closest[[q0]], cfg, raw=True)[0])
    finally:
        batch.wait_all()
        batch.close()
    kf.destroy()
    assert kf.h is None


def test_cxx_client(tmp_path, store, seq):
    """A C++ client ingests the sequence, submits every candidate query in batches of 16 (the job searches the candidates)
    and waits, through include/b200reg.h alone; its records equal the Python binding's."""
    from b200reg.build import build_native
    build_native()
    exe = str(tmp_path / "kf_batch_client")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-pthread", "-o", exe,
                           os.path.join(REPO, "tests", "cpp", "keyframe_batch_client.cpp"), "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    cfg = _cfg()
    cand, closest = _candidates(store, cfg)
    q = cand[:3 * B]
    nk = int(q.max()) + 1
    np.ascontiguousarray(np.stack(seq["clouds"][:nk]), np.float32).tofile(str(tmp_path / "clouds.bin"))
    np.ascontiguousarray(seq["poses"][:nk], np.float64).tofile(str(tmp_path / "poses.bin"))
    np.ascontiguousarray(seq["stamps"][:nk], np.float64).tofile(str(tmp_path / "stamps.bin"))
    q.astype(np.int32).tofile(str(tmp_path / "queries.bin"))
    txt = subprocess.check_output([exe, str(tmp_path), str(nk), str(len(seq["clouds"][0])), str(len(q)), "3"], timeout=600).decode()
    out = json.loads([ln for ln in txt.splitlines() if ln.startswith("{")][-1])
    assert out["status"] == 0 and out["keyframes"] == nk and out["destroy_in_flight"] == -4 and out["destroy_after"] == 0
    assert out["valid"] > 0
    res, qi = store.perform_loop_closure(q, closest[q], cfg, raw=True)
    assert bytes.fromhex(out["results"]) == bytes(res)
    assert bytes.fromhex(out["quatro"]) == bytes(qi)
