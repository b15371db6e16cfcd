"""The loop clouds of the batched loop-closure calls (b200reg_ctx_set_loop_clouds / b200reg_loop_clouds): the source, target,
coarse-aligned and final-aligned clouds loopTimerFunc publishes (fast_lio_sam_qn.cpp:245-248), bit for bit against the CPU
oracle, with empty rows exactly where the reference has no such cloud.  Capture changes no result, trace or launch count."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import voxel_cases

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc")
CLIENT_SRC = os.path.join(REPO, "tests", "cpp", "loop_clouds_client.cpp")
EINVAL, ESTATE = -1, -4
SOURCE, TARGET, COARSE, FINAL = 1, 2, 4, 8
KINDS = (SOURCE, TARGET, COARSE, FINAL)
QUERIES = [137, 139, 20, 118]  # 20 has no candidate; the others close loops at the start of the lap


def _build_client(tmp):
    from b200reg.build import build_native
    build_native()
    exe = os.path.join(tmp, "loop_clouds_client")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), "-o", exe,
                           CLIENT_SRC, "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    return exe


def test_loop_clouds_client_compiles(tmp_path):
    """The ABI alone is enough to feed the four publishes (no GPU needed to build)."""
    assert os.path.exists(_build_client(str(tmp_path)))


def _records(x4, stride):
    """(n, 4) x, y, z, intensity -> records of `stride` bytes: bare xyz, packed xyzi, or pcl::PointXYZI (x, y, z, 1, i, pad)."""
    if stride == 12:
        return np.ascontiguousarray(x4[:, :3])
    if stride == 16:
        return np.ascontiguousarray(x4)
    r = np.zeros((len(x4), 8), np.float32)
    r[:, :3] = x4[:, :3]
    r[:, 3] = 1.0
    r[:, 4] = x4[:, 3]
    return r


def _intensity(x4, stride):
    """b200reg_keyframes_add's rule: float 3 for 16-31-byte records, float 4 from 32 bytes, 0 for bare xyz."""
    return np.zeros(len(x4), np.float32) if stride == 12 else x4[:, 3]


def _fetch(ctx, kinds=KINDS):
    return {k: ctx.loop_clouds(k) for k in kinds}


def _captured(ctx, call, mask=15):
    """-> (what call() returned, {kind: rows}); capture is off again afterwards."""
    ctx.set_loop_clouds(mask)
    try:
        out = call()
        return out, _fetch(ctx, [k for k in KINDS if mask & k])
    finally:
        ctx.set_loop_clouds(0)


def _blobs():
    rng = np.random.default_rng(0)  # no structure at FPFH radii: Quatro finds no valid solution
    return rng.normal(0, 20, (300, 4)).astype(np.float32), rng.normal(0, 20, (280, 4)).astype(np.float32)


@pytest.fixture(scope="module")
def seq(synth):
    """The loop-capable sequence of the keyframe tests plus two structureless keyframes far away (indices 140, 141), whose
    pair fails the coarse stage.  -> (clouds, poses, stamps)"""
    s = synth.make_sequence(7, 140, pts_per_keyframe=6000, spacing=3.0, speed=8.0)
    far = synth.se3(t=(5000.0, 0.0, 0.0))
    return list(s["clouds"]) + list(_blobs()), list(s["poses"]) + [far, far], list(s["stamps"]) + [1000.0, 1001.0]


def _store(ctx, seq):
    kf = ctx.keyframes()
    for c, T, t in zip(*seq):
        kf.add(c, T, t)
    return kf


@pytest.fixture(scope="module")
def store(ctx, seq):
    kf = _store(ctx, seq)
    yield kf
    kf.destroy()


@pytest.fixture(scope="module")
def batch(store):
    """Fetched candidates of QUERIES plus the explicit structureless pair (141, 140) -> (queries, closest)."""
    closest = store.fetch_closest(np.array(QUERIES, np.int32))
    return np.array(QUERIES + [141], np.int32), np.append(closest, 140).astype(np.int32)


def _cfg(**kv):
    import b200reg
    cfg = b200reg.default_loop_config()
    for k, v in kv.items():
        setattr(cfg, k, v)
    return cfg


def _check_keyframe_rows(ctx, oracle, seq, q, closest, cfg, res, qi, cl):
    """Every row of a b200reg_perform_loop_closure capture against the oracle and the semantics of include/b200reg.h."""
    clouds, poses, _ = seq
    quatro = bool(cfg.enable_quatro)
    for k in KINDS:
        assert len(cl[k]) == len(q)
    for i in range(len(q)):
        S, T, Co, F = (cl[k][i] for k in KINDS)
        if closest[i] < 0:  # no candidate: the reference registers nothing
            assert len(S) == len(T) == len(Co) == len(F) == 0
            continue
        es, ed = oracle.set_src_and_dst_cloud(clouds, poses, int(q[i]), int(closest[i]), submap_range=cfg.num_submap_keyframes,
                                              voxel_res=cfg.voxel_res, enable_quatro=quatro,
                                              enable_submap_matching=bool(cfg.enable_submap_matching), n_keyframes=int(q[i]) + 1)
        assert S.shape == es.shape and S.tobytes() == es.tobytes()
        assert T.shape == ed.shape and T.tobytes() == ed.tobytes()
        if quatro and not qi[i]["valid"]:  # coarse_aligned_ cleared (loop_closure.cpp:142), no fine stage
            assert len(Co) == 0 and len(F) == 0
            continue
        if quatro:
            assert Co.tobytes() == oracle.transform_pcd(S, qi[i]["T"]).tobytes()
            fine_src = Co
            # the fine stage of this pair alone: the engine's solve of a pair does not depend on its batch
            Tf = ctx.icp_alignment([Co], [T], params=cfg.gicp)[0]["Tf"]
        else:
            assert len(Co) == 0
            fine_src, Tf = S, res[i]["Tf"]
        assert len(F) == len(fine_src)
        assert F[:, :3].tobytes() == oracle.transform_output(Tf, fine_src).tobytes()
        assert F[:, 3].tobytes() == fine_src[:, 3].tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
@pytest.mark.gpu
def test_keyframe_path_quatro(ctx, oracle, seq, store, batch):
    q, closest = batch
    cfg = _cfg()
    (res, qi), cl = _captured(ctx, lambda: store.perform_loop_closure(q, closest, cfg))
    has = closest >= 0
    valid = np.array([x["valid"] for x in qi])
    assert (~has).any() and (has & ~valid).any() and (has & valid).any()
    _check_keyframe_rows(ctx, oracle, seq, q, closest, cfg, res, qi, cl)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["gicp_only", "submap"])
def test_keyframe_path_variants(ctx, oracle, seq, store, batch, variant):
    q, closest = batch
    cfg = _cfg(enable_quatro=0) if variant == "gicp_only" else _cfg(enable_submap_matching=1)
    (res, qi), cl = _captured(ctx, lambda: store.perform_loop_closure(q, closest, cfg))
    if variant == "gicp_only":
        assert all(len(r) == 0 for r in cl[COARSE])
        assert all(len(cl[FINAL][i]) > 0 for i in range(len(q)) if closest[i] >= 0)  # converged or not
    _check_keyframe_rows(ctx, oracle, seq, q, closest, cfg, res, qi, cl)


@pytest.mark.gpu
def test_keyframe_path_voxel_overflow(ctx, oracle):
    """voxel_res 1 over a cloud whose voxel count passes int32: PCL returns the merged cloud unfiltered, intensities included."""
    cloud = voxel_cases.guard_above(16)
    seq2 = ([cloud, cloud], [np.eye(4), np.eye(4)], [0.0, 100.0])
    kf = _store(ctx, seq2)
    try:
        q, closest = np.array([1], np.int32), np.array([0], np.int32)
        cfg = _cfg(enable_quatro=0, voxel_res=1.0)
        (res, qi), cl = _captured(ctx, lambda: kf.perform_loop_closure(q, closest, cfg))
        assert cl[SOURCE][0].tobytes() == cloud.tobytes() and cl[TARGET][0].tobytes() == cloud.tobytes()
        _check_keyframe_rows(ctx, oracle, seq2, q, closest, cfg, res, qi, cl)
    finally:
        kf.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("stride", [12, 16, 32])
def test_raw_buffer_calls(ctx, oracle, synth, stride):
    # icpAlignment: FINAL only, the source through the solve's own transform
    pairs = [synth.make_pair(1100 + i, 4000 + 500 * i, 5000 - 300 * i) for i in range(3)]
    res, cl = _captured(ctx, lambda: ctx.icp_alignment([_records(p[0], stride) for p in pairs], [_records(p[1], stride) for p in pairs]))
    for k in (SOURCE, TARGET, COARSE):
        assert [len(r) for r in cl[k]] == [0, 0, 0]
    for i, (src, _, _) in enumerate(pairs):
        F = cl[FINAL][i]
        assert F[:, :3].tobytes() == oracle.transform_output(res[i]["Tf"], src).tobytes()
        assert F[:, 3].tobytes() == _intensity(src, stride).tobytes()
    # coarseToFineAlignment: COARSE and FINAL where the coarse stage is valid
    qpairs = [synth.make_pair(2100 + i, 5000 + 400 * i, 6000 - 300 * i, mode="quatro") for i in range(2)]
    blob_a, blob_b = _blobs()
    srcs, dsts = [qpairs[0][0], blob_a, qpairs[1][0]], [qpairs[0][1], blob_b, qpairs[1][1]]
    (res, qi), cl = _captured(ctx, lambda: ctx.loop_closure([_records(s, stride) for s in srcs], [_records(d, stride) for d in dsts]))
    assert [x["valid"] for x in qi] == [True, False, True]
    assert [len(r) for r in cl[SOURCE]] == [len(r) for r in cl[TARGET]] == [0, 0, 0]
    assert len(cl[COARSE][1]) == len(cl[FINAL][1]) == 0
    for i in (0, 2):
        Co, F = cl[COARSE][i], cl[FINAL][i]
        assert Co[:, :3].tobytes() == oracle.transform_pcd(srcs[i], qi[i]["T"])[:, :3].tobytes()
        assert Co[:, 3].tobytes() == F[:, 3].tobytes() == _intensity(srcs[i], stride).tobytes()
        Tf = ctx.icp_alignment([Co], [dsts[i]])[0]["Tf"]
        assert F[:, :3].tobytes() == oracle.transform_output(Tf, Co).tobytes()


@pytest.mark.gpu
def test_full_size_final_clouds(ctx, oracle, synth):
    """16 raw 100k x 100k pairs, FINAL only: every point against the oracle's fp32 transform."""
    pairs = [synth.make_pair(3000 + i, 100000) for i in range(16)]
    res, cl = _captured(ctx, lambda: ctx.icp_alignment([p[0] for p in pairs], [p[1] for p in pairs]), mask=FINAL)
    for i, (src, _, _) in enumerate(pairs):
        F = cl[FINAL][i]
        assert F.shape == (100000, 4)
        assert F[:, :3].tobytes() == oracle.transform_output(res[i]["Tf"], src).tobytes()
        assert F[:, 3].tobytes() == src[:, 3].tobytes()
    from b200reg import native
    with pytest.raises(native.B200RegError):  # not captured
        ctx.loop_clouds(SOURCE)


@pytest.mark.gpu
def test_capture_changes_nothing(seq, synth, native):
    """Results and LM traces are byte-identical with capture on and off; with it off the launch count is what it was before
    any capture; an uncaptured call discards the stored clouds."""
    import b200reg
    c = b200reg.Context(0)
    kf = _store(c, seq)
    try:
        closest = np.append(kf.fetch_closest(np.array(QUERIES, np.int32)), 140).astype(np.int32)
        q = np.array(QUERIES + [141], np.int32)
        qpairs = [synth.make_pair(2100 + i, 5000 + 400 * i, 6000 - 300 * i, mode="quatro") for i in range(2)]
        srcs, dsts = [p[0] for p in qpairs], [p[1] for p in qpairs]
        calls = {"perform": lambda: kf.perform_loop_closure(q, closest, raw=True),
                 "loop_closure": lambda: c.loop_closure_ptrs([a.ctypes.data for a in srcs], [len(a) for a in srcs],
                                                             [a.ctypes.data for a in dsts], [len(a) for a in dsts], 16, 0),
                 "icp": lambda: (c.icp_alignment(srcs, dsts, raw=True),)}
        c.set_lm_trace(True)
        for name, call in calls.items():
            def run():
                l0 = c.launch_count
                out = call()
                return b"".join(bytes(x) for x in out), c.launch_count - l0, c.lm_trace()
            off_before = run()
            c.set_loop_clouds(15)
            on = run()
            assert len(c.loop_clouds(FINAL)) == (len(q) if name == "perform" else 2)
            c.set_loop_clouds(0)
            off_after = run()
            assert on[0] == off_before[0] == off_after[0], name
            assert off_after[1] == off_before[1] and on[1] > off_before[1], name
            for tr in (on[2], off_after[2]):
                assert len(tr) == len(off_before[2]) and all(a.tobytes() == b.tobytes() for a, b in zip(tr, off_before[2])), name
            with pytest.raises(native.B200RegError):
                c.loop_clouds(FINAL)
    finally:
        kf.destroy()
        c.close()


@pytest.mark.gpu
def test_abi_contract(synth, native):
    import b200reg
    lib = native.lib()
    c = b200reg.Context(0)
    try:
        offsets = np.full(4, -7, np.int64)
        assert lib.b200reg_loop_clouds(c.h, SOURCE, offsets.ctypes.data_as(C.c_void_p), C.c_size_t(100), None) == ESTATE  # before any capture
        assert (offsets == -7).all()
        for bad in (0, 3, 16, -1):
            assert lib.b200reg_loop_clouds(c.h, bad, None, C.c_size_t(0), None) == EINVAL
        assert lib.b200reg_ctx_set_loop_clouds(c.h, 16) == EINVAL
        pairs = [synth.make_pair(1100 + i, 3000 + 500 * i, 3500) for i in range(2)]
        c.set_loop_clouds(FINAL)
        c.icp_alignment([p[0] for p in pairs], [p[1] for p in pairs])
        c.set_loop_clouds(0)
        assert lib.b200reg_loop_clouds(c.h, FINAL, None, C.c_size_t(0), None) == 2  # offsets only: the pair count
        for k in (SOURCE, TARGET, COARSE):  # kinds outside the mask
            assert lib.b200reg_loop_clouds(c.h, k, None, C.c_size_t(0), None) == ESTATE
        rows = c.loop_clouds(FINAL)
        total = sum(len(r) for r in rows)
        assert total == 3000 + 3500
        sentinel = np.frombuffer(bytes(range(256)) * (total * 16 // 256 + 1), np.uint8)[:total * 16].copy()
        buf = sentinel.copy()
        off = np.full(3, -7, np.int64)
        rc = lib.b200reg_loop_clouds(c.h, FINAL, off.ctypes.data_as(C.c_void_p), C.c_size_t(total - 1), buf.ctypes.data_as(C.c_void_p))
        assert rc == ESTATE and off.tolist() == [0, len(rows[0]), total] and np.array_equal(buf, sentinel)
        rc = lib.b200reg_loop_clouds(c.h, FINAL, off.ctypes.data_as(C.c_void_p), C.c_size_t(total), buf.ctypes.data_as(C.c_void_p))
        assert rc == 0 and buf.tobytes() == b"".join(r.tobytes() for r in rows)
        # a refused call and a call that fails in a stage both discard the clouds
        src, dst = pairs[0][0], pairs[0][1]
        kf = c.keyframes()
        c.set_loop_clouds(FINAL)
        try:
            with pytest.raises(native.B200RegError):  # an empty source cloud
                c.icp_alignment_ptrs([src.ctypes.data], [0], [dst.ctypes.data], [len(dst)], 16, False)
            assert lib.b200reg_loop_clouds(c.h, FINAL, None, C.c_size_t(0), None) == ESTATE
            kf.add(src, np.eye(4), 0.0)
            kf.add(dst, np.eye(4), 1.0)
            c.icp_alignment([src], [dst])
            assert lib.b200reg_loop_clouds(c.h, FINAL, None, C.c_size_t(0), None) == 1
            bad = _cfg()
            bad.quatro.estimate_scale = 1  # refused by the Quatro stage, after sub-map assembly
            with pytest.raises(native.B200RegError):
                kf.perform_loop_closure([1], [0], bad)
            assert lib.b200reg_loop_clouds(c.h, FINAL, None, C.c_size_t(0), None) == ESTATE
        finally:
            c.set_loop_clouds(0)
            kf.destroy()
    finally:
        c.close()


@pytest.mark.gpu
def test_client_matches_binding(tmp_path, ctx, seq, store):
    exe = _build_client(str(tmp_path))
    clouds, poses, stamps = seq
    path = str(tmp_path / "keyframes.bin")
    with open(path, "wb") as f:
        f.write(np.int32(len(clouds)).tobytes())
        for cl, T, t in zip(clouds, poses, stamps):
            cl = np.ascontiguousarray(cl, np.float32)
            f.write(np.int64(len(cl)).tobytes() + np.ascontiguousarray(T, np.float64).tobytes() + np.float64(t).tobytes() + cl.tobytes())
    prefix = str(tmp_path / "out")
    got = json.loads(subprocess.check_output([exe, path, prefix] + [str(x) for x in QUERIES]).decode())
    q = np.array(QUERIES, np.int32)
    closest = store.fetch_closest(q)
    (res, qi), cl = _captured(ctx, lambda: store.perform_loop_closure(q, closest))
    assert got["closest"] == closest.tolist()
    assert got["quatro_valid"] == [int(x["valid"]) for x in qi] and got["valid"] == [int(r["valid"]) for r in res]
    for k in KINDS:
        rows = cl[k]
        assert got["offsets"][str(k)] == np.cumsum([0] + [len(r) for r in rows]).tolist()
        with open("%s_%d.bin" % (prefix, k), "rb") as f:
            assert f.read() == b"".join(r.tobytes() for r in rows)
