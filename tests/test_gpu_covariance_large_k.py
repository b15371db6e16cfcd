"""NanoGICP covariances for k_correspondences > 32 (k_covariance_large, knn_large.cu): one warp per point.

CPU part: the oracle's covariances at k > 32 and at k >= n equal a numpy restatement of nano_gicp_impl.hpp:298-357 (fp32 d2
in the reference's order, (d2, index) order, sequential fp64 sums divided by k), so the oracle itself is pinned before the
GPU is compared with it; the facade client with setCorrespondenceRandomness(48) compiles in both type configurations.
GPU part: unregularised covariances bit-identical to the oracle (both list tiers, tiny clouds, ties, duplicates), all five
regularisation methods within the round-off of the k <= 32 tests, batches, the per-cloud cache, and registration end to end
through every entry point at k > 32.
"""
import json
import os
import subprocess

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(REPO, "fast-lio-sam-qn_b200", "host")
CSRC = os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc")
CLIENT_SRC = os.path.join(REPO, "tests", "cpp", "large_k_client.cpp")
MOCK_PCL = os.path.join(REPO, "tests", "cpp", "mock_pcl")
ROT_TOL = 1e-4    # rad
TRANS_TOL = 1e-3  # m


@pytest.fixture(autouse=True)
def own_kdtree(oracle):
    """Bit-exact checks use the oracle's own kd-tree: its ties resolve to the lower index, as on the device."""
    oracle.use_ref_nanoflann(False)
    yield


def _numpy_covariances(pts, k):
    """nano_gicp_impl.hpp:298-357 without regularisation, restated: the k nearest points of each point (itself included; all
    of them when k >= n) by fp32 d2 = ((dx*dx) + dy*dy) + dz*dz and lower index on ties; fp64 sums in that order, / k."""
    p = np.ascontiguousarray(pts[:, :3], np.float32)
    n = len(p)
    m = min(k, n)
    d = p[:, None, :] - p[None, :, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    assert d2.dtype == np.float32
    idx = np.arange(n)
    order = np.empty((n, m), np.int64)
    for i in range(n):
        order[i] = np.lexsort((idx, d2[i]))[:m]
    X = p.astype(np.float64)[order]  # (n, m, 3)
    mean = np.zeros((n, 3))
    for j in range(m):  # sequential, in list order
        mean = mean + X[:, j]
    mean = mean / k
    V = X - mean[:, None, :]
    cov = np.zeros((n, 3, 3))
    for j in range(m):
        cov = cov + V[:, j, :, None] * V[:, j, None, :]
    return cov / k


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def _lattice():
    rng = np.random.default_rng(8)
    g = np.stack(np.meshgrid(np.arange(9), np.arange(9), np.arange(9), indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    return (g[rng.permutation(len(g))] * np.float32(0.5)).astype(np.float32)


def _duplicates():
    rng = np.random.default_rng(9)
    base = rng.normal(0, 2, (300, 3)).astype(np.float32)
    return np.concatenate([base, base, base])[rng.permutation(900)]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
@pytest.mark.parametrize("k", [33, 64, 256])
def test_oracle_covariances_equal_numpy_restatement(oracle, synth, k):
    pts = synth.make_pair(1001, 1500, 1600)[1][:, :3]
    assert _bits_equal(oracle.covariances_ex(pts, k, 0), _numpy_covariances(pts, k))


@pytest.mark.parametrize("n,k", [(10, 33), (40, 64), (300, 300), (300, 1000)])
def test_oracle_covariances_k_at_least_n(oracle, n, k):
    """k >= n: every point is a neighbour, the divisor is still k."""
    pts = np.random.default_rng(n).normal(0, 3, (n, 3)).astype(np.float32)
    assert _bits_equal(oracle.covariances_ex(pts, k, 0), _numpy_covariances(pts, k))


@pytest.mark.parametrize("pts", ["lattice", "duplicates"])
def test_oracle_covariances_ties_equal_numpy_restatement(oracle, pts):
    p = _lattice() if pts == "lattice" else _duplicates()
    for k in (33, 100):
        assert _bits_equal(oracle.covariances_ex(p, k, 0), _numpy_covariances(p, k)), k


def _build_client(tmp, pcl_config=False):
    from b200reg.build import build_native
    build_native()
    exe = os.path.join(tmp, "large_k_client_pcl" if pcl_config else "large_k_client")
    extra = ["-I" + MOCK_PCL, "-DB200REG_EXPECT_PCL"] if pcl_config else []
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-I" + HOST] + extra + ["-o", exe, CLIENT_SRC,
                           "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    return exe


@pytest.mark.parametrize("pcl_config", [False, True])
def test_large_k_client_compiles(tmp_path, pcl_config):
    """setCorrespondenceRandomness(48) + align through the facade compile as C++14 in both type configurations."""
    assert os.path.exists(_build_client(str(tmp_path), pcl_config))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
@pytest.fixture(scope="module")
def voxel_scan(synth):
    """A 100k scan voxelised at 0.3 m (the sub-map resolution of loop_closure.cpp)."""
    raw = synth.make_pair(1004, 100000)[1]
    return np.ascontiguousarray(synth.voxelize(raw, 0.3)[:, :3])


def _gpu_cov(ctx, pts, k, method=0):
    cl, = ctx.create_clouds([pts])
    try:
        ctx.covariances([cl], k, method)
        return ctx.get_covariances(cl)
    finally:
        cl.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("k", [33, 48, 64, 100, 256, 257, 1000])
def test_none_bit_identical_to_oracle(ctx, oracle, pair20k, voxel_scan, k):
    """Unregularised covariances: all six values of every point bit-identical to the oracle, shared-memory lists
    (k <= 256) and slab lists (k > 256)."""
    for name, pts in (("20k", pair20k[1][:, :3]), ("voxel", voxel_scan)):
        g = _gpu_cov(ctx, pts, k)
        o = oracle.covariances_ex(pts, k, 0)
        assert _bits_equal(g, o), (name, k, int((g != o).any(axis=(1, 2)).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [33, 64, 300])
def test_all_methods_match_oracle(ctx, oracle, pair5k, k):
    """MIN_EIG, NORMALIZED_MIN_EIG, PLANE and FROBENIUS regularise like the k <= 32 path (closed form / Jacobi against the
    oracle's SVD: round-off), NONE bit for bit."""
    dst = pair5k[1]
    cl, = ctx.create_clouds([dst])
    try:
        for method in (0, 1, 2, 3, 4):
            ctx.covariances([cl], k, method)
            g = ctx.get_covariances(cl)
            o = oracle.covariances_ex(dst, k, method)
            scale = np.maximum(np.abs(o).reshape(len(o), -1).max(1), 1.0)
            err = np.abs(g - o).reshape(len(o), -1).max(1) / scale
            assert np.median(err) < 1e-11 and np.quantile(err, 0.995) < 1e-5, (method, k, np.median(err), np.quantile(err, 0.995))
            if method == 0:
                assert _bits_equal(g, o)
    finally:
        cl.destroy()


@pytest.mark.gpu
def test_tiny_clouds_ties_and_duplicates(ctx, oracle):
    """k >= n (every point a neighbour, divisor k), lattice shells that straddle rank k, exact duplicates."""
    rng = np.random.default_rng(4)
    for n in (10, 40):
        pts = rng.normal(0, 3, (n, 3)).astype(np.float32)
        for k in (33, 64):
            assert _bits_equal(_gpu_cov(ctx, pts, k), oracle.covariances_ex(pts, k, 0)), (n, k)
    for name, pts in (("lattice", _lattice()), ("duplicates", _duplicates())):
        for k in (33, 57, 100, 300):
            assert _bits_equal(_gpu_cov(ctx, pts, k), oracle.covariances_ex(pts, k, 0)), (name, k)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [48, 300])
def test_ragged_batch_equals_single_calls_and_repeats(ctx, synth, k):
    rng = np.random.default_rng(12)
    sizes = (7, 40, 3000, 20000, 257)
    pts = [np.ascontiguousarray(synth.make_pair(1200 + i, n)[1][:, :3]) if n >= 1000 else rng.normal(0, 2, (n, 3)).astype(np.float32)
           for i, n in enumerate(sizes)]
    batch = ctx.create_clouds(pts)
    try:
        ctx.covariances(batch, k, 0)
        got = [ctx.get_covariances(c) for c in batch]
        for p, g in zip(pts, got):
            assert _bits_equal(g, _gpu_cov(ctx, p, k))
        ctx.covariances(batch, k, 3)  # another method forces a recompute ...
        ctx.covariances(batch, k, 0)  # ... and back: the same bytes again
        for c, g in zip(batch, got):
            assert _bits_equal(ctx.get_covariances(c), g)
    finally:
        for c in batch:
            c.destroy()


@pytest.mark.gpu
def test_cache_follows_k(ctx, oracle, pair5k):
    """The per-cloud cache keys on k: switching between two k > 32 recomputes, and each answer is that k's."""
    dst = pair5k[1]
    cl, = ctx.create_clouds([dst])
    try:
        want = {k: oracle.covariances_ex(dst, k, 0) for k in (40, 64)}
        for k in (40, 64, 40, 32, 64):
            ctx.covariances([cl], k, 0)
            got = ctx.get_covariances(cl)
            if k == 32:  # the one-thread-per-point kernel: its own answer, not k = 40's
                assert not _bits_equal(got, want[40])
            else:
                assert _bits_equal(got, want[k]), k
    finally:
        cl.destroy()


def _params(k):
    import b200reg
    from oracle.oracle import GicpParams
    p, o = b200reg.default_params(), GicpParams.default()
    p.k_correspondences = k
    o.k_correspondences = k
    return p, o


def _same_record(a, b):
    return (np.array_equal(a["T"], b["T"]) and a["fitness"] == b["fitness"] and a["converged"] == b["converged"]
            and a["n_linearize"] == b["n_linearize"] and a["n_error"] == b["n_error"] and a["iterations"] == b["iterations"])


@pytest.mark.gpu
def test_gicp_align_k48_matches_oracle(ctx, oracle, synth, pair20k):
    src, dst, Texp = pair20k
    prm, oprm = _params(48)
    cs, ct = ctx.create_clouds([src, dst])
    try:
        g = ctx.gicp_align([cs], [ct], params=prm)[0]
        o = oracle.gicp_align(src, dst, params=oprm)
        rot, trans = synth.se3_error(g["T"], o["T"])
        assert rot < ROT_TOL and trans < TRANS_TOL, (rot, trans)
        assert g["converged"] == o["converged"] and g["iterations"] == o["iterations"]
        assert g["n_linearize"] == o["n_linearize"] and g["n_error"] == o["n_error"]
        rot, trans = synth.se3_error(g["T"], Texp)
        assert rot < 5e-3 and trans < 5e-2, ("ground truth", rot, trans)
        # the first linearize: correspondences and their distances bit-exact
        lin = ctx.linearize(cs, ct, np.eye(4))
        olin = oracle.linearize(src, dst, oracle.covariances(src, 48), oracle.covariances(dst, 48), np.eye(4))
        assert np.array_equal(lin["corr"], olin["corr"]) and np.array_equal(lin["sqd"], olin["sqd"])
    finally:
        cs.destroy(); ct.destroy()


@pytest.mark.gpu
def test_icp_alignment_k64_equals_gicp_align(ctx, pair5k):
    src, dst, _ = pair5k
    prm, _ = _params(64)
    r = ctx.icp_alignment([src], [dst], params=prm)[0]
    cs, ct = ctx.create_clouds([src, dst])
    try:
        g = ctx.gicp_align([cs], [ct], params=prm)[0]
    finally:
        cs.destroy(); ct.destroy()
    assert _same_record(r, g)
    r15 = ctx.icp_alignment([src], [dst])[0]
    assert not np.array_equal(r15["T"], r["T"])  # k reaches the covariances


@pytest.mark.gpu
def test_perform_loop_closure_k64_equals_gicp_align(ctx, synth):
    import b200reg
    seq = synth.make_sequence(7, 140, pts_per_keyframe=6000, spacing=3.0, speed=8.0)
    kf = ctx.keyframes()
    try:
        for c, T, t in zip(seq["clouds"], seq["poses"], seq["stamps"]):
            kf.add(c, T, t)
        queries = np.array([137, 139, 118], np.int32)
        closest = kf.fetch_closest(queries)
        assert (closest >= 0).all()
        cfg = b200reg.default_loop_config()
        cfg.enable_quatro = 0  # the fine stage on the assembled sub-maps, no guess
        cfg.gicp.k_correspondences = 64
        res, _ = kf.perform_loop_closure(queries, closest, cfg)
        sc, dc = kf.assemble(queries, closest, cfg, n_keyframes=queries + 1)
        try:
            prm, _ = _params(64)
            g = ctx.gicp_align(sc, dc, params=prm)
        finally:
            for c in sc + dc:
                c.destroy()
        for r, want in zip(res, g):
            assert _same_record(r, want)
    finally:
        kf.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("pcl_config", [False, True])
def test_large_k_client_equals_python_binding(tmp_path, ctx, synth, pcl_config):
    exe = _build_client(str(tmp_path), pcl_config)
    src, dst, _ = synth.make_pair(1001, 6000, 7000)
    sp, dp = str(tmp_path / "s.bin"), str(tmp_path / "d.bin")
    src.tofile(sp)
    dst.tofile(dp)
    out = json.loads(subprocess.check_output([exe, sp, dp]).decode())
    prm, _ = _params(48)
    r = ctx.icp_alignment([src], [dst], params=prm)[0]
    assert out["n_cov"] == [len(src), len(dst)]
    assert bool(out["converged"]) == r["converged"] and out["score"] == r["fitness"]
    assert np.array_equal(np.array(out["T"], np.float32).reshape(4, 4), r["Tf"])
