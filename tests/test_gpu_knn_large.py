"""b200reg_knn with k > 32 (one warp per query, knn_large.cu) on the GPU: against the reference kd-tree's answers, the CPU
brute force at 20k and 100k points, the k <= 32 path, the edges of the C ABI (padding, ties, far offsets, strides, NaN),
chunking, determinism, query order, and the C++ facade."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

from test_knn_large_golden import all_d2, brute_knn, build_knn_client, golden_cases

pytestmark = pytest.mark.gpu

EINVAL = -1
FLT_MAX = np.finfo(np.float32).max


def same(a, b):
    (ai, ad), (bi, bd) = a, b
    return ai.shape == bi.shape and np.array_equal(ai, bi) and ad.tobytes() == bd.tobytes()


def scan_clouds(synth, n):
    """A raw KITTI-shaped scan of n points and a 0.3 m-voxelised map of about the same size."""
    raw = np.ascontiguousarray(synth.make_pair(41, n)[1][:, :3])
    scans = n // 10000 + 1
    poses = [synth.se3(t=(15.0 * k, 0.0, 1.73)) for k in range(scans)]
    merged = np.concatenate([synth.to_map_frame(synth.scan(41, 200 + k, P, 100000), P) for k, P in enumerate(poses)])
    vox = np.ascontiguousarray(synth.voxelize(merged, 0.3)[:, :3])
    return {"raw": raw, "vox": np.ascontiguousarray(vox[:max(n, 1)])}


def queries(cloud, rng, m):
    rows = rng.choice(len(cloud), m, replace=False)
    return {"self": np.ascontiguousarray(cloud[rows]),
            "shift": np.ascontiguousarray(cloud[rows] + rng.normal(0, 0.5, (m, 3)).astype(np.float32)),
            "far": np.ascontiguousarray(cloud[rows[:m // 4]] + np.float32(400.0))}


def test_golden_reference_kdtree(ctx):
    """The engine equals the brute force exactly and the reference kd-tree wherever its first-visited tie rule allows."""
    clouds, cases = golden_cases()
    handles = dict(zip(clouds, ctx.create_clouds(list(clouds.values()))))
    for tag, qn, k, q, ridx, rd2 in cases:
        idx, d2 = ctx.knn(handles[tag], q, k)
        assert d2.tobytes() == rd2.tobytes(), (tag, qn, k)
        for i in range(len(q)):
            assert same((idx[i], d2[i]), brute_knn(clouds[tag], q[i], k)), (tag, qn, k, i)
            vals, counts = np.unique(all_d2(clouds[tag], q[i]), return_counts=True)
            untied = counts[np.searchsorted(vals, rd2[i])] == 1
            assert np.array_equal(idx[i][untied], ridx[i][untied]), (tag, qn, k, i)
    for h in handles.values():
        h.destroy()


def test_20k_clouds_equal_oracle_brute_force(ctx, synth, oracle):
    rng = np.random.default_rng(21)
    for tag, cloud in scan_clouds(synth, 20000).items():
        cl, = ctx.create_clouds([cloud])
        for qn, q in queries(cloud, rng, 160).items():
            for k in (33, 63, 64, 65, 127, 128, 129, 256, 257, 1000):  # 257, 1000: above the shared-memory tier (256)
                got = ctx.knn(cl, q, k)
                assert same(got, oracle.knn(cloud, q, k, brute=True)), (tag, qn, k)
        cl.destroy()


@pytest.mark.parametrize("voxel", [False, True])
def test_full_size_100k(ctx, synth, oracle, voxel):
    cloud = scan_clouds(synth, 100000)["vox" if voxel else "raw"]
    assert len(cloud) >= 100000 or voxel
    rng = np.random.default_rng(22)
    qs = queries(cloud, rng, 2000)
    q = np.ascontiguousarray(np.concatenate([qs["self"], qs["shift"]]))
    cl, = ctx.create_clouds([cloud])
    for k in (64, 512):
        assert same(ctx.knn(cl, q, k), oracle.knn(cloud, q, k, brute=True)), k
    cl.destroy()


def test_prefix_equals_k32_path(ctx, synth):
    """The first 32 columns at k = 64 are the k <= 32 kernels' answer at k = 32, bit for bit."""
    rng = np.random.default_rng(23)
    for cloud in scan_clouds(synth, 20000).values():
        cl, = ctx.create_clouds([cloud])
        q = np.ascontiguousarray(np.concatenate(list(queries(cloud, rng, 1000).values())))
        i32, d32 = ctx.knn(cl, q, 32)
        i64, d64 = ctx.knn(cl, q, 64)
        assert np.array_equal(i64[:, :32], i32) and d64[:, :32].tobytes() == d32.tobytes()
        cl.destroy()


def test_tiny_clouds_padding_and_return_values(ctx, oracle):
    rng = np.random.default_rng(24)
    for n in (1, 2, 7, 8, 9, 33, 65):
        cloud = np.ascontiguousarray(rng.uniform(-1, 1, (n, 3)).astype(np.float32))
        q = np.ascontiguousarray(np.concatenate([cloud, rng.uniform(-2, 2, (20, 3)).astype(np.float32)]))
        cl, = ctx.create_clouds([cloud])
        for k in (n - 1, n, n + 1, n + 1000):
            if k < 1:
                continue
            idx, d2 = ctx.knn(cl, q, k)
            assert same((idx, d2), oracle.knn(cloud, q, k, brute=True)), (n, k)
            assert np.all(np.sum(idx >= 0, 1) == min(k, n)), (n, k)  # what nearestKSearch returns
            assert np.all(idx[:, n:] == -1) and np.all(d2[:, n:] == FLT_MAX), (n, k)
        cl.destroy()


def test_duplicates_lattice_and_far_offsets(ctx, oracle):
    """Equal distances resolve to the lower index, inside the list and across rank k; 25 km from the origin the fp32
    distances are coarse and ties are everywhere."""
    rng = np.random.default_rng(25)
    base = rng.uniform(-2, 2, (400, 3)).astype(np.float32)
    dup = np.ascontiguousarray(np.concatenate([base, base, base[:100], base]))
    g = np.arange(10, dtype=np.float32) * np.float32(0.5)
    lattice = np.ascontiguousarray(np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3))
    far = np.ascontiguousarray(rng.uniform(-30, 30, (6000, 3)).astype(np.float32) + np.float32([25000.0, -25000.0, 3.0]))
    for cloud in (dup, lattice, far):
        cl, = ctx.create_clouds([cloud])
        q = np.ascontiguousarray(np.concatenate([cloud[::13], cloud[::29] + np.float32(0.25)]))
        for k in (33, 64, 100, 300):
            assert same(ctx.knn(cl, q, k), oracle.knn(cloud, q, k, brute=True)), (len(cloud), k)
        cl.destroy()
    cl, = ctx.create_clouds([dup])
    idx, d2 = ctx.knn(cl, base[:1], 40)
    assert list(idx[0, :4]) == [0, 400, 800, 900] and np.all(d2[0, :4] == 0)  # every copy, lowest index first
    cl.destroy()


def raw_knn(ctx, cl, q, stride_floats, k):
    from b200reg import native
    rec = np.zeros((len(q), stride_floats), np.float32)
    rec[:, :3] = q
    idx = np.full((len(q), k), 0x5A, np.int32)
    d2 = np.full((len(q), k), 0x5A, np.int32).view(np.float32)
    rc = native.lib().b200reg_knn(ctx.h, cl.h, rec.ctypes.data_as(C.c_void_p), C.c_size_t(len(q)), C.c_size_t(stride_floats * 4),
                                  int(k), idx.ctypes.data_as(C.c_void_p), d2.ctypes.data_as(C.c_void_p))
    return rc, idx, d2


def test_abi_strides_nan_and_errors(ctx, synth):
    from b200reg import native
    cloud = np.ascontiguousarray(synth.make_pair(42, 8000)[1][:, :3])
    q = np.ascontiguousarray(cloud[::10] + np.float32(0.1))
    cl, = ctx.create_clouds([cloud])
    for k in (40, 300):
        want = ctx.knn(cl, q, k)
        for stride in (3, 4, 8):  # 12, 16 and 32 bytes
            rc, i, d = raw_knn(ctx, cl, q, stride, k)
            assert rc == 0 and same((i, d), want), (k, stride)
    # a query with a NaN coordinate has no neighbours: its row is all padding, on every path; the other rows are untouched
    qn = q[:6].copy()
    qn[1, 0] = np.nan
    qn[3] = np.nan
    qn[4, 2] = np.nan
    for k in (8, 40, 300, len(cloud), len(cloud) + 5):
        idx, d2 = ctx.knn(cl, qn, k)
        for r in (1, 3, 4):
            assert np.all(idx[r] == -1) and np.all(d2[r] == FLT_MAX), (k, r)
        for r in (0, 2, 5):
            assert same((idx[r], d2[r]), brute_knn(cloud, qn[r], k)), (k, r)
    for k in (0, -1):
        assert native.lib().b200reg_knn(ctx.h, cl.h, q.ctypes.data_as(C.c_void_p), C.c_size_t(len(q)), C.c_size_t(12), int(k),
                                        q.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p)) == EINVAL
    out = np.empty((len(q), 33), np.int32)
    assert native.lib().b200reg_knn(ctx.h, cl.h, q.ctypes.data_as(C.c_void_p), C.c_size_t(len(q)), C.c_size_t(10), 33,
                                    out.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) == EINVAL
    assert native.lib().b200reg_knn_bruteforce(ctx.h, cl.h, q.ctypes.data_as(C.c_void_p), C.c_size_t(len(q)), C.c_size_t(12), 33,
                                               out.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) == EINVAL
    cl.destroy()


def test_chunks_determinism_and_query_order(ctx, synth):
    """Calls spanning several chunks (2^23 entries each) equal the same queries one by one; repeated calls return identical
    bytes; permuting the queries permutes the rows."""
    cloud = np.ascontiguousarray(synth.make_pair(43, 20000)[1][:, :3])
    rng = np.random.default_rng(26)
    cl, = ctx.create_clouds([cloud])
    for k, m in ((64, 300000), (1000, 20000)):  # shared-memory and device-scratch lists, three chunks each
        assert m * k > 2 * (1 << 23)
        q = np.ascontiguousarray(cloud[rng.integers(0, len(cloud), m)] + rng.normal(0, 0.3, (m, 3)).astype(np.float32))
        a = ctx.knn(cl, q, k)
        for i in range(0, m, m // 40):
            assert same(tuple(x[i:i + 1] for x in a), ctx.knn(cl, q[i:i + 1], k)), (k, i)
        assert same(a, ctx.knn(cl, q, k))
        perm = rng.permutation(m)
        p = ctx.knn(cl, np.ascontiguousarray(q[perm]), k)
        assert same(p, (a[0][perm], a[1][perm]))
        del a, p
    cl.destroy()


@pytest.mark.parametrize("pcl_config", [False, True])
def test_kdtree_facade_nearest_k_search_100(tmp_path, ctx, synth, pcl_config):
    """nearestKSearch(p, 100, ...) through NanoGICP::target_kdtree_ and a standalone tree = the Python binding; it returns
    min(k, n)."""
    exe = build_knn_client(str(tmp_path), pcl_config)
    dst = synth.make_pair(1002, 6000, 7000)[1]
    rng = np.random.default_rng(27)
    q = np.concatenate([dst[:20], dst[20:40] + rng.normal(0, 0.4, (20, 4)).astype(np.float32)]).astype(np.float32)
    paths = [str(tmp_path / n) for n in ("d.bin", "q.bin")]
    for a, p in zip((dst, q), paths):
        np.ascontiguousarray(a, np.float32).tofile(p)
    out = json.loads(subprocess.check_output([exe] + paths + ["100"]).decode())
    cd, = ctx.create_clouds([np.ascontiguousarray(dst[:, :3])])
    idx, d2 = ctx.knn(cd, np.ascontiguousarray(q[:, :3]), 100)
    for name in ("target_knn", "standalone_knn"):
        r = out[name]
        assert r["count"] == [100] * len(q), name
        assert r["idx"] == idx.ravel().tolist() and np.array_equal(np.array(r["d2"], np.float32), d2.ravel()), name
    cd.destroy()
