"""b200reg_radius_search (KdTreeFLANN::radiusSearch with CSR output) on the GPU: against the reference kd-tree's answers, a
device brute force at full size, the edge cases of the bound and of the C ABI, determinism, and the C++ facade."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from test_radius_golden import _build, brute_force, golden_cases

pytestmark = pytest.mark.gpu

EINVAL, ESTATE = -1, -4


def rows(off, idx, d2, i):
    return idx[off[i]:off[i + 1]], d2[off[i]:off[i + 1]]


def check_sorted(gi, gd, oi, od):
    """Same set, same d2 bits per index, order ascending (d2, index): the reference's order wherever d2 has no ties."""
    want = np.lexsort((gi, gd))
    assert np.array_equal(oi, gi[want]) and np.array_equal(od.view(np.uint32), gd[want].view(np.uint32))


def check_unsorted(gi, gd, oi, od):
    want = np.argsort(gi, kind="stable")
    assert np.array_equal(oi, gi[want]) and np.array_equal(od.view(np.uint32), gd[want].view(np.uint32))


def test_golden_reference_kdtree_both_orders(ctx):
    clouds, cases = golden_cases()
    handles = dict(zip(clouds, ctx.create_clouds(list(clouds.values()))))
    for tag, qn, r2, q, off, idx, d2 in cases:
        for sorted_, check in ((True, check_sorted), (False, check_unsorted)):
            o, oi, od = ctx.radius_search(handles[tag], q, r2, sorted=sorted_)
            assert np.array_equal(o, off), (tag, qn, r2, sorted_)
            for i in range(len(q)):
                check(*rows(off, idx, d2, i), *rows(o, oi, od, i))
    for h in handles.values():
        h.destroy()


def torch_brute(cloud_t, q_t, r2):
    """Per query: boolean mask and d2 with the reference's fp32 expression, elementwise on the device (no fused ops)."""
    import torch
    diff = q_t[:, None, :] - cloud_t[None, :, :]
    d2 = (diff[..., 0] * diff[..., 0] + diff[..., 1] * diff[..., 1]) + diff[..., 2] * diff[..., 2]
    return d2 < torch.tensor(r2, dtype=torch.float32, device=d2.device), d2


@pytest.mark.parametrize("voxel", [None, 0.3])
def test_full_size_100k_self_queries(ctx, synth, voxel):
    """A 100k cloud, all of its points as queries, sq_radius 2.25: every count against the device brute force, a seeded
    sample of 2000 queries index- and bit-exact."""
    import torch
    if voxel is None:
        cloud = np.ascontiguousarray(synth.make_pair(31, 100000)[1][:, :3])
    else:  # ten 100k scans 15 m apart, voxelised together: a ~108k-point map
        poses = [synth.se3(t=(15.0 * k, 0.0, 1.73)) for k in range(10)]
        scans = np.concatenate([synth.to_map_frame(synth.scan(31, 100 + k, P, 100000), P) for k, P in enumerate(poses)])
        cloud = np.ascontiguousarray(synth.voxelize(scans, voxel)[:, :3])
    assert len(cloud) >= 100000
    cl, = ctx.create_clouds([cloud])
    off, idx, d2 = ctx.radius_search(cl, cloud, 2.25, sorted=True)
    off_u, idx_u, d2_u = ctx.radius_search(cl, cloud, 2.25, sorted=False)
    assert np.array_equal(off, off_u)
    ct = torch.from_numpy(cloud).cuda()
    counts = []
    for s in range(0, len(cloud), 1000):
        m, _ = torch_brute(ct, ct[s:s + 1000], 2.25)
        counts.append(m.sum(1).cpu().numpy())
    assert np.array_equal(np.diff(off), np.concatenate(counts))
    sample = np.random.default_rng(5).choice(len(cloud), 2000, replace=False)
    for s in range(0, len(sample), 250):
        rows_ = sample[s:s + 250]
        m, dd = torch_brute(ct, ct[torch.from_numpy(rows_).cuda()], 2.25)
        m, dd = m.cpu().numpy(), dd.cpu().numpy()
        for j, i in enumerate(rows_):
            bi = np.flatnonzero(m[j]).astype(np.int32)
            check_sorted(bi, dd[j][bi], *rows(off, idx, d2, i))
            check_unsorted(bi, dd[j][bi], *rows(off_u, idx_u, d2_u, i))
    cl.destroy()


def test_chunked_output_equals_brute_force(ctx, synth):
    """More neighbours than one chunk holds (2^23): the per-chunk output blocks land where the offsets say."""
    cloud = np.ascontiguousarray(synth.make_pair(32, 20000)[1][:, :3])
    q = cloud[::20]
    cl, = ctx.create_clouds([cloud])
    off, idx, d2 = ctx.radius_search(cl, q, 1e12, sorted=False)
    assert off[-1] == len(q) * len(cloud) > (1 << 23)
    assert np.array_equal(idx.reshape(len(q), -1), np.broadcast_to(np.arange(len(cloud), dtype=np.int32), (len(q), len(cloud))))
    offs, idxs, d2s = ctx.radius_search(cl, q, 1e12, sorted=True)
    for i in range(0, len(q), 97):
        bi, bd = brute_force(cloud, q[i], 1e12)
        check_unsorted(bi, bd, *rows(off, idx, d2, i))
        check_sorted(bi, bd, *rows(offs, idxs, d2s, i))
    cl.destroy()


def raw_call(ctx, cl, q, stride_floats, r2, sorted_, cap, with_outputs=True, fill=0x5A):
    from b200reg import native
    nq = len(q)
    rec = np.zeros((nq, stride_floats), np.float32)
    rec[:, :3] = q
    off = np.full(nq + 1, -7, np.int64)
    idx = np.full(max(cap, 1), fill, np.int32)
    d2 = np.full(max(cap, 1), fill, np.int32).view(np.float32)
    rc = native.lib().b200reg_radius_search(ctx.h, cl.h, rec.ctypes.data_as(C.c_void_p), C.c_size_t(nq), C.c_size_t(stride_floats * 4),
                                            C.c_double(r2), int(sorted_), off.ctypes.data_as(C.c_void_p), C.c_size_t(cap),
                                            idx.ctypes.data_as(C.c_void_p) if with_outputs else None,
                                            d2.ctypes.data_as(C.c_void_p) if with_outputs else None)
    return rc, off, idx, d2


def test_bound_is_strict_and_radius_is_squared(ctx):
    g = np.arange(4, dtype=np.float32) * np.float32(0.5)
    lattice = np.ascontiguousarray(np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3))
    cl, = ctx.create_clouds([lattice])
    off, idx, d2 = ctx.radius_search(cl, lattice[:1], 0.25)  # neighbours at exactly d2 = 0.25 are excluded
    assert list(idx) == [0] and d2[0] == 0
    off, idx, d2 = ctx.radius_search(cl, lattice[:1], 0.2500001)  # the squared radius, not the radius
    assert sorted(idx) == [0, 1, 4, 16] and np.all(d2[1:] == np.float32(0.25))
    off, idx, _ = ctx.radius_search(cl, lattice[:1], np.nextafter(np.float32(0.25), np.float32(1), dtype=np.float32).item())
    assert len(idx) == 4
    for r2 in (0.0, -1.0, float("nan")):  # nothing is closer than 0, or than NaN
        off, idx, _ = ctx.radius_search(cl, lattice, r2)
        assert np.all(off == 0) and len(idx) == 0
    for r2 in (1e30, 1e300):  # 1e300 converts to +inf in fp32: still every point
        off, idx, _ = ctx.radius_search(cl, lattice, r2, sorted=False)
        assert np.all(np.diff(off) == len(lattice)) and np.array_equal(idx.reshape(len(lattice), -1)[3], np.arange(len(lattice)))
    cl.destroy()


def test_duplicates_tiny_clouds_and_far_offsets(ctx, synth):
    rng = np.random.default_rng(3)
    base = rng.uniform(-2, 2, (300, 3)).astype(np.float32)
    dup = np.ascontiguousarray(np.concatenate([base, base, base[:50]]))
    far = np.ascontiguousarray(rng.uniform(-30, 30, (5000, 3)).astype(np.float32) + np.float32([25000.0, -25000.0, 3.0]))
    clouds = [dup, far] + [np.ascontiguousarray(rng.uniform(-1, 1, (n, 3)).astype(np.float32)) for n in (1, 2, 9)]
    handles = ctx.create_clouds(clouds)
    for cloud, h in zip(clouds, handles):
        q = np.ascontiguousarray(np.concatenate([cloud[:40], cloud[:40] + rng.normal(0, 0.3, (min(40, len(cloud)), 3)).astype(np.float32)]))
        for r2 in (0.04, 0.5, 9.0):
            off, idx, d2 = ctx.radius_search(h, q, r2, sorted=True)
            off_u, idx_u, d2_u = ctx.radius_search(h, q, r2, sorted=False)
            for i in range(len(q)):
                bi, bd = brute_force(cloud, q[i], r2)
                check_sorted(bi, bd, *rows(off, idx, d2, i))
                check_unsorted(bi, bd, *rows(off_u, idx_u, d2_u, i))
    # every copy of a duplicated point is returned
    off, idx, _ = ctx.radius_search(handles[0], base[:1], 1e-12, sorted=False)
    assert list(idx) == [0, 300, 600]
    for h in handles:
        h.destroy()


def test_abi_strides_count_only_capacity_and_errors(ctx, synth):
    cloud = np.ascontiguousarray(synth.make_pair(33, 8000)[1][:, :3])
    q = np.ascontiguousarray(cloud[::10] + np.float32(0.1))
    cl, = ctx.create_clouds([cloud])
    off, idx, d2 = ctx.radius_search(cl, q, 0.81)
    total = int(off[-1])
    for stride in (3, 4, 8):  # 12, 16 and 32 bytes
        rc, o, i, d = raw_call(ctx, cl, q, stride, 0.81, 1, total)
        assert rc == 0 and np.array_equal(o, off) and np.array_equal(i, idx) and np.array_equal(d.view(np.uint32), d2.view(np.uint32))
    rc, o, i, d = raw_call(ctx, cl, q, 4, 0.81, 1, 0, with_outputs=False)  # count only
    assert rc == 0 and np.array_equal(o, off)
    rc, o, i, d = raw_call(ctx, cl, q, 4, 0.81, 1, total - 1)  # too small: offsets filled, outputs untouched
    assert rc == ESTATE and np.array_equal(o, off)
    assert np.all(i == 0x5A) and np.all(d.view(np.int32) == 0x5A)
    from b200reg import native
    assert str(total) in native.lib().b200reg_last_error().decode()
    rc, o, _, _ = raw_call(ctx, cl, q[:0], 4, 0.81, 1, 10)  # nq == 0
    assert rc == EINVAL
    bad = native.lib().b200reg_radius_search(ctx.h, cl.h, q.ctypes.data_as(C.c_void_p), C.c_size_t(len(q)), C.c_size_t(10), C.c_double(1.0),
                                             1, o.ctypes.data_as(C.c_void_p), C.c_size_t(0), None, None)
    assert bad == EINVAL
    cl.destroy()


def test_deterministic_and_independent_of_query_order(ctx, synth):
    cloud = np.ascontiguousarray(synth.make_pair(34, 30000)[1][:, :3])
    q = np.ascontiguousarray(cloud[::3] + np.float32(0.05))
    cl, = ctx.create_clouds([cloud])
    for sorted_ in (True, False):
        a = ctx.radius_search(cl, q, 2.25, sorted=sorted_)
        b = ctx.radius_search(cl, q, 2.25, sorted=sorted_)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
        perm = np.random.default_rng(9).permutation(len(q))
        p = ctx.radius_search(cl, np.ascontiguousarray(q[perm]), 2.25, sorted=sorted_)
        for j in range(0, len(q), 7):
            pi, pd = rows(*p, j)
            ai, ad = rows(*a, perm[j])
            assert np.array_equal(pi, ai) and pd.tobytes() == ad.tobytes()
    cl.destroy()


@pytest.mark.parametrize("pcl_config", [False, True])
def test_kdtree_facade_equals_python_binding(tmp_path, ctx, synth, pcl_config):
    """NanoGICP::source_kdtree_ / target_kdtree_ (before and after swapSourceAndTarget), a standalone KdTreeFLANN over an
    index subset (sorted / unsorted), nearestKSearch (k > n included) through the C++ facade = the Python binding."""
    exe = _build(str(tmp_path), pcl_config)
    src, dst, _ = synth.make_pair(1001, 6000, 7000)
    rng = np.random.default_rng(11)
    q = np.concatenate([dst[:20], src[:20] + rng.normal(0, 0.4, (20, 4)).astype(np.float32)]).astype(np.float32)
    paths = [str(tmp_path / n) for n in ("s.bin", "d.bin", "q.bin")]
    for a, p in zip((src, dst, q), paths):
        np.ascontiguousarray(a, np.float32).tofile(p)
    r2 = 2.25
    out = json.loads(subprocess.check_output([exe] + paths + [repr(r2)]).decode())
    assert out["same_cloud"] == 1
    sub = np.ascontiguousarray(dst[::3])
    cs, cd, cb, ct = ctx.create_clouds([src, dst, sub, np.ascontiguousarray(dst[:4])])
    q3 = np.ascontiguousarray(q[:, :3])

    def same_radius(name, cl, sorted_):
        off, idx, d2 = ctx.radius_search(cl, q3, r2, sorted=sorted_)
        r = out[name]
        assert r["count"] == list(np.diff(off)), name
        assert r["idx"] == idx.tolist() and np.array_equal(np.array(r["d2"], np.float32), d2), name

    same_radius("source_radius", cs, False)
    same_radius("target_radius_sorted", cd, True)
    same_radius("swapped_source_radius_sorted", cd, True)  # the trees moved with the clouds, each kept its own settings
    same_radius("swapped_target_radius", cs, False)
    same_radius("subset_radius", cb, False)
    same_radius("subset_radius_sorted", cb, True)
    for name, cl, k, n in (("target_knn5", cd, 5, 5), ("tiny_knn6", ct, 6, 4)):
        idx, d2 = ctx.knn(cl, q3, k)
        r = out[name]
        assert r["count"] == [n] * len(q), name
        assert r["idx"] == idx.ravel().tolist() and np.array_equal(np.array(r["d2"], np.float32), d2.ravel()), name
    for c in (cs, cd, cb, ct):
        c.destroy()
