"""The index build (k_bbox, k_morton_ghist, the three k_sort_pass, k_lbvh_topology, k_lbvh_aabb) and the shared radix sort
(launch_radix_sort) against the exact restatement of tests/index_ref.py, through b200reg_index_tap and b200reg_sort_tap:
keys, order, rank, topology, leaf collapse, boxes and depth bit for bit, at the sizes where the grids and the look-back
change shape, on degenerate and adversarial geometry, and in every input form.  Then the consumers of the tree on the
adversarial clouds: the k-NN (k = 1, 15, 40) and radius taps and the linearize pass's 1-NN against a brute force, and the
neighbours, covariances and alignment of a cloud with NaN points against the same cloud without them."""
import numpy as np
import pytest

import gicp_ref as R
import index_ref as X

pytestmark = pytest.mark.gpu


def uniform(n, seed=0):
    return np.random.default_rng(seed).uniform(-40, 40, (n, 3)).astype(np.float32)


def geometries(synth):
    rng = np.random.default_rng(3)
    g = {}
    raw = synth.make_pair(1000, 100000, 100000)[1][:, :3]
    g["raw100k"] = np.ascontiguousarray(raw)
    g["vox0.3"] = np.ascontiguousarray(synth.make_pair(1000, 100000, 100000, voxel=0.3)[1][:, :3])
    g["identical"] = np.tile(np.float32([[1.5, -2.0, 0.25]]), (5000, 1))
    two = np.tile(np.float32([[0, 0, 0]]), (3001, 1))
    two[rng.random(3001) < 0.5] = (1.0, 2.0, 3.0)
    g["two_values"] = two
    t = rng.uniform(0, 10, 4000).astype(np.float32)
    g["collinear"] = np.stack([t, 2 * t, -t], 1).astype(np.float32)
    g["coplanar"] = np.stack([rng.uniform(0, 10, 4000), rng.uniform(0, 3, 4000), np.full(4000, 7.0)], 1).astype(np.float32)
    a = np.arange(16, dtype=np.float32) * 0.5
    g["lattice"] = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)[rng.permutation(4096)]
    top = uniform(3000, 4)
    top[::7] = top.max(0)  # points exactly at the box maximum (q = 1023 on every axis, or 1024 clamped)
    top[1::7, 0] = top[:, 0].max()
    g["box_max"] = top
    sub = np.zeros((2000, 3), np.float32)
    sub[:, 0] = rng.integers(0, 4, 2000).astype(np.float32) * np.float32(1e-45)  # extent 3 denormals: 1023 / ext = +inf
    sub[:, 1] = np.float32(2e-44) * rng.integers(0, 2, 2000)
    g["subnormal"] = sub
    g["offset25km"] = (raw[:30000] + np.float32([25000.0, -25000.0, 10.0])).astype(np.float32)
    nan = uniform(5000, 5)
    nan[[0, 1, 17, 2048, 4999]] = np.nan
    nan[100:300, 1] = np.nan
    g["nan"] = nan
    inf = uniform(3000, 6)
    inf[5, 0], inf[6, 2], inf[7] = np.inf, -np.inf, np.nan
    g["inf"] = inf
    g["all_nan"] = np.full((20, 3), np.nan, np.float32)
    g["comb20"] = X.comb_cloud(20)
    return g


@pytest.fixture(scope="module")
def geo(synth):
    return geometries(synth)


def one(ctx, xyz, **kw):
    return ctx.index_tap([xyz], **kw)[0]


SIZES = (1, 2, X.LEAF, X.LEAF + 1, 2 * X.LEAF - 1, 2 * X.LEAF + 1, X.SORT_TILE - 1, X.SORT_TILE, X.SORT_TILE + 1,
         75775, 75776, 75777, 1 << 20, 1 << 22)


@pytest.mark.parametrize("n", SIZES)
def test_sizes(ctx, n):
    xyz = uniform(n, n)
    depth = X.check(xyz, one(ctx, xyz))
    assert depth <= X.depth_bound(n)


def test_geometries(ctx, geo):
    depths = {}
    for name, xyz in geo.items():
        depths[name] = X.check(xyz, one(ctx, xyz))
    n = len(geo["comb20"])
    assert depths["comb20"] == X.depth_bound(n) == 48, depths["comb20"]
    print("\ndepth / bound: " + ", ".join("%s %d/%d" % (k, d, X.depth_bound(len(geo[k]))) for k, d in depths.items()))


def test_comb_4m_reaches_its_bound(ctx):
    xyz = X.comb_cloud(22)
    depth = X.check(xyz, one(ctx, xyz))
    assert depth == X.depth_bound(len(xyz)) == 50 and X.DEPTH_BOUND <= X.MAX_STACK


def _reachable_bytes(t):
    ids, _ = X.reachable(t["tnodes"], t["root_ref"])
    return ids, t["tnodes"][ids].tobytes()


def _same(a, b):
    assert a["root_ref"] == b["root_ref"]
    for k in ("keys", "pts", "rank"):
        assert a[k].tobytes() == b[k].tobytes(), k
    ia, ba = _reachable_bytes(a)
    ib, bb = _reachable_bytes(b)
    assert np.array_equal(ia, ib) and ba == bb


def test_ragged_batch_equals_alone_and_builds_are_deterministic(ctx, geo):
    clouds = [uniform(n, n) for n in (1, 9, 2049, 75777, 300000)] + [geo["nan"], geo["comb20"], geo["identical"]]
    batch = ctx.index_tap(clouds)
    again = ctx.index_tap(clouds)
    for xyz, b, c in zip(clouds, batch, again):
        X.check(xyz, b)
        _same(b, c)
        _same(b, one(ctx, xyz))


def test_strides_and_device_input(ctx, geo):
    import torch
    xyz = geo["raw100k"]
    base = one(ctx, xyz)
    for width in (4, 8):
        rec = np.random.default_rng(width).normal(size=(len(xyz), width)).astype(np.float32)
        rec[:, :3] = xyz
        _same(base, one(ctx, rec))
        _same(base, ctx.index_tap([torch.from_numpy(rec).cuda()], device=True)[0])
    _same(base, ctx.index_tap([torch.from_numpy(xyz).cuda()], device=True)[0])


# ---------------------------------------------------------------------------------------------------------------------
# the shared radix sort
def _check_sort(ctx, keys, key_bits, vals=None):
    got = ctx.sort_tap(keys, vals, key_bits)
    for i, (k, (gk, gv)) in enumerate(zip(keys, got)):
        o = X.argsort_stable(k)
        v = np.arange(len(k), dtype=np.uint32) if vals is None else np.asarray(vals[i], np.uint32)
        assert np.array_equal(gk, np.asarray(k, np.uint32)[o]), (key_bits, len(k))
        assert np.array_equal(gv, v[o]), (key_bits, len(k))


def _distributions(n, bits, rng):
    top = (1 << bits) - 1
    d = {"zero": np.zeros(n, np.uint32), "max": np.full(n, top, np.uint32),
         "descending": (top - np.arange(n, dtype=np.uint64)).astype(np.uint32),
         "random": rng.integers(0, top + 1, n, dtype=np.uint64).astype(np.uint32),
         "runs": np.repeat(rng.integers(0, top + 1, 5, dtype=np.uint64), -(-n // 5))[:n].astype(np.uint32)}
    dbits = 10 if bits == 30 else 11
    for p in range(3):
        base = np.uint32(rng.integers(0, top + 1) & ~(((1 << dbits) - 1) << (dbits * p)) & top)
        d["digit%d" % p] = (base | ((rng.integers(0, 1 << dbits, n).astype(np.uint32) << np.uint32(dbits * p)) & np.uint32(top)))
    return d


@pytest.mark.parametrize("key_bits", [30, 32])
def test_sort_small_sizes_and_distributions(ctx, key_bits):
    rng = np.random.default_rng(key_bits)
    for n in (1, 2, 3, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4097, 65537):
        ds = _distributions(n, key_bits, rng)
        vals = [rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32) for _ in ds]
        _check_sort(ctx, list(ds.values()), key_bits, vals)


@pytest.mark.parametrize("key_bits", [30, 32])
def test_sort_large(ctx, key_bits):
    rng = np.random.default_rng(7 + key_bits)
    for n in (1 << 20, 1 << 24):
        ds = _distributions(n, key_bits, rng)
        for name in (("random", "runs", "descending", "digit2") if n == 1 << 20 else ("random", "runs")):
            _check_sort(ctx, [ds[name]], key_bits)


def test_sort_ragged_batch_equals_single_calls_and_rejects_bad_input(ctx):
    from b200reg.native import B200RegError
    rng = np.random.default_rng(9)
    keys = [rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32) for n in (1, 2049, 70000, 5, 300000)]
    batch = ctx.sort_tap(keys)
    for k, b in zip(keys, batch):
        a = ctx.sort_tap([k])[0]
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    with pytest.raises(B200RegError):
        ctx.sort_tap([keys[0]], key_bits=31)
    with pytest.raises(B200RegError):
        ctx.sort_tap([np.zeros(0, np.uint32)])


# ---------------------------------------------------------------------------------------------------------------------
# consumers of the tree on the adversarial clouds
def consumer_clouds(geo):
    small = {k: geo[k][:2500] for k in ("identical", "two_values", "collinear", "coplanar", "lattice", "box_max",
                                         "subnormal", "offset25km")}
    small["comb12"] = X.comb_cloud(12)
    return small


def brute_radius(xyz, r2):
    d2 = R.d2_f32(xyz[:, None, :], xyz[None, :, :])
    out = []
    for i in range(len(xyz)):
        j = np.flatnonzero(d2[i] < np.float32(r2))
        out.append((j[np.lexsort((j, d2[i, j]))], d2[i, j][np.lexsort((j, d2[i, j]))]))
    return out


def test_knn_and_radius_on_adversarial_clouds(ctx, geo):
    for name, xyz in consumer_clouds(geo).items():
        cl, = ctx.create_clouds([xyz])
        try:
            for k in (1, 15, 40):
                want_i, want_d = R.knn(xyz, k)
                gi, gd = ctx.knn(cl, xyz, k)
                assert np.array_equal(gi, want_i) and np.array_equal(gd, want_d), (name, k)
            ext = float(np.nanmax(xyz.max(0) - xyz.min(0)))
            r2 = max((0.05 * ext) ** 2, 1e-30)
            off, gi, gd = ctx.radius_search(cl, xyz, r2)
            for i, (wi, wd) in enumerate(brute_radius(xyz, r2)):
                assert np.array_equal(gi[off[i]:off[i + 1]], wi) and np.array_equal(gd[off[i]:off[i + 1]], wd), (name, i)
        finally:
            cl.destroy()


def test_linearize_one_nn_on_the_comb(ctx):
    """The comb target is 44 records deep: the LM search's walks run far past the 6 stack entries it keeps on chip."""
    tgt = X.comb_cloud(16)
    rng = np.random.default_rng(4)
    src = np.concatenate([rng.uniform(0, 1023, (3000, 3)), rng.uniform(-0.5, 3, (1000, 3))]).astype(np.float32)
    a, b = ctx.create_clouds([src, tgt])
    try:
        ctx.set_covariances(a, np.tile(np.eye(3), (len(src), 1, 1)))
        ctx.set_covariances(b, np.tile(np.eye(3), (len(tgt), 1, 1)))
        for mcd in (52.5, 2000.0):
            corr, sqd = R.correspondences(src, tgt, np.eye(4), mcd)
            g = ctx.linearize(a, b, np.eye(4), max_corr_dist=mcd)
            assert np.array_equal(g["corr"], corr) and np.array_equal(g["sqd"], sqd), mcd
    finally:
        a.destroy(); b.destroy()


@pytest.fixture(scope="module")
def nan_pair(synth):
    """A scan pair, and the same pair with 256 NaN points (index 0 among them; some NaN on one axis only) interleaved."""
    src, dst, _ = synth.make_pair(1001, 5000, 6000)
    out = []
    for seed, clean in ((1, src[:, :3]), (2, dst[:, :3])):
        clean = np.ascontiguousarray(clean, np.float32)
        rng = np.random.default_rng(seed)
        n = len(clean) + 256
        bad = np.sort(np.concatenate([[0], rng.choice(np.arange(1, n), 255, replace=False)]))
        keep = np.setdiff1d(np.arange(n), bad)
        dirty = np.zeros((n, 3), np.float32)
        dirty[keep] = clean
        dirty[bad] = np.nan
        dirty[bad[::5], 0] = 3.0  # a NaN on the other axes only
        out.append((clean, dirty, keep))
    return out


def test_nan_points_are_never_neighbours(ctx, nan_pair):
    """The finite points of a NaN-bearing cloud get the neighbours and covariances of the same cloud without the NaN
    points (indices mapped back): k = 15 (KnnHeap, Morton-window seeds among the NaN points at key 0) and k = 40."""
    clean, dirty, keep = nan_pair[0]
    cc, cd = ctx.create_clouds([clean, dirty])
    try:
        for k in (1, 15, 40):
            wi, wd = ctx.knn(cc, clean, k)
            gi, gd = ctx.knn(cd, clean, k)
            assert np.array_equal(keep[wi], gi) and np.array_equal(wd, gd), k
        for k in (15, 40):
            ctx.covariances([cc, cd], k, 0)
            got = ctx.get_covariances(cd)[keep]
            r, _ = R.Cov(clean, k).check(got, 0)
            assert (r <= 1).all(), (k, int((~(r <= 1)).sum()), np.flatnonzero(~(r <= 1))[:5])
            if k == 40:  # summed in list order: the same bits
                assert got.tobytes() == ctx.get_covariances(cc).tobytes()
    finally:
        cc.destroy(); cd.destroy()


def test_nan_points_leave_the_alignment_unchanged(ctx, nan_pair, synth):
    (cs, ds, _), (ct, dt, _) = nan_pair
    T = synth.se3(yaw=0.02, pitch=-0.004, t=(0.3, -0.2, 0.05))
    src_c = R.transform_query(T, cs)
    src_d = R.transform_query(T, ds)
    a = ctx.icp_alignment([src_c], [ct])[0]
    b = ctx.icp_alignment([src_d], [dt])[0]
    assert a["iterations"] == b["iterations"] and a["converged"] == b["converged"]
    assert np.abs(a["T"] - b["T"]).max() <= 1e-9, np.abs(a["T"] - b["T"]).max()
