"""k_normals, k_spfh and k_fpfh against the fp64 restatement (tests/fpfh_ref.py) at raw-scan density and at their edges.

Normals: the NaN pattern is exact; every finite normal is unit to 4e-7 and, up to sign, within
    NRM_C1 * 2^-23 + NRM_C2 * eps64 * lam3 / (lam2 - lam1)
of the fp64 normal.  NRM_C1 = 2 covers the two float casts (each moves a unit vector by <= sqrt(3) 2^-24 rad).  NRM_C2 = 64
covers the device's one-pass fp64 moments about the query point and its eigen-solver: a backward-stable computation errs by
a small multiple of eps64 * |C| / gap.  The sign must equal the reference's wherever the flip test p . n is farther from 0
than its fp32 rounding plus what the allowed angle can move it.
FPFH (fed the GPU's own normals, exact integer SPFH counts): every bin within the rigorous per-bin bound of fpfh_ref.Fpfh.
"""
import numpy as np
import pytest

import fpfh_ref as R

pytestmark = pytest.mark.gpu
NRM_C1, NRM_C2 = 2.0, 64.0


def _patch(seed=7):
    """About 30k points in a 12 m box: two planes, a pole, a noisy blob and a near-collinear edge."""
    rng = np.random.default_rng(seed)
    floor = np.c_[rng.uniform(-6, 6, (12000, 2)), rng.normal(0, 0.01, 12000) - 1.5]
    wall = np.c_[rng.uniform(-6, 6, 8000), np.full(8000, 4.0) + rng.normal(0, 0.01, 8000), rng.uniform(-1.5, 4, 8000)]
    t = rng.uniform(0, 2 * np.pi, 3000)
    pole = np.c_[2 + 0.08 * np.cos(t), -1 + 0.08 * np.sin(t), rng.uniform(-1.5, 4, 3000)]
    blob = rng.normal(0, 0.6, (4000, 3)) + [-3, -3, 1]
    s = rng.uniform(-5, 5, 3000)
    edge = np.c_[s, np.full(3000, 2.0) + rng.normal(0, 2e-4, 3000), 2.5 + rng.normal(0, 2e-4, 3000)]
    return np.concatenate([floor, wall, pole, blob, edge]).astype(np.float32)


def _edge_scene():
    """Isolated clusters of 1..4 points (0..3 neighbours), exact duplicates, a 0.5 m lattice with points exactly on both
    radii (1.0 and 1.5: d2 = 1 and 2.25 are exact), and a copy of all of it 1 km from the origin."""
    pts = []
    for k in range(4):
        c = np.float32([30 + 10 * k, 30, 0])
        pts += [c + np.float32([0.2 * j, 0.05 * j * j, 0]) for j in range(k + 1)]
    g = np.arange(-5, 6) * 0.5
    X, Y = np.meshgrid(g, g)
    lat = np.c_[X.ravel(), Y.ravel(), np.full(X.size, -2.0)]
    lat3 = np.stack(np.meshgrid(g[3:8], g[3:8], g[3:6]), -1).reshape(-1, 3) + [10, 0, 0]
    dup = np.repeat(np.float32([[0.5, 0.5, -2], [-1, 1.5, -2], [10.5, 0.5, -0.5]]), 2, 0)
    one = np.concatenate([np.float32(pts), lat, lat3, dup]).astype(np.float32)
    return np.concatenate([one, one + np.float32([1000, 0, 0])]).astype(np.float32)


CLOUDS = {
    "raw100k": (0.9, 1.5),
    "vox0.3": (0.9, 1.5),
    "patch": (0.9, 1.5),
    "patch_r0.5": (0.5, 0.75),
    "patch_r1.2": (1.2, 2.5),
    "edges": (1.0, 1.5),
}


@pytest.fixture(scope="module")
def clouds(synth):
    src, dst, _ = synth.make_pair(2000, 100000, 100000, mode="quatro")
    _, vox, _ = synth.make_pair(2000, 100000, 100000, mode="quatro", voxel=0.3)
    patch = _patch()
    return {"raw100k": dst, "vox0.3": vox, "patch": patch, "patch_r0.5": patch, "patch_r1.2": patch, "edges": _edge_scene(),
            "raw_src": src}


def _gpu(ctx, pts, nr, fr):
    cl, = ctx.create_clouds([pts])
    ctx.fpfh([cl], nr, fr)
    gn, gf = ctx.get_fpfh(cl)
    cl.destroy()
    return gn, gf


@pytest.mark.parametrize("name", list(CLOUDS))
def test_normals_and_fpfh_against_fp64(ctx, clouds, name):
    nr, fr = CLOUDS[name]
    pts = clouds[name]
    xyz = np.ascontiguousarray(pts[:, :3], np.float32)
    gn, gf = _gpu(ctx, pts, nr, fr)
    cn = R.radius_csr(xyz, R.kernel_r2(nr))
    rn, lam, dot, derr = R.normals(xyz, cn)
    # ---- normals
    ok = ~np.isnan(rn[:, 0])
    assert np.array_equal(np.isnan(gn).any(1), ~ok), "NaN pattern differs from the exact neighbour counts"
    assert np.isfinite(gn[ok]).all()
    g64, r64 = gn[ok].astype(np.float64), rn[ok].astype(np.float64)
    assert np.abs(np.linalg.norm(g64, axis=1) - 1.0).max() <= 4e-7
    L = lam[ok]
    gap = L[:, 1] - L[:, 0]
    with np.errstate(divide="ignore"):
        bound = NRM_C1 * 2.0 ** -23 + NRM_C2 * R.EPS64 * np.where(gap > 0, L[:, 2] / gap, np.inf)
    c = (g64 * r64).sum(1)
    ang = np.arctan2(np.linalg.norm(np.cross(g64, r64), axis=1), np.abs(c))
    nratio = ang / bound
    bad = np.flatnonzero(nratio > 1)
    assert len(bad) == 0, ("normals beyond the eigen-gap bound", len(bad), ang[bad][:5], (gap / L[:, 2])[bad][:5])
    p = xyz[ok].astype(np.float64)
    sure = np.abs(dot[ok]) > derr[ok] + np.linalg.norm(p, axis=1) * np.minimum(bound, 2.0)
    assert np.all(c[sure] > 0), "normal flipped against the viewpoint rule where the sign is decided"
    # ---- FPFH from the GPU's own normals
    cf = R.radius_csr(xyz, R.kernel_r2(fr))
    counts, amb, cnt = R.spfh_counts(xyz, gn, cf)
    rng = np.random.default_rng(0)
    sel = np.arange(len(xyz)) if len(xyz) <= 40000 else np.sort(rng.choice(len(xyz), 20000, replace=False))
    F = R.Fpfh(cf.take(sel), counts, amb, cnt, gn)
    g = gf[sel].astype(np.float64)
    err = np.abs(g - F.v)
    fratio = err / np.where(F.bound > 0, F.bound, 1.0)
    worst = np.unravel_index(np.argmax(fratio), fratio.shape)
    assert np.all(err <= F.bound), ("FPFH beyond its bound", sel[worst[0]], worst[1], g[worst], F.v[worst], F.bound[worst])
    zero = (F.v == 0) & (F.slack == 0)
    assert np.all(g[zero] == 0), "a bin that is exactly 0 in the reference is not 0"
    refz = (F.v == 0).all(1)
    assert np.array_equal((g == 0).all(1), refz), "all-zero descriptors differ"
    sums = g[~refz].reshape(-1, 3, 11).sum(2)
    assert np.all(np.abs(sums - 100.0) <= F.bound[~refz].reshape(-1, 3, 11).sum(2) + 1e-9)
    nb = cnt[sel]
    print("\n%-10s n=%6d radii (%.2f, %.2f): normal-ball sizes %s, FPFH-ball sizes (min/1%%/50%%/99%%/max) %s, %d NaN normals,"
          " %d ambiguous f1 pairs" % (name, len(xyz), nr, fr, np.quantile(cn.counts, [0, 0.5, 1]).astype(int).tolist(),
                                      np.quantile(nb, [0, 0.01, 0.5, 0.99, 1]).astype(int).tolist(), (~ok).sum(), amb.sum()))
    print("           normals: max angle %.3g rad, max angle/bound %.3g; FPFH (%d points checked): max |err| %.3g, "
          "err/bound max %.3g median %.3g" % (ang.max(), nratio.max(), len(sel), err.max(), fratio.max(),
                                               np.median(fratio[F.v > 0])))


def test_fpfh_same_handle_new_radii_equals_fresh_handle(ctx, clouds):
    pts = clouds["patch"]
    cl, = ctx.create_clouds([pts])
    ctx.fpfh([cl], 0.9, 1.5)
    ctx.fpfh([cl], 1.2, 2.5)  # new key: recomputed in place (the SPFH table aliases the sorted descriptors)
    n1, f1 = ctx.get_fpfh(cl)
    ctx.fpfh([cl], 0.5, 0.75)
    ctx.fpfh([cl], 0.5, 0.75)  # same key: cached
    n2, f2 = ctx.get_fpfh(cl)
    cl.destroy()
    for (nr, fr), n, f in [((1.2, 2.5), n1, f1), ((0.5, 0.75), n2, f2)]:
        gn, gf = _gpu(ctx, pts, nr, fr)
        assert np.array_equal(n, gn, equal_nan=True) and np.array_equal(f.view(np.uint32), gf.view(np.uint32)), (nr, fr)


def test_fpfh_batch_equals_single_calls(ctx, clouds):
    raw = clouds["raw100k"]
    parts = [np.ascontiguousarray(p[:, :3]) for p in (clouds["vox0.3"], clouds["patch"], clouds["edges"], raw[np.abs(raw[:, 0] - 5) < 4])]
    cls = ctx.create_clouds(parts)
    ctx.fpfh(cls, 0.9, 1.5)
    batch = [ctx.get_fpfh(c) for c in cls]
    for c in cls:
        c.destroy()
    for pts, (bn, bf) in zip(parts, batch):
        for _ in range(2):  # one call per cloud, twice
            gn, gf = _gpu(ctx, pts, 0.9, 1.5)
            assert np.array_equal(bn, gn, equal_nan=True) and np.array_equal(bf.view(np.uint32), gf.view(np.uint32))


@pytest.mark.parametrize("mode", ["optimized", "advanced"])
def test_matching_at_raw_density_equals_oracle(ctx, oracle, native, clouds, mode):
    src, dst = clouds["raw_src"], clouds["raw100k"]
    prm = native.default_quatro_params()
    prm.use_optimized_matching = int(mode == "optimized")
    cs, cd = ctx.create_clouds([src, dst])
    info = ctx.quatro_align([cs], [cd], params=prm, want_corr=True)[0]
    _, fs = ctx.get_fpfh(cs)
    _, fd = ctx.get_fpfh(cd)
    cs.destroy(); cd.destroy()
    if mode == "optimized":
        corr, mutual = oracle.match(src, dst, fs, fd)
        assert info["n_mutual"] == len(mutual)
    else:
        corr = oracle.match_advanced(src, dst, fs, fd)
    assert info["n_corr"] == len(corr) > 0
    assert np.array_equal(info["corr"], corr), "correspondences (order included) differ from the oracle's on the same descriptors"
