"""k_covariance (k <= 32), k_covariance_large (k > 32) and the linearize pass against the fp64 restatement
(tests/gicp_ref.py): every point within its bound, at the edge scenes and on a raw and a voxelised 100k scan.

Neighbour sets: the covariance kernel keeps its neighbours in KnnHeap (knn.cuh), with a cold tie path in offer, a pop for
k < K and a Morton seeding window the walk skips; none of that is reached by ctx.knn.  A wrong tied neighbour moves the
unregularised covariance far outside the NONE bound (test_gicp_reference.py shows it for the higher-index rule), so NONE
within its bound at every point checks the set without a tap, for k across the four capacities (8, 15, 20, 32), their
boundaries and the pop path.
NORMALIZED_MIN_EIG is NaN exactly where the raw covariance is zero, as in the reference.
Linearize: crafted covariances through set_covariances isolate the pass; correspondences and their fp32 d2 equal the
restatement's exactly (ties on a lattice, a gate exactly at a representable d2), H, b and err are within the per-entry bound.
"""
import numpy as np
import pytest

import gicp_ref as R

pytestmark = pytest.mark.gpu
KS_SETS = (1, 2, 7, 8, 9, 14, 15, 16, 19, 20, 21, 31, 32)
KS_REG = (1, 5, 15, 20, 32, 33, 64)
METHODS = (0, 1, 2, 3, 4)
NAMES = ("NONE", "MIN_EIG", "NORMALIZED_MIN_EIG", "PLANE", "FROBENIUS")


@pytest.fixture(scope="module")
def scenes():
    return R.scenes()


@pytest.fixture(scope="module")
def scans(synth):
    """The bench's first pair's target (seed 1000, 100k points) raw and voxelised at 0.3 m."""
    raw = synth.make_pair(1000, 100000, 100000)[1]
    vox = synth.make_pair(1000, 100000, 100000, voxel=0.3)[1]
    return {"raw100k": np.ascontiguousarray(raw[:, :3]), "vox0.3": np.ascontiguousarray(vox[:, :3])}


def _gpu_cov(ctx, pts, k, methods):
    cl, = ctx.create_clouds([pts])
    try:
        out = {}
        for m in methods:
            ctx.covariances([cl], k, m)
            out[m] = ctx.get_covariances(cl)
        return out
    finally:
        cl.destroy()


def _within(ref, got, method, tag):
    r, kind = ref.check(got, method)
    bad = np.flatnonzero(~(r <= 1))
    assert len(bad) == 0, (tag, NAMES[method], len(bad), bad[:5], r[bad[:5]], float(np.nanmax(r)))
    return r, kind


@pytest.mark.parametrize("k", KS_SETS)
def test_neighbour_sets_none_within_bound(ctx, scenes, k):
    _, d2 = R.knn(scenes["lattice"], k + 1)
    assert k == 1 or R.straddles(d2, k).any(), "the lattice has no tie across rank %d" % k
    for name, pts in list(scenes.items()) + [("n=%d" % len(p), p) for p in R.tiny(k)]:
        _within(R.Cov(pts, k), _gpu_cov(ctx, pts, k, (0,))[0], 0, (name, k))


@pytest.mark.parametrize("k", KS_REG)
def test_regularisation_edge_scenes_within_bound(ctx, scenes, k):
    for name, pts in list(scenes.items()) + [("n=%d" % len(p), p) for p in R.tiny(min(k, 33))]:
        ref = R.Cov(pts, k)
        got = _gpu_cov(ctx, pts, k, METHODS)
        for m in METHODS:
            _within(ref, got[m], m, (name, k))
        # the reference's NaN (k = 1; runs of copies longer than k), and nowhere else
        assert np.array_equal(np.isnan(got[2]).any((1, 2)), ref.zero), (name, k)
        assert all(np.isfinite(got[m]).all() for m in (0, 1, 3, 4)), (name, k)


@pytest.mark.parametrize("k", [15, 20, 33, 64])
@pytest.mark.parametrize("cloud", ["raw100k", "vox0.3"])
def test_regularisation_scan_within_bound(ctx, scans, cloud, k):
    pts = scans[cloud]
    ref = R.Cov(pts, k)
    got = _gpu_cov(ctx, pts, k, METHODS)
    line = []
    for m in METHODS:
        r, kind = _within(ref, got[m], m, (cloud, k))
        line.append("%s %.3g" % (NAMES[m], r.max()))
        if m == 3:
            line.append("PLANE checks vector/subspace/eigenvalues-only %s" % np.bincount(kind, minlength=3).tolist())
    print("\n%s k=%d worst fraction of the bound: %s" % (cloud, k, "; ".join(line)))


def test_mixed_batch_equals_single_calls(ctx, scenes, scans):
    """One call over the edge clouds, the tiny ones (n = 1..21) and the 100k scan equals one call per cloud, bit for bit."""
    clouds = list(scenes.values()) + R.tiny(20) + [scans["raw100k"]]
    batch = ctx.create_clouds(clouds)
    try:
        for k, m in ((20, 3), (15, 0), (9, 2), (40, 1)):
            ctx.covariances(batch, k, m)
            got = [ctx.get_covariances(c) for c in batch]
            for p, g in zip(clouds, got):
                want = _gpu_cov(ctx, p, k, (m,))[m]
                assert np.array_equal(g.view(np.uint64), want.view(np.uint64)), (k, m, len(p))
    finally:
        for c in batch:
            c.destroy()


def _lin(ctx, src, tgt, cs, ct, T, mcd, T_trial=None):
    a, b = ctx.create_clouds([src, tgt])
    try:
        ctx.set_covariances(a, cs)
        ctx.set_covariances(b, ct)
        g = ctx.linearize(a, b, T, max_corr_dist=mcd)
        e = None if T_trial is None else ctx.compute_error(a, b, T, T_trial, max_corr_dist=mcd)
        return g, e
    finally:
        a.destroy(); b.destroy()


def _lin_within(g, ref):
    rh = np.abs(g["H"] - ref.H) / ref.Hb
    rb = np.abs(g["b"] - ref.b) / ref.bb
    re = abs(g["err"] - ref.err) / ref.errb
    assert rh.max() <= 1 and rb.max() <= 1 and re <= 1, (rh.max(), rb.max(), re)


@pytest.mark.parametrize("offset", [(0.0, 0.0, 0.0), (1000.0, 0.0, 0.0)])
def test_linearize_lattice_gate_ties_and_conditioning(ctx, offset):
    src, tgt, want = R.lattice_pair(offset)
    Q = np.linalg.qr(np.random.default_rng(3).normal(size=(3, 3)))[0]
    cs = R.crafted_covariances(len(src), 1e8, 1, Q)
    ct = R.crafted_covariances(len(tgt), 1e8, 2, Q)
    T = np.eye(4)
    T_trial = np.array(T)
    T_trial[:3, 3] = [0.01, -0.02, 0.005]
    for mcd in (0.5, 1.0, 52.5):
        corr, sqd = R.correspondences(src, tgt, T, mcd)
        g, e = _lin(ctx, src, tgt, cs, ct, T, mcd, T_trial)
        assert np.array_equal(g["sqd"], sqd) and np.array_equal(g["sqd"].astype(np.float64), want)
        assert np.array_equal(g["corr"], corr), ("correspondences differ from the (d2, lower index) rule", mcd)
        if mcd == 0.5:  # exactly at the gate: rejected, and not in H
            assert (g["corr"][want == 0.25] == -1).all() and (g["corr"][want < 0.25] >= 0).all()
        ref = R.Linearize(src, tgt, cs, ct, T, corr)
        assert ref.kappa.max() > 1e7
        _lin_within(g, ref)
        et = R.Linearize(src, tgt, cs, ct, T, corr, T_trial=T_trial)
        assert abs(e - et.err) <= et.errb, (e, et.err, et.errb)


def test_linearize_scan_pair(ctx, synth):
    """A scan pair at a non-identity pose with the engine's own PLANE covariances and with crafted ill-conditioned ones."""
    src, dst, _ = synth.make_pair(1001, 5000, 6000)
    src, dst = src[:, :3].copy(), dst[:, :3].copy()
    T = synth.se3(yaw=0.02, pitch=-0.004, t=(0.3, -0.2, 0.05))
    cs_p = _gpu_cov(ctx, src, 15, (3,))[3]
    ct_p = _gpu_cov(ctx, dst, 15, (3,))[3]
    cs_c = R.crafted_covariances(len(src), 1e8, 5)
    ct_c = R.crafted_covariances(len(dst), 1e8, 6)
    for cs, ct in ((cs_p, ct_p), (cs_c, ct_c)):
        for mcd in (52.5, 0.3):
            corr, sqd = R.correspondences(src, dst, T, mcd)
            g, e = _lin(ctx, src, dst, cs, ct, T, mcd, np.eye(4))
            assert np.array_equal(g["corr"], corr) and np.array_equal(g["sqd"], sqd)
            _lin_within(g, R.Linearize(src, dst, cs, ct, T, corr))
            et = R.Linearize(src, dst, cs, ct, T, corr, T_trial=np.eye(4))
            assert abs(e - et.err) <= et.errb, (e, et.err, et.errb)
