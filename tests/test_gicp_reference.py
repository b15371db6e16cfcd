"""The CPU oracle's NanoGICP covariances and linearize pass against the fp64 restatement (tests/gicp_ref.py), every point
within its bound, at the edge scenes; known answers for the scenes; and the wrong variant of each rule (higher index on
ties, divisor min(n, k), gate <=) shown to leave the bound, so that the bound can tell them apart.

NORMALIZED_MIN_EIG at a zero raw covariance (k = 1, or k copies of one point) is NaN, as the reference's
(s / s.maxCoeff()).array().max(1e-3) gives: 0 / 0 under std::max keeps the NaN.
"""
import numpy as np
import pytest

import gicp_ref as R

KS = (1, 5, 15, 20, 32)
METHODS = (0, 1, 2, 3, 4)


@pytest.fixture(autouse=True)
def own_kdtree(oracle):
    """The oracle's own kd-tree resolves ties to the lower index, as the engine does."""
    oracle.use_ref_nanoflann(False)
    yield


@pytest.fixture(scope="module")
def scenes():
    return R.scenes()


# ---------------------------------------------------------------------------------------------------------------------
# the scenes reach their edges: known answers
def test_scene_known_answers(scenes):
    # every tested k >= 2 has points whose tie shell is cut at rank k (k = 1 keeps only the point itself: no tie can move it)
    for k in (2, 5, 7, 8, 9, 14, 15, 16, 19, 20, 21, 31, 32):
        _, d2 = R.knn(scenes["lattice"], k + 1)
        assert R.straddles(d2, k).sum() > 0, k
    # duplicates: runs longer than k give exactly zero covariances, shorter ones do not
    c = R.Cov(scenes["duplicates"], 15)
    assert c.zero.sum() > 0 and (~c.zero).sum() > 0
    # a line: rank 1 exactly (the two smaller eigenvalues vanish in exact arithmetic)
    c = R.Cov(scenes["collinear"], 15)
    assert np.abs(c.w[:, :2]).max() <= 1e-15 * c.w[:, 2].min() and c.w[:, 2].min() > 0
    # the tilted plane: the normal is (-0.5, 0.25, 1) / |.|, lam1 = 0 up to the fp64 two-pass round-off
    c = R.Cov(scenes["tilted_plane"], 15)
    nrm = np.array([-0.5, 0.25, 1.0]) / np.linalg.norm([-0.5, 0.25, 1.0])
    assert np.abs(np.abs(c.U[:, :, 0] @ nrm) - 1).max() < 1e-12
    assert np.abs(c.w[:, 0]).max() < 1e-15 * c.w[:, 2].max() and c.w[:, 1].min() > 1e-3
    # isotropic: octahedron + centre at k = 7 and cube + centre at k = 9 are multiples of I
    for k, r2 in ((7, 2 * 0.0625 / 7), (9, 8 * 0.0625 / 9)):
        c = R.Cov(scenes["isotropic"], k)
        iso = np.abs(c.C - r2 * np.eye(3)).reshape(len(c.C), 9).max(1) < 1e-16
        assert iso.sum() >= 6, (k, iso.sum())
    # millimetre clusters: MIN_EIG clamps every eigenvalue to 1e-3
    c = R.Cov(scenes["millimetre"], 15)
    assert c.w.max() < 1e-4
    assert np.abs(c.reference(1) - 1e-3 * np.eye(3)).max() < R.C_EIG * R.EPS64 * 1e-3
    # k = 1: every covariance is zero
    assert R.Cov(scenes["near"], 1).zero.all()
    # the far copies: the same geometry, the absolute-coordinate bound grows with the distance
    a, b = R.Cov(scenes["near"], 15), R.Cov(scenes["far3km"], 15)
    assert np.median(b.dF / a.dF) > 100


def test_knn_kdtree_path_equals_brute_force(synth):
    """The cKDTree + fp32 re-rank path (100k scans) returns what the brute force returns, ties included."""
    pts = np.concatenate([synth.make_pair(1001, 5000, 6000)[1][:, :3], R.lattice() + np.float32(50)])
    for k in (1, 15, 32):
        bi, bd = R.knn(pts, k)
        old = R.BRUTE_MAX
        R.BRUTE_MAX = 100
        try:
            ki, kd = R.knn(pts, k)
        finally:
            R.BRUTE_MAX = old
        assert np.array_equal(bi, ki) and np.array_equal(bd, kd), k


def test_knn_equals_oracle_bruteforce(oracle, scenes):
    for name in ("lattice", "duplicates", "collinear"):
        p = scenes[name]
        for k in (1, 15, 32):
            ri, rd = R.knn(p, k)
            oi, od = oracle.knn(p, p, k, brute=True)
            assert np.array_equal(ri, oi) and np.array_equal(rd, od), (name, k)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle within the bounds
def _oracle_within(oracle, pts, k, methods=METHODS, tag=""):
    c = R.Cov(pts, k)
    for m in methods:
        o = oracle.covariances_ex(pts, k, m)
        r, kind = c.check(o, m, solver=R.ORACLE_SVD)
        assert np.all(r <= 1), (tag, k, m, float(np.max(r)), int((r > 1).sum()), np.bincount(kind, minlength=3))


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", ["lattice", "duplicates", "collinear", "thin_edges", "tilted_plane", "isotropic",
                                  "millimetre", "near", "far1km", "far3km"])
def test_oracle_covariances_within_bound(oracle, scenes, name, k):
    _oracle_within(oracle, scenes[name], k, tag=name)


@pytest.mark.parametrize("k", KS)
def test_oracle_covariances_tiny_clouds(oracle, k):
    for pts in R.tiny(k):
        _oracle_within(oracle, pts, k, tag=len(pts))


def test_oracle_covariances_scan(oracle, synth):
    pts = synth.make_pair(1001, 5000, 6000)[1][:, :3]
    for k in (15, 20):
        _oracle_within(oracle, pts, k, tag="scan")


def test_normalized_min_eig_nan_at_zero_covariance(oracle, scenes):
    """k copies of one point (and k = 1): the reference's 0 / 0 under std::max is NaN, and so is the oracle."""
    p = scenes["duplicates"]
    c = R.Cov(p, 15)
    o = oracle.covariances_ex(p, 15, 2)
    assert c.zero.sum() > 0
    assert np.isnan(o[c.zero]).all() and np.isfinite(o[~c.zero]).all()
    assert np.isnan(oracle.covariances_ex(p, 1, 2)).all()
    for m in (0, 1, 3, 4):
        assert np.isfinite(oracle.covariances_ex(p, 15, m)).all(), m


# ---------------------------------------------------------------------------------------------------------------------
# the wrong variants leave the bound
def test_wrong_tie_rule_leaves_the_bound(oracle, scenes):
    p = scenes["lattice"]
    for k in (5, 15, 20, 32):
        o = oracle.covariances_ex(p, k, 0)
        r, _ = R.Cov(p, k).check(o, 0)
        assert np.all(r <= 1)
        r, _ = R.Cov(p, k, tie="high").check(o, 0)
        assert (r > 1e3).sum() > 0, k


def test_wrong_divisor_leaves_the_bound(oracle):
    for k in (5, 15, 32):
        for pts in R.tiny(k)[1:k - 1]:  # 2 <= n < k
            o = oracle.covariances_ex(pts, k, 0)
            r, _ = R.Cov(pts, k, divisor=lambda m, kk: min(m, kk)).check(o, 0)
            assert (r > 1e3).all(), (k, len(pts))


def _lin_check(o, ref):
    assert np.all(np.abs(o["H"] - ref.H) <= ref.Hb), np.max(np.abs(o["H"] - ref.H) / ref.Hb)
    assert np.all(np.abs(o["b"] - ref.b) <= ref.bb), np.max(np.abs(o["b"] - ref.b) / ref.bb)
    assert abs(o["err"] - ref.err) <= ref.errb, (o["err"], ref.err, ref.errb)


@pytest.mark.parametrize("offset", [(0.0, 0.0, 0.0), (1000.0, 0.0, 0.0)])
def test_oracle_linearize_at_the_gate_and_ties(oracle, offset):
    """Source points exactly 0.5 m from the target (d2 = 0.25, exactly representable) with max_corr_dist = 0.5: strict '<'
    rejects them; correspondence ties on the lattice go to the lower index."""
    src, tgt, want = R.lattice_pair(offset)
    Q = np.linalg.qr(np.random.default_rng(3).normal(size=(3, 3)))[0]
    cs = R.crafted_covariances(len(src), 1e8, 1, Q)
    ct = R.crafted_covariances(len(tgt), 1e8, 2, Q)
    T = np.eye(4)
    for mcd in (0.5, 1.0, 52.5):
        corr, sqd = R.correspondences(src, tgt, T, mcd)
        assert np.array_equal(sqd.astype(np.float64), want)
        if mcd == 0.5:
            assert (corr[want == 0.25] == -1).all() and (corr[want < 0.25] >= 0).all()
            wrong, _ = R.correspondences(src, tgt, T, mcd, gate="le")
            assert (wrong[want == 0.25] >= 0).all()
        o = oracle.linearize(src, tgt, cs, ct, T, max_corr_dist=mcd)
        assert np.array_equal(o["corr"], corr) and np.array_equal(o["sqd"], sqd), mcd
        ref = R.Linearize(src, tgt, cs, ct, T, corr)
        assert ref.kappa.max() > 1e6
        _lin_check(o, ref)
        if mcd == 0.5:  # the gate <= variant moves H outside the bound
            bad = R.Linearize(src, tgt, cs, ct, T, wrong)
            assert (np.abs(o["H"] - bad.H) > bad.Hb).any()


def test_oracle_linearize_and_compute_error_scan(oracle, synth):
    src, dst, _ = synth.make_pair(1001, 3000, 3500)
    cs = oracle.covariances(src, 15)
    ct = oracle.covariances(dst, 15)
    T = synth.se3(yaw=0.02, pitch=-0.004, t=(0.3, -0.2, 0.05))
    for T_lin in (np.eye(4), T):
        corr, sqd = R.correspondences(src, dst, T_lin, 52.5)
        o = oracle.linearize(src, dst, cs, ct, T_lin)
        assert np.array_equal(o["corr"], corr) and np.array_equal(o["sqd"], sqd)
        _lin_check(o, R.Linearize(src, dst, cs, ct, T_lin, corr))
        e = oracle.compute_error(src, dst, cs, ct, T_lin, T)
        ref = R.Linearize(src, dst, cs, ct, T_lin, corr, T_trial=T)
        assert abs(e - ref.err) <= ref.errb, (e, ref.err, ref.errb)
