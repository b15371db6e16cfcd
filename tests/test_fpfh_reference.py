"""The fp64 restatement of the feature stage (tests/fpfh_ref.py): known answers, and the CPU oracle pinned against it.

The oracle's SPFH adds incr once per pair in fp32, so at hundreds of neighbours it is the less accurate side of an
oracle-vs-kernel comparison.  Here both of its outputs are stated against fp64 instead: the SPFH counts it implies must be
the exact counts (up to ambiguous f1 bins), and its FPFH must lie within a bound derived for its own order of fp32 sums.
"""
import numpy as np
import pytest

import fpfh_ref as R


def _full(xyz, nr, fr, r2=R.kernel_r2):
    cn = R.radius_csr(xyz, r2(nr))
    nrm, lam, dot, err = R.normals(xyz, cn)
    cf = R.radius_csr(xyz, r2(fr))
    counts, amb, cnt = R.spfh_counts(xyz, nrm, cf)
    return cn, nrm, lam, cf, counts, amb, cnt


def test_planar_lattice_known_answer():
    g = np.arange(-6, 7) * 0.25
    X, Y = np.meshgrid(g, g)
    xyz = np.stack([X.ravel() + 3.0, Y.ravel() - 2.0, np.full(X.size, 1.5)], 1).astype(np.float32)
    cn, nrm, lam, cf, counts, amb, cnt = _full(xyz, 0.9, 1.5)
    # viewpoint at the origin, plane at z = 1.5: every normal points down
    assert np.array_equal(nrm, np.tile(np.float32([0, 0, -1]), (len(xyz), 1)))
    assert np.all(lam[:, 0] == 0.0)
    # n1 = n2 = -z, d in the plane: f2 = f3 = 0, so the middle bin (5) of blocks 2 and 3 gets every pair
    pairs = cnt - 1
    assert np.array_equal(counts[:, 11 + 5], pairs) and np.array_equal(counts[:, 22 + 5], pairs)
    assert counts[:, 11:22].sum() == counts[:, 11 + 5].sum() and counts[:, 22:].sum() == counts[:, 22 + 5].sum()
    assert np.array_equal(counts[:, :11].sum(1), pairs)
    F = R.Fpfh(cf, counts, amb, cnt, nrm)
    assert np.allclose(F.v[:, 16], 100.0) and np.allclose(F.v[:, 27], 100.0)
    assert np.allclose(F.v.reshape(-1, 3, 11).sum(2), 100.0)


def test_tiny_clusters_and_collinear_points():
    xyz = np.float32([[0, 0, 10], [0.1, 0, 10],                      # two points: no normal
                      [20, 0, 0], [20.1, 0, 0], [20.2, 0, 0]])       # three collinear points: degenerate, but a normal
    cn, nrm, lam, cf, counts, amb, cnt = _full(xyz, 0.9, 1.5)
    assert np.array_equal(cn.counts, [2, 2, 3, 3, 3])
    assert np.isnan(nrm[:2]).all() and np.isfinite(nrm[2:]).all()
    assert np.allclose(np.linalg.norm(nrm[2:], axis=1), 1.0, atol=1e-7)
    assert np.allclose(nrm[2:, 0], 0.0, atol=1e-7)  # orthogonal to the line; which vector of the plane is free
    assert np.allclose(lam[2:, :2], 0.0, atol=1e-12)
    assert np.array_equal(cnt, [2, 2, 3, 3, 3])
    # points without a normal have no SPFH; the line's pairs are all valid (d not along any normal)
    assert counts[:2].sum() == 0 and np.array_equal(counts[2:].reshape(-1, 3, 11).sum(2), np.full((3, 3), 2))


def test_duplicates_and_vn_zero_rejected():
    n = np.float32([[0, 0, 1], [0, 0, 1], [0, 0, 1], [0, 0, 1]])
    p1 = np.float32([[0, 0, 0]] * 4)
    p2 = np.float32([[0, 0, 0],        # exact duplicate: f4 == 0
                     [0, 0, 0.5],      # d along n1 (and n2): vn == 0
                     [0.5, 0, 0],      # in-plane: valid, f2 = f3 = 0
                     [0, 0.5, 0]])
    valid, f1, f2, f3 = R.pair_features(p1, n, p2, n)
    assert valid.tolist() == [False, False, True, True]
    assert f2[2:].tolist() == [0.0, 0.0] and f3[2:].tolist() == [0.0, 0.0]
    # a cloud with a duplicated point: the duplicate counts as a neighbour (cnt, incr) but adds no pair and no FPFH weight
    g = np.arange(-3, 4) * 0.3
    X, Y = np.meshgrid(g, g)
    xyz = np.stack([X.ravel(), Y.ravel(), np.full(X.size, -2.0)], 1).astype(np.float32)
    xyz = np.concatenate([xyz, xyz[24:25]])
    cn, nrm, lam, cf, counts, amb, cnt = _full(xyz, 0.9, 1.5)
    d = len(xyz) - 1
    assert np.array_equal(counts[24], counts[d])
    assert counts[24, :11].sum() == cnt[24] - 2  # self and the duplicate add no pair
    F = R.Fpfh(cf, counts, amb, cnt, nrm)
    assert F.n[24] == cnt[24] - 2 and np.array_equal(F.v[24], F.v[d])


def test_points_exactly_on_the_radius_are_excluded():
    g = np.arange(-6, 7) * 0.5
    X, Y = np.meshgrid(g, g)
    xyz = np.stack([X.ravel(), Y.ravel(), np.full(X.size, 4.0)], 1).astype(np.float32)
    c = len(xyz) // 2
    assert np.array_equal(xyz[c], [0, 0, 4])
    cf = R.radius_csr(xyz, R.kernel_r2(1.5), queries=[c])
    assert R.kernel_r2(1.5) == np.float32(2.25)
    d2 = ((xyz - xyz[c]) ** 2).sum(1)
    on = np.flatnonzero(d2 == 2.25)  # (1.5, 0) and its rotations
    assert len(on) == 4 and not np.isin(on, cf.indices).any()
    assert np.array_equal(np.sort(cf.indices), np.flatnonzero(d2 < 2.25))


@pytest.fixture(scope="module")
def dense_crop(synth):
    """A crop of the bench's raw scan: 20k-some points, thousands of neighbours per FPFH ball."""
    _, dst, _ = synth.make_pair(2000, 100000, 100000, mode="quatro")
    c = np.median(dst[:, :2], 0)
    for h in np.arange(2.0, 12.0, 0.5):  # the smallest square around the scan's median point that holds 20k points
        m = (np.abs(dst[:, 0] - c[0]) < h) & (np.abs(dst[:, 1] - c[1]) < h)
        if m.sum() >= 20000:
            break
    return np.ascontiguousarray(dst[m])


def test_oracle_against_fp64_restatement_on_dense_crop(oracle, dense_crop):
    xyz = dense_crop
    on, osp, of = oracle.fpfh(xyz, 0.9, 1.5)
    # the oracle's own normals go in; its radius passes through float before squaring
    cf = R.radius_csr(xyz[:, :3], R.oracle_r2(1.5))
    counts, amb, cnt = R.spfh_counts(xyz[:, :3], on, cf)
    nb = cnt
    print("\ndense crop: %d points, FPFH-ball sizes min/median/99%%/max %s, ambiguous f1 pairs %d"
          % (len(xyz), np.quantile(nb, [0, 0.5, 0.99, 1.0]).astype(int).tolist(), amb.sum()))
    assert 20000 <= len(xyz) <= 40000 and np.median(nb) >= 200
    # 1. the SPFH counts the oracle implies equal the exact counts, except for ambiguous f1 pairs
    incr = np.where(cnt >= 2, np.float32(100) / np.maximum(cnt - 1, 1).astype(np.float32), np.float32(0))
    rec = np.rint(osp / np.where(incr > 0, incr, 1)[:, None]).astype(np.int64)
    assert np.array_equal(rec[:, 11:], counts[:, 11:]), "f2/f3 bins are exact fp32 arithmetic"
    assert np.array_equal(rec[:, :11].sum(1), counts[:, :11].sum(1))
    diff = np.abs(rec[:, :11] - counts[:, :11])
    assert np.all(diff <= R.amb_touch(amb)[:, :11]), "an f1 count differs away from any ambiguous pair"
    # 2. the oracle's FPFH lies within the bound of its own fp32 order of operations
    F = R.Fpfh(cf, counts, amb, cnt, on, m=R.oracle_m(cf, cnt))
    err = np.abs(of.astype(np.float64) - F.v)
    assert np.all(err <= F.bound), np.argwhere(err > F.bound)[:5]
    K = R.Fpfh(cf, counts, amb, cnt, on)  # the same reference with the kernel's (fma, block sums at the end) bound
    r_o, r_k = err / np.where(F.bound > 0, F.bound, 1), err / np.where(K.bound > 0, K.bound, 1)
    print("oracle FPFH vs fp64: max |err| %.3g, max err/bound %.3f (oracle's order), %.3f (measured against the kernel's "
          "tighter bound); median err/bound %.3g" % (err.max(), r_o.max(), r_k.max(), np.median(r_o[F.v > 0])))
