"""Independent cross-checks of the oracle stages that the reference itself cannot pin (PCL / Eigen / FLANN / TEASER++ are
not installable here, SURVEY.md §8(c)): every stage is re-derived with a DIFFERENT tool (numpy / scipy / sklearn /
itertools) and compared with oracle/.  CPU only.

  covariance + PLANE & co.   numpy svd                         vs linalg.hpp one-sided Jacobi (nano_gicp_impl.hpp:298-357)
  Mahalanobis + linearize    numpy einsum restatement          vs oracle linearize          (nano_gicp_impl.hpp:173-270)
  LM optimum                 scipy.optimize.least_squares      vs oracle LM fixed point     (lsq_registration_impl.hpp:88-208)
  6x6 solve                  numpy.linalg.solve                vs the step the LM trace implies
  33-D feature 1-NN + mutual sklearn brute force               vs oracle.match              (matcher.cc:378-455)
  max clique                 exhaustive search (<= 20 nodes)   vs the greedy k-core clique  (PMC_HEU substitute)
  pcl::VoxelGrid             numpy fp32 restatement            vs orc_voxelize              (voxel_grid.hpp, SURVEY App. B.1)
"""
import itertools

import numpy as np
import pytest

import voxel_cases as vc


@pytest.fixture(scope="module")
def small(synth):
    return synth.make_pair(1001, 3000, 3500)


def _np_cov(pts, idx):
    nb = pts[idx].astype(np.float64)             # (n, k, 3)
    d = nb - nb.mean(1, keepdims=True)
    return np.einsum("nki,nkj->nij", d, d) / idx.shape[1]


def test_covariance_regularisation_vs_numpy_svd(oracle, small):
    _, dst, _ = small
    pts = dst[:, :3]
    _, knn = oracle.covariances(dst, 15, return_knn=True)
    cov = _np_cov(pts, knn)
    U, s, Vt = np.linalg.svd(cov)
    plane = np.einsum("nij,j,njk->nik", U, np.array([1.0, 1.0, 1e-3]), Vt)
    o = oracle.covariances_ex(dst, 15, 3)
    gap = s[:, 1] - s[:, 2]
    well = gap > 1e-6 * s[:, 0]                  # the plane normal is well defined
    assert well.mean() > 0.98
    assert np.abs(plane - o)[well].max() < 1e-7, np.abs(plane - o)[well].max()
    assert np.abs(oracle.covariances_ex(dst, 15, 0) - cov).max() < 1e-12   # NONE: the raw covariance
    mn = np.einsum("nij,nj,njk->nik", U, np.maximum(s, 1e-3), Vt)          # MIN_EIG
    assert np.abs(mn - oracle.covariances_ex(dst, 15, 1))[well].max() < 1e-7
    nmn = np.einsum("nij,nj,njk->nik", U, np.maximum(s / s[:, :1], 1e-3), Vt)  # NORMALIZED_MIN_EIG
    assert np.abs(nmn - oracle.covariances_ex(dst, 15, 2))[well].max() < 1e-7
    lam = cov + 1e-3 * np.eye(3)                                           # FROBENIUS
    li = np.linalg.inv(lam)
    fro = np.linalg.inv(li / np.linalg.norm(li.reshape(-1, 9), axis=1)[:, None, None])
    assert np.abs(fro - oracle.covariances_ex(dst, 15, 4)).max() < 1e-6 * np.abs(fro).max()


def _np_linearize(src, dst, cov_s, cov_t, T, corr):
    """nano_gicp_impl.hpp:205-209, 236-254 in numpy."""
    m = corr >= 0
    a, b = src[m, :3].astype(np.float64), dst[corr[m], :3].astype(np.float64)
    R, t = T[:3, :3], T[:3, 3]
    RCR = cov_t[corr[m]] + R @ cov_s[m] @ R.T
    M = np.linalg.inv(RCR)
    ta = a @ R.T + t
    e = b - ta
    J = np.zeros((len(a), 3, 6))
    J[:, 0, 1], J[:, 0, 2] = -ta[:, 2], ta[:, 1]
    J[:, 1, 0], J[:, 1, 2] = ta[:, 2], -ta[:, 0]
    J[:, 2, 0], J[:, 2, 1] = -ta[:, 1], ta[:, 0]
    J[:, :, 3:] = -np.eye(3)
    H = np.einsum("nia,nij,njb->ab", J, M, J)
    bb = np.einsum("nia,nij,nj->a", J, M, e)
    return H, bb, float(np.einsum("ni,nij,nj->", e, M, e)), M, m


def test_linearize_vs_numpy_restatement(oracle, synth, small):
    src, dst, _ = small
    cov_s, cov_t = oracle.covariances(src, 15), oracle.covariances(dst, 15)
    for T in (np.eye(4), synth.se3(yaw=0.01, pitch=0.002, t=(0.2, -0.1, 0.03))):
        o = oracle.linearize(src, dst, cov_s, cov_t, T)
        # correspondences from sklearn's brute-force NN on the fp32-transformed queries (ties aside, same answer)
        from sklearn.neighbors import NearestNeighbors
        q = oracle.transform_queries(T, src)
        _, nn = NearestNeighbors(n_neighbors=1, algorithm="brute").fit(dst[:, :3]).kneighbors(q)
        assert (nn[:, 0] == o["corr"]).mean() > 0.9999
        H, b, err, M, m = _np_linearize(src, dst, cov_s, cov_t, T, o["corr"])
        assert np.abs(H - o["H"]).max() < 1e-9 * np.abs(H).max()
        assert np.abs(b - o["b"]).max() < 1e-9 * max(np.abs(b).max(), 1.0)
        assert abs(err - o["err"]) < 1e-9 * err
        assert np.abs(M - o["mahal"][m]).max() < 1e-8 * np.abs(M).max()


def test_lm_fixed_point_vs_scipy_least_squares(oracle, synth):
    """A 200-point problem: at the oracle's final pose, with the correspondences and Mahalanobis matrices of a linearize
    there, scipy's trust-region least squares on the whitened residuals must not move further than the LM stopping
    tolerance (rotation_eps 2e-3, transformation_eps 1e-2), and the gradient the oracle reports must be that of the
    scipy objective."""
    from scipy.optimize import least_squares
    src, dst, Texp = synth.make_pair(1006, 200, 3000)  # 200 source points against a 3000-point target
    r = oracle.gicp_align(src, dst)
    assert r["converged"]
    cov_s, cov_t = oracle.covariances(src, 15), oracle.covariances(dst, 15)
    lin = oracle.linearize(src, dst, cov_s, cov_t, r["T"])
    m = lin["corr"] >= 0
    a = src[m, :3].astype(np.float64)
    b = dst[lin["corr"][m], :3].astype(np.float64)
    L = np.linalg.cholesky(lin["mahal"][m])       # M = L L^T, residual = L^T e

    def expm(w):
        th = np.linalg.norm(w)
        K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        if th < 1e-12:
            return np.eye(3) + K
        return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K

    def resid(x):
        Rd, td = expm(x[:3]), x[3:]
        R = Rd @ r["T"][:3, :3]
        t = Rd @ r["T"][:3, 3] + td
        e = b - (a @ R.T + t)
        return np.einsum("nji,nj->ni", L, e).ravel()
    f0 = resid(np.zeros(6))
    assert abs(f0 @ f0 - lin["err"]) < 1e-9 * lin["err"]
    # gradient of 1/2 |r|^2 at x = 0 is J^T M e with the oracle's sign convention b = sum J^T M e (J = d e / d x)
    eps = 1e-6
    g = np.array([(resid(eps * np.eye(6)[k]) @ resid(eps * np.eye(6)[k]) - resid(-eps * np.eye(6)[k]) @ resid(-eps * np.eye(6)[k])) / (4 * eps)
                  for k in range(6)])
    assert np.abs(g - lin["b"]).max() < 1e-5 * max(np.abs(lin["b"]).max(), 1.0)
    sol = least_squares(resid, np.zeros(6), method="trf", xtol=1e-14, ftol=1e-14, gtol=1e-14)
    assert np.abs(sol.x[:3]).max() < 2e-3 and np.abs(sol.x[3:]).max() < 1e-2, sol.x
    # and the step numpy's solver takes from (H, b) is the Gauss-Newton step scipy converges along
    gn = np.linalg.solve(lin["H"], -lin["b"])
    assert np.abs(gn - sol.x).max() < 5e-2 * max(np.abs(sol.x).max(), 1e-6) + 1e-7


def test_lm_trace_steps_vs_numpy_solve(oracle, synth, small):
    """Every accepted LM step of the trace: pose_{k+1} = exp(d) * pose_k with d = solve(H + lambda I, -b) by numpy
    (lsq_registration_impl.hpp:170-176) for SOME lambda in the geometric LM ladder that starts at 1e-9 * max diag H."""
    src, dst, _ = small
    r = oracle.gicp_align(src, dst, want_trace=True)
    tr = r["trace"]
    assert len(tr) >= 2
    for k in range(len(tr) - 1):
        P0, P1 = tr[k, :16].reshape(4, 4), tr[k + 1, :16].reshape(4, 4)
        H, b = tr[k, 16:52].reshape(6, 6), tr[k, 52:58]
        assert np.allclose(H, H.T, rtol=0, atol=1e-9 * np.abs(H).max())
        D = P1 @ np.linalg.inv(P0)
        lam_after, trials = tr[k, 59], int(tr[k, 60])
        # the lambda used lies between the initial 1e-9 * max|H_ii| and that times 2^(trials(trials-1)/2) of rejections, before
        # the acceptance rescaling by max(1/3, 1 - (2 rho - 1)^3) in [1/3, 2]: test the whole admissible ladder
        lam0 = 1e-9 * np.abs(np.diag(tr[0, 16:52].reshape(6, 6))).max()
        ok = False
        for lam in np.geomspace(lam0 / 3 ** (k + 1), lam0 * 2.0 ** (k + 10 * trials + 4), 400):
            d = np.linalg.solve(H + lam * np.eye(6), -b)
            if np.abs(d[3:] - D[:3, 3]).max() < 1e-6 * max(np.abs(d[3:]).max(), 1e-3):
                w = d[:3]
                th = np.linalg.norm(w)
                K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
                Rd = np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K if th > 0 else np.eye(3)
                ok = np.abs(Rd - D[:3, :3]).max() < 1e-6
                if ok:
                    break
        # lambda is tiny against H (1e-9 relative): the step is the Gauss-Newton step to 1e-6, whatever rung was used
        assert ok, (k, lam_after)


def test_feature_matching_vs_sklearn_bruteforce(oracle, synth):
    from sklearn.neighbors import NearestNeighbors
    src, dst, _ = synth.make_pair(2000, 2500, 2800, mode="quatro")
    _, _, fs = oracle.fpfh(src, 0.9, 1.5)
    _, _, fd = oracle.fpfh(dst, 0.9, 1.5)
    corr, mutual = oracle.match(src, dst, fs, fd)
    # matcher.cc:364-369: fi = larger cloud, fj = smaller; forward search fj -> fi, gate 35^2 in feature space; for the
    # FIRST j that reaches an unvisited i the reverse search i -> fj must return j (:424-431)
    fi, fj = (fd, fs) if len(dst) > len(src) else (fs, fd)
    use_i, use_j = np.abs(fi).sum(1) > 0, np.abs(fj).sum(1) > 0   # all-zero descriptors take no part (oracle/README.md)
    ii, jj = np.flatnonzero(use_i), np.flatnonzero(use_j)
    dfw, nfw = NearestNeighbors(n_neighbors=1, algorithm="brute").fit(fi[ii]).kneighbors(fj[jj])
    drv, nrv = NearestNeighbors(n_neighbors=1, algorithm="brute").fit(fj[jj]).kneighbors(fi[ii])
    want, seen = [], set()
    for a, j in enumerate(jj):
        i = ii[nfw[a, 0]]
        if dfw[a, 0] ** 2 > 35.0 ** 2 or i in seen:
            continue
        seen.add(i)
        if jj[nrv[nfw[a, 0], 0]] == j:
            want.append((i, j))
    want = np.array(want, np.int32)
    # fp32 ties between near-identical ground-plane descriptors may resolve differently in sklearn's float64 path:
    # require the overwhelming majority to agree and every oracle pair to be a true mutual nearest pair
    got = set(map(tuple, mutual.tolist()))
    assert len(got & set(map(tuple, want.tolist()))) >= 0.97 * max(len(got), len(want)), (len(got), len(want))
    for i, j in list(got)[:200]:
        d_ij = ((fi[i].astype(np.float64) - fj[j]) ** 2).sum()
        assert d_ij <= ((fi[ii].astype(np.float64) - fj[j]) ** 2).sum(1).min() * (1 + 1e-5) + 1e-6
        assert d_ij <= ((fj[jj].astype(np.float64) - fi[i]) ** 2).sum(1).min() * (1 + 1e-5) + 1e-6
    assert len(corr) > 0


def test_greedy_clique_vs_exhaustive_max_clique(oracle):
    """The PMC_HEU substitute (greedy clique in k-core order) against an exhaustive maximum clique on small TIM graphs:
    quantifies the substitution (the heuristic may legitimately be smaller; on inlier-dominated graphs it is not)."""
    rng = np.random.default_rng(4)
    gaps = []
    for trial in range(40):
        n_in, n_out = int(rng.integers(5, 12)), int(rng.integers(3, 9))
        n = n_in + n_out
        src = rng.uniform(-20, 20, (n, 3)).astype(np.float32)
        yaw = rng.uniform(-0.3, 0.3)
        R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
        dst = (src.astype(np.float64) @ R.T + np.array([3.0, -2.0, 0.2]) + rng.normal(0, 0.03, (n, 3))).astype(np.float32)
        dst[n_in:] += rng.uniform(-15, 15, (n_out, 3)).astype(np.float32)  # outliers
        corr = np.c_[np.arange(n), np.arange(n)].astype(np.int32)
        o = oracle.quatro_solve(src, dst, corr)
        # the consistency graph in numpy (TEASER++: | |b_ij| - |a_ij| | <= 2 * noise_bound, cbar2 = 1)
        A = np.linalg.norm(src[:, None].astype(np.float64) - src[None].astype(np.float64), axis=2)
        B = np.linalg.norm(dst[:, None].astype(np.float64) - dst[None].astype(np.float64), axis=2)
        adj = np.abs(B - A) <= 2 * 0.3
        np.fill_diagonal(adj, False)
        best = 0
        for k in range(n, 0, -1):
            if any(all(adj[a, b] for a, b in itertools.combinations(c, 2)) for c in itertools.combinations(range(n), k)):
                best = k
                break
        clique = o["clique"]
        assert all(adj[a, b] for a, b in itertools.combinations(clique.tolist(), 2)), "the oracle's set must be a clique"
        assert len(clique) <= best
        gaps.append(best - len(clique))
        if len(clique) >= 3 and o["valid"]:
            est_yaw = np.arctan2(o["T"][1, 0], o["T"][0, 0])
            assert abs(est_yaw - yaw) < 0.05
    gaps = np.array(gaps)
    assert (gaps == 0).mean() >= 0.9 and gaps.max() <= 1, gaps  # measured: the greedy clique is maximum on these graphs


def _np_voxel_grid(pts, leaf):
    """pcl::VoxelGrid::applyFilter (PCL 1.10) in numpy, fp32 wherever PCL is: inverse leaf 1.0f / L; the int64 guard on
    trunc((max - min) * inv) + 1 per axis; min_b = floor(min * inv), div_b = floor(max * inv) - min_b + 1; the index
    ijk0 + ijk1 * div_b0 + ijk2 * div_b0 * div_b1 wrapped to unsigned int as PCL stores it; a stable sort by that
    index alone (ascending point index inside a voxel); fp32 running sums added strictly in that order, divided once.
    -> (points, dict(overflow, cells = guard product, max_key))."""
    p = np.ascontiguousarray(pts, np.float32)
    xyz = p[:, :3]
    inv = np.float32(1) / np.float32(leaf)
    mn, mx = xyz.min(0), xyz.max(0)
    cells = int(np.prod(((mx - mn) * inv).astype(np.int64) + 1, dtype=object))
    if cells > vc.INT32_MAX:
        return p.copy(), dict(overflow=True, cells=cells, max_key=None)
    min_b = np.floor(mn * inv).astype(np.int64)
    div_b = np.floor(mx * inv).astype(np.int64) - min_b + 1
    ijk = (np.floor(xyz * inv) - min_b.astype(np.float32)).astype(np.int64)
    key = ((ijk[:, 0] + ijk[:, 1] * div_b[0] + ijk[:, 2] * (div_b[0] * div_b[1])) & 0xFFFFFFFF).astype(np.uint32)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    counts = np.diff(np.r_[starts, len(ks)])
    s = np.zeros((len(starts), 4), np.float32)
    for k in range(int(counts.max())):  # k-th point of every voxel that has one: sequential per voxel (np.sum is pairwise)
        live = counts > k
        s[live] = s[live] + p[order[starts[live] + k]]
    return s / counts[:, None].astype(np.float32), dict(overflow=False, cells=cells, max_key=int(ks[-1]))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_voxel_grid_vs_numpy_restatement(oracle, synth):
    """orc_voxelize equals the numpy restatement bit for bit (count, order, centroids incl. intensity) on every crafted
    cloud of voxel_cases and on keyframes of the test sequence at five leaf sizes; the cases reach what they are meant to."""
    info = {}
    for name, leaf, cloud in vc.crafted():
        want, info[name] = _np_voxel_grid(cloud, leaf)
        got = oracle.voxelize(cloud, leaf)
        assert got.shape == want.shape and np.array_equal(_bits(got), _bits(want)), name
    seq = vc.sweep_sequence(synth)
    for k in vc.SWEEP_KEYFRAMES:
        for leaf in vc.SWEEP_LEAVES:
            want, info[(k, leaf)] = _np_voxel_grid(seq["clouds"][k], leaf)
            got = oracle.voxelize(seq["clouds"][k], leaf)
            assert got.shape == want.shape and np.array_equal(_bits(got), _bits(want)), (k, leaf)
    assert info["guard_below"]["cells"] == vc.INT32_MAX - 1 and not info["guard_below"]["overflow"]
    assert info["guard_above"]["cells"] == 2 ** 31 and info["guard_above"]["overflow"]
    assert not info["index_wrap"]["overflow"] and info["index_wrap"]["max_key"] > vc.INT32_MAX
    # the third 11-bit pass of the device sort sees real digits: keys above 2^28
    big = sorted(str(c) for c, i in info.items() if not i["overflow"] and i["max_key"] >= 2 ** 28)
    assert big == sorted(map(str, ["guard_below", "index_wrap", (0, 0.05), (70, 0.05)])), big
    assert [c for c, i in info.items() if i["overflow"]] == ["guard_above"]
    assert len(oracle.voxelize(vc.one_voxel(13), 0.3)) == 1
    assert len(oracle.voxelize(vc.own_voxels(14), 1.0)) == 3000
