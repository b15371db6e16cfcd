"""An fp64 restatement of the NanoGICP half (nano_gicp_impl.hpp:173-357), numpy / scipy only.

It states what k_covariance / k_covariance_large (covariances and their regularisation) and k_gicp_search / k_gicp_accum
(correspondences, Mahalanobis matrices, H, b and the error sum) compute, and how far an fp64 implementation may lie from
it, so that the kernels (and the CPU oracle) are checked against a per-point bound derived from the arithmetic instead of
against each other on a quantile:

* neighbour sets are exact: fp32 ``d2 = ((dx*dx) + dy*dy) + dz*dz`` with ``d = query - point``, ordered by (d2, lower
  original index), the point itself included; when n < k all n points are used and the divisor is still k;
* the raw covariance is a two-pass fp64 one about the query point (free of the cancellation of a far origin), with
  ``eigh`` for its eigenvalues; ``Cov.bound`` is a rigorous per-entry bound on the device's two sequential passes in
  absolute coordinates (NONE), and the other methods' bounds follow from it (``Cov.check``);
* correspondences are the exact fp32 1-NN of the fp32-transformed source under the strict gate ``(double)d2 < r*r``;
  ``Linearize`` restates H, b and the error sum in 64-bit-mantissa long double, with a per-entry bound.
"""
import math

import numpy as np
from scipy.spatial import cKDTree

U64 = 2.0 ** -53  # unit round-off of fp64
EPS64 = 2.0 ** -52
U32 = 2.0 ** -24
PLANE_EPS = 1e-3  # the regularisation constant of every method (nano_gicp_impl.hpp:325-350)
BRUTE_MAX = 30000
# Eigen-solver constants (see Cov.check).  C_EIG: a backward-stable 3x3 solver (cyclic Jacobi, the oracle's SVD, the
# cofactor inverse) errs by a small multiple of eps |C|; 64 covers it with room.  C_PLANE: sym3_smallest_evec's closed form
# turns eps into an eigenvalue error ~ eps p^2 / g and an eigenvector error ~ eps (p/g)^2 (smallmath.cuh), i.e. eps (p/g) *
# (lam3 / g); it hands over to Jacobi below phi = 1e-3, where g / p ~ 2 sqrt(3) phi, so p / g <= 1 / (2 sqrt(3) 1e-3) on the
# closed-form path and C_PLANE = C_EIG / (2 sqrt(3) 1e-3) ~ 1.8e4.
C_EIG = 64.0
C_PLANE = C_EIG / (2.0 * math.sqrt(3.0) * 1e-3)
# Forward error of the cofactor (adjugate / det) 3x3 inverse of the engine: the adjugate's 2x2 minors carry eps s1^2 of
# absolute error, so |dM| <= C_INV eps kappa (s1 / s2) |M|_F (s1 >= s2 >= s3 the singular values; it is not backward stable
# and exceeds eps kappa |M| where s2 is small too).  Measured up to 0.42 eps kappa (s1 / s2) |M|_F at kappa ~ 1e8.
C_INV = 16.0
# The CPU oracle's SVD (oracle/linalg.hpp, one-sided Jacobi) forms U column by column as A v_j / s_j: a column of a small
# singular value carries eps s_1 / s_j of noise, so U diag(.) V^T is not exactly symmetric.  Measured: up to 4.1e3 times
# the device's solver bound on these scenes; the oracle is held to 2^13 times it.
ORACLE_SVD = 8192.0
VACUOUS = 0.05  # a perturbation bound on an angle above this says nothing: check a subspace instead


def gamma(m, u=U64):
    """gamma_m = m u / (1 - m u) (Higham, Lemma 3.1)."""
    mu = np.asarray(m, np.float64) * u
    return mu / (1.0 - mu)


def d2_f32(q, p):
    """The engine's fp32 squared distance, no contraction: ((dx*dx) + dy*dy) + dz*dz, d = q - p."""
    d = np.asarray(q, np.float32) - np.asarray(p, np.float32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _keys(d2, idx, tie):
    """(d2, index) as one int64 order key: fp32 bits of a non-negative d2 are monotone; tie='high' inverts the index rule."""
    bits = np.ascontiguousarray(d2, np.float32).view(np.int32).astype(np.int64) << 32
    return bits | (idx if tie == "low" else (0x7FFFFFFF - idx))


def knn(xyz, k, queries=None, tie="low", margin=16):
    """Exact k-NN of the query rows (default: every point) in xyz under the engine's rule -> (idx (q, m), d2 (q, m)),
    m = min(k, n), ascending.  tie='high' is the wrong variant (higher index first on equal d2).
    Up to BRUTE_MAX points a chunked brute force; beyond, cKDTree candidates (k + margin) re-ranked by the fp32 d2, with the
    margin asserted: every point outside the candidates is farther (exactly) than the last candidate, whose fp32 d2 lies
    within 6 u32 of its exact value, so if that exceeds the k-th fp32 d2 by more than 1e-6 relative no outsider can enter."""
    xyz = np.ascontiguousarray(np.asarray(xyz)[:, :3], np.float32)
    n = len(xyz)
    q = np.arange(n) if queries is None else np.asarray(queries, np.int64)
    m = min(k, n)
    out_i = np.empty((len(q), m), np.int64)
    out_d = np.empty((len(q), m), np.float32)
    if n <= BRUTE_MAX or m + margin >= n:
        step = max(1, (1 << 22) // n)
        ar = np.arange(n, dtype=np.int64)
        for s in range(0, len(q), step):
            qs = q[s:s + step]
            d2 = d2_f32(xyz[qs][:, None, :], xyz[None, :, :])
            key = _keys(d2, ar[None, :], tie)
            part = np.argpartition(key, m - 1, axis=1)[:, :m] if m < n else np.broadcast_to(ar, (len(qs), n))
            kp = np.take_along_axis(key, part, 1)
            o = np.argsort(kp, axis=1)
            sel = np.take_along_axis(part, o, 1)
            out_i[s:s + step] = sel
            out_d[s:s + step] = np.take_along_axis(d2, sel, 1)
        return out_i, out_d
    kk = m + margin
    dist, cand = cKDTree(xyz.astype(np.float64)).query(xyz[q].astype(np.float64), k=kk, workers=-1)
    d2 = d2_f32(xyz[q][:, None, :], xyz[cand])
    o = np.argsort(_keys(d2, cand, tie), axis=1)[:, :m]
    out_i[:] = np.take_along_axis(cand, o, 1)
    out_d[:] = np.take_along_axis(d2, o, 1)
    held = dist[:, -1] ** 2 * (1.0 - 1e-6) > out_d[:, -1].astype(np.float64)
    assert held.all(), ("kNN candidate margin did not hold", int((~held).sum()))
    return out_i, out_d


def straddles(d2_sorted, k):
    """Rows whose tie at rank k is cut by the k-NN: the k-th and (k+1)-th nearest are at the same d2 (needs k+1 columns)."""
    return d2_sorted[:, k - 1] == d2_sorted[:, k]


class Cov:
    """Raw NanoGICP covariances of every point of xyz with k neighbours (nano_gicp_impl.hpp:298-321), and the bounds.

    ``C`` (n,3,3) fp64; ``w`` ascending eigenvalues, ``U`` eigenvectors; ``bound`` (n,3,3) the most the device's
    computation may differ per entry; ``dF`` its Frobenius norm.  ``divisor`` (default k) and ``tie`` exist for the wrong
    variants only."""

    def __init__(self, xyz, k, tie="low", divisor=None, idx=None):
        xyz = np.ascontiguousarray(np.asarray(xyz)[:, :3], np.float32)
        self.k = k
        if idx is None:
            idx, _ = knn(xyz, k, tie=tie)
        self.idx = idx
        n, m = idx.shape
        kd = float(k if divisor is None else divisor(m, k))
        X = xyz.astype(np.float64)[idx]                      # (n, m, 3) absolute, exact
        qp = xyz.astype(np.float64)[:, None, :]
        L = X - qp                                           # exact: the difference of two nearby fp32 values
        # mean - q = sum(x_j - q) / k - (1 - m / k) q: the divisor-k mean is not the centroid when m < k
        mu = L.sum(1) / kd - (1.0 - m / kd) * qp[:, 0, :]
        V = L - mu[:, None, :]
        self.C = np.einsum("nja,njb->nab", V, V) / kd
        self.w, self.U = np.linalg.eigh(self.C)
        # Device (and oracle), per coordinate a, with sequential fp64 sums over the m neighbours:
        #   mu^ = fl(fl(sum_j p_ja) / k)                 |mu^ - mu| <= gamma_m sum_j |p_ja| / k =: dm_a
        #   c^_ab = fl(fl(sum_j fl(fl(p_ja - mu^_a) fl(p_jb - mu^_b))) * fl(1 / k))
        #        = (1/k) sum_j (v_ja - dmu_a)(v_jb - dmu_b) (1 + theta_j),  |theta_j| <= gamma_{m+4}
        # so |c^_ab - c_ab| <= (1 + gamma_{m+4}) S_ab - (1/k) sum_j |v_ja||v_jb| with S_ab = (1/k) sum_j (|v_ja| + dm_a)(|v_jb| + dm_b).
        # The restatement's own error (local coordinates; the (1 - m/k) q term rounds once) is below gamma_{m+4} times
        # the same sums, so the bound uses 2 gamma_{m+4} and adds u |1 - m/k| |q| to dm.
        dm = gamma(m) * np.abs(X).sum(1) / kd + U64 * abs(1.0 - m / kd) * np.abs(qp[:, 0, :])
        A = np.abs(V)
        S = np.einsum("nja,njb->nab", A + dm[:, None, :], A + dm[:, None, :]) / kd
        P = np.einsum("nja,njb->nab", A, A) / kd
        self.bound = (1.0 + 2.0 * gamma(m + 4)) * S - P
        self.dF = np.sqrt((self.bound ** 2).sum((1, 2)))

    def reference(self, method):
        """The regularised covariance of nano_gicp_impl.hpp:323-353 from the fp64 eigen-decomposition."""
        w, U, n = self.w, self.U, len(self.C)
        if method == 0:
            return self.C.copy()
        if method == 3:
            u = U[:, :, 0]
            return np.eye(3) - (1.0 - PLANE_EPS) * u[:, :, None] * u[:, None, :]
        if method == 4:
            A = self.C + PLANE_EPS * np.eye(3)
            return np.linalg.norm(np.linalg.inv(A), axis=(1, 2))[:, None, None] * A
        s = np.maximum(w, 0.0)
        with np.errstate(invalid="ignore", divide="ignore"):
            v = s / s[:, 2:3] if method == 2 else s
        v = np.where(v < PLANE_EPS, PLANE_EPS, v)  # std::max(v, 1e-3): NaN stays NaN
        out = np.einsum("nac,nc,nbc->nab", U, v, U)
        if method == 2:
            out[self.zero] = np.nan
        return out.reshape(n, 3, 3)

    @property
    def zero(self):
        """Points whose raw covariance is exactly zero (k copies of one point, or k = 1)."""
        return ~self.C.reshape(len(self.C), 9).any(1)

    def check(self, got, method, solver=1.0):
        """got (n,3,3) -> (ratio (n,), kind (n,)): error / bound per point (<= 1 passes; NaN where both are NaN counts as 0,
        NaN on one side only as inf).  kind: 0 vector / Frobenius check, 1 PLANE subspace check, 2 PLANE eigenvalues only.

        NONE: max over entries of |got - C| / bound.
        PLANE: got = I - (1 - 1e-3) n n^T.  With E = C_PLANE eps lam3 + |dC|_F (solver + covariance error), Davis-Kahan gives
          sin(n, u1) <= E / (lam2 - lam1 - E); |nn^T - u1u1^T|_F = sqrt(2) sin.  Where that is vacuous (> VACUOUS) but
          E / (lam3 - lam2 - E) is not, n must lie in span(u1, u2): |n . u3| <= that, read off as |got u3 - u3| / (1 - 1e-3).  Every point: eigenvalues of got are
          (1e-3, 1, 1) within C_EIG eps.
        MIN_EIG: lam -> max(lam, 1e-3) is 1-Lipschitz, hence (Frobenius norm) |f(C^) - f(C)|_F <= |dC|_F, plus the solver's
          C_EIG eps max(lam3, 1e-3).
        NORMALIZED_MIN_EIG: the same on C / lam_max, whose perturbation is <= (1 + sqrt 3) |dC|_F / (lam3 - |dC|_F); NaN
          exactly where the raw covariance is zero (0 / 0 under std::max, as the reference's Eigen expression).
        FROBENIUS: A = C + 1e-3 I, out = |A^-1|_F A; |d out|_F / |out|_F <= (1 + kappa) sqrt 3 |dC|_F / (lam1 + 1e-3)
          + C_EIG eps kappa, kappa = (lam3 + 1e-3) / (lam1 + 1e-3).
        solver multiplies C_EIG and C_PLANE (ORACLE_SVD for the CPU oracle)."""
        got = np.asarray(got, np.float64)
        n = len(got)
        ref = self.reference(method)
        c_eig, c_plane = C_EIG * solver, C_PLANE * solver
        kind = np.zeros(n, np.int64)
        w = self.w
        lam3 = np.maximum(w[:, 2], 0.0)
        if method == 0:
            with np.errstate(invalid="ignore", divide="ignore"):
                r = np.abs(got - ref) / self.bound
            r = np.where(np.abs(got - ref) == 0, 0.0, r)
            return r.reshape(n, 9).max(1), kind
        diff = np.sqrt(((got - ref) ** 2).sum((1, 2)))
        if method == 1:
            return diff / (self.dF + c_eig * EPS64 * np.maximum(lam3, PLANE_EPS)), kind
        if method == 2:
            nan_g = np.isnan(got).any((1, 2))
            z = self.zero
            with np.errstate(invalid="ignore", divide="ignore"):
                b = (1.0 + math.sqrt(3.0)) * self.dF / (lam3 - self.dF) + c_eig * EPS64
                r = np.where(lam3 > self.dF, diff / b, np.inf)
            r = np.where(z, np.where(nan_g & np.isnan(got).all((1, 2)), 0.0, np.inf), np.where(nan_g, np.inf, r))
            return r, kind
        if method == 4:
            l1 = np.maximum(w[:, 0], 0.0) + PLANE_EPS
            kap = (lam3 + PLANE_EPS) / l1
            rel = (1.0 + kap) * math.sqrt(3.0) * self.dF / l1 + c_eig * EPS64 * kap
            return diff / (rel * np.sqrt((ref ** 2).sum((1, 2)))), kind
        assert method == 3
        E = c_plane * EPS64 * lam3 + self.dF
        g12, g23 = w[:, 1] - w[:, 0], w[:, 2] - w[:, 1]
        with np.errstate(divide="ignore", invalid="ignore"):
            vb = np.where(g12 > E, E / (g12 - E), np.inf)
            sb = np.where(g23 > E, E / (g23 - E), np.inf)
        ev = np.linalg.eigvalsh(got)
        ev_r = np.abs(ev - [PLANE_EPS, 1.0, 1.0]).max(1) / (c_eig * EPS64)
        wv = 1.0 - PLANE_EPS
        r_vec = diff / (math.sqrt(2.0) * wv * vb + c_eig * EPS64)
        # |got u3 - u3| = (1 - 1e-3) |n . u3|, linear in the entries of got (a quadratic form would put a sqrt(eps) floor
        # under |n . u3|)
        u3 = self.U[:, :, 2]
        nu3 = np.linalg.norm(np.einsum("nab,nb->na", got, u3) - u3, axis=1)
        r_sub = nu3 / (wv * sb + c_eig * EPS64)
        kind = np.where(vb <= VACUOUS, 0, np.where(sb <= VACUOUS, 1, 2))
        r = np.where(kind == 0, r_vec, np.where(kind == 1, r_sub, 0.0))
        return np.maximum(r, ev_r), kind


# ---------------------------------------------------------------------------------------------------------------------
# correspondences and the linearize pass (nano_gicp_impl.hpp:173-296)
def transform_query(T, pts):
    """trans.cast<float>() * p in fp32, ((r0 x + r1 y) + r2 z) + t, no contraction (nano_gicp_impl.hpp:178, 190)."""
    Tf = np.asarray(T, np.float64).astype(np.float32)
    p = np.asarray(pts, np.float32)[:, :3]
    out = np.empty((len(p), 3), np.float32)
    for r in range(3):
        out[:, r] = ((Tf[r, 0] * p[:, 0] + Tf[r, 1] * p[:, 1]) + Tf[r, 2] * p[:, 2]) + Tf[r, 3]
    return out


def nn1(tgt, q, tie="low"):
    """Exact fp32 1-NN of the rows of q in tgt, (d2, lower index) -> (idx, d2)."""
    t = np.ascontiguousarray(np.asarray(tgt)[:, :3], np.float32)
    q = np.ascontiguousarray(q, np.float32)
    idx = np.empty(len(q), np.int64)
    d2 = np.empty(len(q), np.float32)
    ar = np.arange(len(t), dtype=np.int64)
    step = max(1, (1 << 22) // len(t))
    for s in range(0, len(q), step):
        dd = d2_f32(q[s:s + step, None, :], t[None, :, :])
        j = np.argmin(_keys(dd, ar[None, :], tie), axis=1)
        idx[s:s + step] = j
        d2[s:s + step] = dd[np.arange(len(j)), j]
    return idx, d2


def correspondences(src, tgt, T, max_corr_dist, gate="lt"):
    """update_correspondences' search and gate (nano_gicp_impl.hpp:186-199): -> (corr, sqd).  gate='le' is the wrong variant."""
    idx, d2 = nn1(tgt, transform_query(T, src))
    thr2 = float(max_corr_dist) * float(max_corr_dist)
    ok = d2.astype(np.float64) < thr2 if gate == "lt" else d2.astype(np.float64) <= thr2
    return np.where(ok, idx, -1), d2


def _skew_J(ta):
    """J = [skew(T a) | -I] per point: (n, 3, 6)."""
    n = len(ta)
    J = np.zeros((n, 3, 6), ta.dtype)
    J[:, 0, 1], J[:, 0, 2] = -ta[:, 2], ta[:, 1]
    J[:, 1, 0], J[:, 1, 2] = ta[:, 2], -ta[:, 0]
    J[:, 2, 0], J[:, 2, 1] = -ta[:, 1], ta[:, 0]
    J[:, 0, 3] = J[:, 1, 4] = J[:, 2, 5] = -1
    return J


class Linearize:
    """NanoGICP::linearize (nano_gicp_impl.hpp:213-270) given the correspondences and both clouds' covariances (n,3,3).

    ``H`` (6,6), ``b`` (6,), ``err``: the sums over the points with corr >= 0, each term in long double (64-bit mantissa)
    and summed pairwise in long double; ``M`` (n,3,3) the Mahalanobis matrices, ``kappa`` (n,) cond(C_B + R C_A R^T).
    ``Hb``, ``bb``, ``errb``: per-entry bounds on an fp64 evaluation in the engine's order (see the comment in __init__).
    T_trial: evaluate e at another pose with these correspondences and M (compute_error, :272-296): only err / errb."""

    def __init__(self, src, tgt, cov_src, cov_tgt, T, corr, T_trial=None):
        assert np.finfo(np.longdouble).nmant >= 63, "long double is not the 80-bit x87 format here"
        LD = np.longdouble
        T = np.asarray(T, np.float64)
        sel = np.flatnonzero(corr >= 0)
        self.n = len(sel)
        R = T[:3, :3]
        CA = np.asarray(cov_src, np.float64).reshape(-1, 3, 3)[sel]
        CB = np.asarray(cov_tgt, np.float64).reshape(-1, 3, 3)[corr[sel]]
        RCR = CB + np.einsum("ab,nbc,dc->nad", R, CA, R)
        self.M = np.linalg.inv(RCR)
        sv = np.linalg.svd(RCR, compute_uv=False)
        self.kappa = sv[:, 0] / sv[:, 2]
        self.k12 = sv[:, 0] / sv[:, 1]
        Tt = T if T_trial is None else np.asarray(T_trial, np.float64)
        a = np.asarray(src, np.float32)[sel, :3].astype(np.float64)
        bp = np.asarray(tgt, np.float32)[corr[sel], :3].astype(np.float64)
        Rt, tt = Tt[:3, :3], Tt[:3, 3]
        ta = np.einsum("ab,nb->na", Rt.astype(LD), a.astype(LD)) + tt.astype(LD)
        e = bp.astype(LD) - ta
        M = self.M.astype(LD)
        Me = np.einsum("nab,nb->na", M, e)
        err_p = np.einsum("na,na->n", e, Me)
        self.err = float(err_p.sum())
        # Bounds, first order, per point (|.| entrywise):
        #   ta = R a + t: 3 products, 3 sums           |d ta| <= gamma_6 (|R||a| + |t|)
        #   e = b - ta                                 |d e|  <= |d ta| + u |e|
        #   M = inv(C_B + R C_A R^T)                   |d M|  <= C_INV eps kappa (s1/s2) |M|_F   (rcrt, cofactor inverse)
        #   x = J_r^T (M J_c) (3 + 3 products/sums)    |d x|  <= |dJ_r|^T|M||J_c| + |J_r|^T|M||dJ_c|
        #                                                        + |dM|_F (sum|J_r|)(sum|J_c|) + gamma_8 |J_r|^T|M||J_c|
        # The restatement's M (LU) errs by less; the device sums the terms over <= n points:
        #   bound = 2 sum_p |d x_p| + gamma_n sum_p |x_p|.
        dta = gamma(6) * (np.abs(a) @ np.abs(Rt).T + np.abs(tt))
        de = dta + U64 * np.abs(e.astype(np.float64))
        dM = C_INV * EPS64 * self.kappa * self.k12 * np.linalg.norm(self.M, axis=(1, 2))
        aM = np.abs(self.M)
        e64 = np.abs(e.astype(np.float64))
        aMe = np.einsum("nab,nb->na", aM, e64)
        d_err = 2 * de[:, None, :] @ aMe[:, :, None] + (dM * e64.sum(1) ** 2)[:, None, None] + gamma(8) * (e64 * aMe).sum(1)[:, None, None]
        gN = gamma(max(self.n, 1))
        self.errb = float(2 * d_err.sum() + gN * np.abs(err_p.astype(np.float64)).sum())
        if T_trial is not None:
            return
        J = _skew_J(ta)
        MJ = np.einsum("nab,nbc->nac", M, J)
        Hp = np.einsum("nar,nac->nrc", J, MJ)
        bp_ = np.einsum("nar,na->nr", J, Me)
        self.H = Hp.sum(0).astype(np.float64)
        self.b = bp_.sum(0).astype(np.float64)
        aJ = np.abs(J.astype(np.float64))
        dJ = np.abs(_skew_J(dta))
        dJ[:, :, 3:] = 0  # the -I block is exact
        JMJ = np.einsum("nar,nab,nbc->nrc", aJ, aM, aJ)
        dH = (np.einsum("nar,nab,nbc->nrc", dJ, aM, aJ) + np.einsum("nar,nab,nbc->nrc", aJ, aM, dJ)
              + dM[:, None, None] * aJ.sum(1)[:, :, None] * aJ.sum(1)[:, None, :] + gamma(8) * JMJ)
        db = (np.einsum("nar,na->nr", dJ, aMe) + np.einsum("nar,nab,nb->nr", aJ, aM, de)
              + dM[:, None] * aJ.sum(1) * e64.sum(1)[:, None] + gamma(8) * np.einsum("nar,na->nr", aJ, aMe))
        self.Hb = 2 * dH.sum(0) + gN * np.abs(Hp.astype(np.float64)).sum(0)
        self.bb = 2 * db.sum(0) + gN * np.abs(bp_.astype(np.float64)).sum(0)


# ---------------------------------------------------------------------------------------------------------------------
# edge scenes
def _exact(a):
    a = np.asarray(a, np.float64)
    f = a.astype(np.float32)
    assert np.array_equal(f.astype(np.float64), a), "coordinates not exactly representable"
    return f


def lattice():
    """A permuted 0.5 m cubic lattice (7^3) and a 0.5 x 0.75 m planar lattice (13 x 9): shells of exactly equal d2 that
    straddle rank k for every k tested, at boundary and interior points; random original indices decide the ties."""
    rng = np.random.default_rng(21)
    g = np.stack(np.meshgrid(np.arange(7), np.arange(7), np.arange(7), indexing="ij"), -1).reshape(-1, 3) * 0.5
    h = np.stack(np.meshgrid(np.arange(13) * 0.5, np.arange(9) * 0.75, [0.0], indexing="ij"), -1).reshape(-1, 3) + [20.0, 0, 0]
    p = np.concatenate([g, h])
    return _exact(p[rng.permutation(len(p))])


def duplicates():
    """Runs of exact copies, 2 to 40 long (shorter and longer than k), 3 m apart, plus a few singletons between."""
    rng = np.random.default_rng(22)
    runs = [2, 3, 5, 7, 8, 9, 14, 15, 16, 19, 20, 21, 31, 32, 33, 40]
    base = rng.normal(0, 0.3, (len(runs), 3)) + np.arange(len(runs))[:, None] * [3.0, 0, 0]
    pts = np.concatenate([np.repeat(base[i:i + 1], r, 0) for i, r in enumerate(runs)] + [base + [1.5, 0, 0]])
    return pts[rng.permutation(len(pts))].astype(np.float32)


def collinear():
    """A scan ring's worth of exactly collinear points: p0 + i d with p0, d exactly representable and the products exact."""
    i = np.arange(600)[:, None]
    return _exact(np.array([1.5, -2.0, 0.25]) + i * np.array([0.03125, 0.015625, -0.0078125]))


def thin_edges():
    """Near-collinear edges (cross-section 1e-4 to 3e-6 m over 0.1-0.3 m neighbourhoods): lam2 / lam3 from 1e-4 down to 1e-9,
    where the closed-form eigenvector errs most and the Jacobi fallback takes over."""
    rng = np.random.default_rng(23)
    out = []
    for j, s in enumerate((1e-4, 3e-5, 1e-5, 3e-6)):
        t = rng.uniform(-3, 3, 600)
        out.append(np.c_[t, 0.3 * t + rng.normal(0, s, 600), 2.0 + rng.normal(0, s, 600)] + [0, 5.0 * j, 0])
    return np.concatenate(out).astype(np.float32)


def tilted_plane():
    """Exactly coplanar points on z = 0.5 x - 0.25 y with x, y multiples of 1/8: every coordinate exactly representable."""
    rng = np.random.default_rng(24)
    xy = rng.integers(-80, 80, (1500, 2)) / 8.0
    xy = np.unique(xy, axis=0)
    return _exact(np.c_[xy, 0.5 * xy[:, 0] - 0.25 * xy[:, 1]])


def isotropic():
    """Octahedra (6 vertices + centre: isotropic for k = 7) and cubes (8 corners + centre: k = 9), 5 m apart."""
    o = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]]) * 0.25
    c = np.array([[0, 0, 0]] + [[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)]) * 0.25
    pts = [o + [5.0 * i, 0, 0] for i in range(6)] + [c + [5.0 * i, 10.0, 0] for i in range(6)]
    return _exact(np.concatenate(pts))


def millimetre():
    """Clusters of 40 points with a 1 mm spread, 2 m apart: every eigenvalue far below 1e-3 (MIN_EIG clamps all three)."""
    rng = np.random.default_rng(25)
    return np.concatenate([rng.normal(0, 1e-3, (40, 3)) + [2.0 * i, 0, 1] for i in range(30)]).astype(np.float32)


def mixed():
    """A noisy plane, a blob and a pole: the generic geometry that the far copies move."""
    rng = np.random.default_rng(26)
    floor = np.c_[rng.uniform(-3, 3, (1200, 2)), rng.normal(0, 0.01, 1200)]
    blob = rng.normal(0, 0.4, (400, 3)) + [0, 0, 1.5]
    t = rng.uniform(0, 2 * np.pi, 400)
    pole = np.c_[2 + 0.05 * np.cos(t), 2 + 0.05 * np.sin(t), rng.uniform(0, 2, 400)]
    return np.concatenate([floor, blob, pole])


def far(offset):
    return (mixed() + np.asarray(offset, np.float64)).astype(np.float32)


def scenes():
    """name -> float32 (n, 3) cloud."""
    return {"lattice": lattice(), "duplicates": duplicates(), "collinear": collinear(), "thin_edges": thin_edges(),
            "tilted_plane": tilted_plane(), "isotropic": isotropic(), "millimetre": millimetre(),
            "near": far([0.0, 0.0, 0.0]), "far1km": far([1000.0, 0.0, 0.0]), "far3km": far([0.0, -3000.0, 40.0])}


def tiny(k, seed=27):
    """Clouds of n = 1 .. k + 1 points (all of a cloud is every point's neighbour set while n <= k)."""
    rng = np.random.default_rng(seed + k)
    return [(rng.normal(0, 1.0, (n, 3)) + [3.0, -1.0, 0.5]).astype(np.float32) for n in range(1, k + 2)]


# ---------------------------------------------------------------------------------------------------------------------
# crafted covariances for the linearize pass
def crafted_covariances(n, kappa_max, seed, basis=None):
    """n random SPD matrices Q diag(s) Q^T with condition numbers log-uniform in [1, kappa_max] and scale 1e-4..1.  With a
    shared basis (3x3 orthogonal) the source's and the target's small directions coincide and C_B + R C_A R^T keeps the
    condition number (at R = I)."""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.normal(size=(n, 3, 3)))
    if basis is not None:
        Q = np.broadcast_to(basis, (n, 3, 3))
    lk = rng.uniform(0, math.log(kappa_max), n)
    s = np.stack([np.ones(n), np.exp(-lk * rng.uniform(0, 1, n)), np.exp(-lk)], 1) * np.exp(rng.uniform(math.log(1e-4), 0, n))[:, None]
    C = np.einsum("nab,nb,ncb->nac", Q, s, Q)
    return 0.5 * (C + np.swapaxes(C, 1, 2))


def lattice_pair(offset=(0.0, 0.0, 0.0)):
    """Target: a permuted unit lattice (10 x 10 x 4).  Source: lattice points moved by exactly representable offsets, so
    that the fp32 d2 to the nearest target points is exact: 0.0625 (one nearest), 0.25 (two nearest tied, exactly at a
    0.5 m gate), 0.5 (four tied) and 0.75 (eight tied).  -> (src, tgt, kinds) with kinds the intended d2 per source point."""
    rng = np.random.default_rng(28)
    g = np.stack(np.meshgrid(np.arange(10), np.arange(10), np.arange(4), indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    tgt = g[rng.permutation(len(g))]
    inner = g[(g[:, 0] < 9) & (g[:, 1] < 9) & (g[:, 2] < 3)]
    moves = np.array([[0.25, 0, 0], [0.5, 0, 0], [0.5, 0.5, 0], [0.5, 0.5, 0.5], [0, 0.25, 0.0]])
    want = np.array([0.0625, 0.25, 0.5, 0.75, 0.0625])
    pick = rng.integers(0, len(moves), len(inner))
    src = inner + moves[pick]
    off = np.asarray(offset, np.float64)
    return _exact(src + off), _exact(tgt + off), want[pick]
