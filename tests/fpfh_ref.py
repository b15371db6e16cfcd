"""An fp64 restatement of the Quatro feature stage (normals, SPFH, FPFH), numpy / scipy only.

It states what k_normals, k_spfh and k_fpfh (fast-lio-sam-qn_b200/csrc/quatro.cu) compute, and how far a fp32
implementation may lie from it, so that the kernels (and the CPU oracle) can be checked against a bound derived from
the arithmetic instead of against each other:

* neighbour sets are exact: the fp32 rule ``((dx*dx) + dy*dy) + dz*dz < r2`` with ``d = query - point``, strict, self and
  exact duplicates included;
* normals come from a two-pass fp64 covariance and ``np.linalg.eigh``, with the per-point eigenvalues for bounds;
* the SPFH is kept as exact integer bin counts; the f1 (atan2) bin of a pair is *ambiguous* when its bin value lies within
  ``AMBIG`` of an interior integer (f2, f3 and every other operation are IEEE fp32 and bit-identical);
* the FPFH is fp64, with a per-bin rigorous bound for the kernel's fp32 order of operations (``Fpfh``) and for the oracle's
  (``oracle_m``).
"""
import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from scipy import sparse
from scipy.spatial import cKDTree

U32 = 2.0 ** -24  # unit round-off of fp32
EPS64 = 2.0 ** -52
# f1 is the only pair feature whose fp32 value is implementation-defined: CUDA's atan2f is documented to 2 ulp, numpy's
# float32 arctan2 is a different implementation.  A few ulp of f1 (|f1| <= pi, ulp 2.4e-7) move the bin value
# 11 * ((f1 + pi) / 2pi) by < 2e-6, and the three fp32 roundings after atan2 by < 3 ulp of 11 (< 3e-6).  A bin value within
# AMBIG = 1e-5 of an interior integer 1..10 may therefore land in either adjacent bin; farther away it cannot.
AMBIG = 1e-5
F32_PI = np.float32(np.pi)
D_PI = np.float32(1.0) / (np.float32(2.0) * F32_PI)


def gamma(m):
    """gamma_m = m u / (1 - m u) for fp32 (Higham, Lemma 3.1): |prod (1 + d_i)^(+-1) - 1| <= gamma_m for m factors."""
    mu = np.asarray(m, np.float64) * U32
    return mu / (1.0 - mu)


def kernel_r2(r):
    """The device's squared radius: (float)(r * r) from the double radius."""
    return np.float32(float(r) * float(r))


def oracle_r2(r):
    """The oracle's squared radius: the radius passes through float first, (float)((double)rf * (double)rf)."""
    rf = float(np.float32(r))
    return np.float32(rf * rf)


class CSR:
    """Neighbour sets of a list of queries: row q is indices[indptr[q]:indptr[q+1]], with their fp32 d2."""

    def __init__(self, queries, indptr, indices, d2):
        self.queries, self.indptr, self.indices, self.d2 = queries, indptr, indices, d2

    @property
    def counts(self):
        return np.diff(self.indptr)

    def rows(self):
        return np.repeat(np.arange(len(self.queries)), self.counts)

    def take(self, sel):
        """The rows sel (positions into queries), whole: subsampling what is checked never cuts a neighbour set."""
        sel = np.asarray(sel, np.int64)
        c = self.counts[sel]
        src = np.repeat(self.indptr[sel], c) + (np.arange(int(c.sum())) - np.repeat(np.cumsum(c) - c, c))
        return CSR(self.queries[sel], np.concatenate([[0], np.cumsum(c)]), self.indices[src], self.d2[src])


def radius_csr(xyz, r2, queries=None, tree=None, chunk=8192):
    """Exact fp32 radius neighbour sets.  Candidates from a kd-tree on a slightly enlarged radius (the fp32 d2 of a pair is
    within 4 u of its exact value, so 1e-5 relative is ample), then the kernel's own fp32 rule decides."""
    xyz = np.ascontiguousarray(xyz[:, :3], np.float32)
    queries = np.arange(len(xyz)) if queries is None else np.asarray(queries, np.int64)
    x64 = xyz.astype(np.float64)
    tree = tree or cKDTree(x64)
    r2 = np.float32(r2)
    rr = math.sqrt(float(r2)) * (1.0 + 1e-5)
    indptr = [np.zeros(1, np.int64)]
    idx, dd = [], []
    base = 0
    for s in range(0, len(queries), chunk):
        qi = queries[s:s + chunk]
        kmax = max(int(tree.query_ball_point(x64[qi], rr, return_length=True, workers=-1).max()), 1)
        _, cand = tree.query(x64[qi], k=[kmax] if kmax == 1 else kmax, distance_upper_bound=rr, workers=-1)
        cand = cand.reshape(len(qi), kmax)
        rows = np.broadcast_to(np.arange(len(qi))[:, None], cand.shape)
        m = cand < len(xyz)
        cand, rows = cand[m], rows[m]  # row-major: grouped by query
        q, p = xyz[qi[rows]], xyz[cand]
        dx, dy, dz = q[:, 0] - p[:, 0], q[:, 1] - p[:, 1], q[:, 2] - p[:, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        keep = d2 < r2
        idx.append(cand[keep].astype(np.int32))
        dd.append(d2[keep])
        indptr.append(base + np.cumsum(np.bincount(rows[keep], minlength=len(qi))))
        base += int(keep.sum())
    return CSR(queries, np.concatenate(indptr), np.concatenate(idx), np.concatenate(dd))


def normals(xyz, csr):
    """pcl::NormalEstimation restated in fp64 for the rows of csr (the normal-radius sets).
    -> (nrm float32 (q,3) NaN where < 3 neighbours, lam (q,3) ascending eigenvalues, dot (q,) fp64 value of the flip test
    -p . n on the float normal after the flip, err (q,) a bound on the fp32 rounding of that flip expression)."""
    xyz = np.ascontiguousarray(xyz[:, :3], np.float32)
    nq = len(csr.queries)
    cnt = csr.counts
    nrm = np.full((nq, 3), np.nan, np.float32)
    lam = np.full((nq, 3), np.nan)
    dot = np.full(nq, np.nan)
    err = np.full(nq, np.nan)
    ok = cnt >= 3
    rows = csr.rows()
    # coordinates relative to the query point: exact in fp64, and free of the cancellation of a far origin
    x = xyz[csr.indices].astype(np.float64) - xyz[csr.queries[rows]].astype(np.float64)
    m = np.stack([np.bincount(rows, x[:, a], nq) for a in range(3)], 1) / np.maximum(cnt, 1)[:, None]
    x -= m[rows]
    C = np.empty((nq, 3, 3))
    for a in range(3):
        for b in range(a, 3):
            C[:, a, b] = C[:, b, a] = np.bincount(rows, x[:, a] * x[:, b], nq) / np.maximum(cnt, 1)
    w, V = np.linalg.eigh(C[ok])
    n = V[:, :, 0].astype(np.float32)
    p = xyz[csr.queries[ok]]
    ct = ((np.float32(0) - p[:, 0]) * n[:, 0] + (np.float32(0) - p[:, 1]) * n[:, 1]) + (np.float32(0) - p[:, 2]) * n[:, 2]
    n = np.where((ct < 0)[:, None], -n, n)
    nrm[ok], lam[ok] = n, w
    dot[ok] = -(p.astype(np.float64) * n.astype(np.float64)).sum(1)
    # |fl(sum of 3 products) - exact| <= gamma_3 sum |p_i n_i|
    err[ok] = gamma(3) * (np.abs(p.astype(np.float64)) * np.abs(n.astype(np.float64))).sum(1)
    return nrm, lam, dot, err


def pair_features(p1, n1, p2, n2):
    """pcl::computePairFeatures in fp32, operation for operation as quatro.cu's pair_features.
    -> (valid, f1, f2, f3); valid is False where f4 == 0 or vn == 0."""
    d0, d1, d2 = p2[:, 0] - p1[:, 0], p2[:, 1] - p1[:, 1], p2[:, 2] - p1[:, 2]
    f4 = np.sqrt((d0 * d0 + d1 * d1) + d2 * d2)
    valid = f4 != 0
    f4 = np.where(valid, f4, np.float32(1))
    a0, a1, a2, b0, b1, b2 = n1[:, 0], n1[:, 1], n1[:, 2], n2[:, 0], n2[:, 1], n2[:, 2]
    angle1 = ((a0 * d0 + a1 * d1) + a2 * d2) / f4
    angle2 = ((b0 * d0 + b1 * d1) + b2 * d2) / f4
    sw = np.abs(angle1) < np.abs(angle2)
    a0, b0 = np.where(sw, b0, a0), np.where(sw, a0, b0)
    a1, b1 = np.where(sw, b1, a1), np.where(sw, a1, b1)
    a2, b2 = np.where(sw, b2, a2), np.where(sw, a2, b2)
    d0, d1, d2 = np.where(sw, -d0, d0), np.where(sw, -d1, d1), np.where(sw, -d2, d2)
    f3 = np.where(sw, -angle2, angle1)
    v0, v1, v2 = d1 * a2 - d2 * a1, d2 * a0 - d0 * a2, d0 * a1 - d1 * a0
    vn = np.sqrt((v0 * v0 + v1 * v1) + v2 * v2)
    valid &= vn != 0
    vn = np.where(vn != 0, vn, np.float32(1))
    v0, v1, v2 = v0 / vn, v1 / vn, v2 / vn
    w0, w1, w2 = a1 * v2 - a2 * v1, a2 * v0 - a0 * v2, a0 * v1 - a1 * v0
    f2 = (v0 * b0 + v1 * b1) + v2 * b2
    f1 = np.arctan2((w0 * b0 + w1 * b1) + w2 * b2, (a0 * b0 + a1 * b1) + a2 * b2)
    return valid, f1, f2, f3


def _bin11(v):
    return np.clip(np.floor(v), 0, 10).astype(np.int64)


def spfh_counts(xyz, nrm, csr, chunk=1 << 21):
    """Exact SPFH bin counts of the rows of csr (the FPFH-radius sets) from the given float32 normals (NaN = none).
    -> (counts (q,33) int64, amb (q,10) int64, cnt (q,)) where amb[:, b] counts the pairs whose f1 bin may be b or b+1 (the
    reference puts them in the floor bin) and cnt counts every neighbour in the radius, self included: incr = 100/(cnt-1)."""
    xyz = np.ascontiguousarray(xyz[:, :3], np.float32)
    nrm = np.ascontiguousarray(nrm, np.float32)
    nq = len(csr.queries)
    has = ~np.isnan(nrm[:, 0])
    rows_all = csr.rows()

    def part(s):
        rows = rows_all[s:s + chunk]
        i, j = csr.queries[rows], csr.indices[s:s + chunk].astype(np.int64)
        keep = has[i] & has[j] & (i != j)
        rows, i, j = rows[keep], i[keep], j[keep]
        valid, f1, f2, f3 = pair_features(xyz[i], nrm[i], xyz[j], nrm[j])
        rows, f1, f2, f3 = rows[valid], f1[valid], f2[valid], f3[valid]
        v1 = np.float32(11.0) * ((f1 + F32_PI) * D_PI)
        b1 = _bin11(v1)
        b2 = 11 + _bin11(np.float32(11.0) * ((f2 + np.float32(1.0)) * np.float32(0.5)))
        b3 = 22 + _bin11(np.float32(11.0) * ((f3 + np.float32(1.0)) * np.float32(0.5)))
        c = sum(np.bincount(rows * 33 + b, minlength=nq * 33) for b in (b1, b2, b3))
        near = np.rint(v1).astype(np.int64)
        a = (np.abs(v1.astype(np.float64) - near) < AMBIG) & (near >= 1) & (near <= 10)
        return c, np.bincount(rows[a] * 10 + near[a] - 1, minlength=nq * 10)

    counts = np.zeros(nq * 33, np.int64)
    amb = np.zeros(nq * 10, np.int64)
    with ThreadPoolExecutor(min(8, os.cpu_count() or 1)) as ex:  # numpy's array loops run without the GIL
        for c, a in ex.map(part, range(0, len(rows_all), chunk)):
            counts += c
            amb += a
    return counts.reshape(nq, 33), amb.reshape(nq, 10), csr.counts.copy()


def amb_touch(amb):
    """(q,10) ambiguous boundaries -> (q,33): for every f1 bin, the number of ambiguous pairs that may enter or leave it."""
    t = np.zeros((len(amb), 33), np.int64)
    t[:, 0:10] += amb
    t[:, 1:11] += amb
    return t


class Fpfh:
    """Reference FPFH of the rows of csr (queries Q, FPFH radius) from the SPFH counts of every point of the cloud and the
    normals they came from.

    ``v`` (q,33): the exact FPFH (fp64) of the reference counts.  ``bound`` (q,33): the most a fp32 evaluation in the kernel's
    order may differ from ``v``; ``slack`` (q,33): the part of it that comes from ambiguous f1 bins (zero elsewhere).
    ``n`` (q,): the number of terms (neighbours with d2 != 0) of each sum."""

    def __init__(self, csr, counts, amb, cnt, nrm, m=None):
        N = len(counts)
        nz = (csr.d2 != 0) & ~np.isnan(nrm[csr.queries, 0])[csr.rows()]  # a point without a normal has no FPFH
        rows = csr.rows()[nz]
        cols = csr.indices[nz]
        w = 1.0 / csr.d2[nz].astype(np.float64)
        W = sparse.csr_matrix((w, (rows, cols)), shape=(len(csr.queries), N))
        incr = np.where(cnt >= 2, 100.0 / np.maximum(cnt - 1, 1), 0.0)
        H = np.asarray(W @ (counts * incr[:, None]))
        A = np.asarray(W @ (amb_touch(amb) * incr[:, None]))
        S = H.reshape(-1, 3, 11).sum(2)
        sc = np.where(S != 0, 100.0 / np.where(S != 0, S, 1.0), 0.0)
        scale = np.repeat(sc, 11, axis=1)
        self.v = H * scale
        self.slack = A * scale
        self.n = np.bincount(rows, minlength=len(csr.queries))
        # The kernel (k_spfh, k_fpfh), per bin k of one point with n terms, every quantity non-negative:
        #   incr = fl(100 / (cnt - 1))                  1 rounding   (cnt - 1 is exact in fp32)
        #   s_jk = fl(count * incr)                     1            (the count is an exact integer)
        #   w_j  = fl(1 / d2_j)                         1            (d2_j is the same fp32 value here and there)
        #   h_k  = fma(s_jk, w_j, h_k) over n terms     <= n         (term j is rounded by its own and every later fma)
        # so h_k = sum_j t_jk (1 + theta_jk) with |theta_jk| <= gamma_{n+3}; as all t_jk >= 0, h_k = h_k* (1 + theta), same bound.
        #   s_b  = ((h_0 + h_1) + ...) + h_10           <= 10 more   -> s_b = s_b* (1 + theta), |theta| <= gamma_{n+13}
        #   sc   = fl(100 / s_b)                        1
        #   v_k  = fl(h_k * sc)                         1
        # v_k = v_k* (1 + theta_m), m = (n + 3) + (n + 13) + 2 = 2n + 18 factors (1 + d)^(+-1): |v_k - v_k*| <= gamma_{2n+18} v_k*.
        # An ambiguous f1 pair of neighbour j moves incr_j w_j between two adjacent bins of block 0, 100/s_b * that in v; the
        # block sum does not change.  So |v_k - v_k*| <= gamma_m (v_k* + slack_k) + slack_k.
        # m: another order of operations (oracle_m) in place of 2n + 18.
        m = 2 * self.n + 18 if m is None else m
        self.gamma = gamma(m)
        self.bound = self.gamma[:, None] * (self.v + self.slack) + self.slack


def oracle_m(csr, cnt):
    """The oracle's fp32 order (oracle_quatro.cpp spfh + fpfh), per bin of point i with n terms, C = the largest cnt_j - 1 of
    its neighbours j (no SPFH bin of j holds more than C pairs):
      s_jk = incr + incr + ... in fp32, c_jk <= C copies      incr's rounding + c_jk - 1 additions: <= C
      v    = fl(s_jk * fl(1 / d2))                            2
      h_k += v over the n terms                               <= n
      sum_b += v for the 11 bins of every term                <= 11 n, on values carrying C + 2
      sc = fl(100 / sum_b); h_k * sc                          2
    m = (C + 2 + n) + (C + 2 + 11 n) + 2 = 2 C + 12 n + 6."""
    nz = csr.d2 != 0
    rows = csr.rows()[nz]
    C = np.zeros(len(csr.queries), np.int64)
    np.maximum.at(C, rows, np.maximum(cnt[csr.indices[nz]] - 1, 0))
    n = np.bincount(rows, minlength=len(csr.queries))
    return 2 * C + 12 * n + 6
