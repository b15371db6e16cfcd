"""An exact restatement of the device's Levenberg-Marquardt controller (csrc/gicp.cu: solve6, so3_exp_matrix,
lm_prepare_trial, lm_update, delta_converged) and of the reference rules it follows (step_lm and is_converged,
lsq_registration_impl.hpp:88-208), with bounds on what the device's fp64 evaluation may differ by.

The 6x6 algebra is done in fractions.Fraction (exact), the trigonometry in numpy longdouble.  The bounds are what lets a
test tell a faithful fp64 evaluation from a subtly wrong one:

  solve_bound   componentwise forward error of solve6's unpivoted LDL^T against the exact solution of its own system
  so3_bound     of so3_exp_matrix against so3_exp_ref
  rho_ref       the exact rho of the device's step, with the error of its fp64 evaluation

decide() applies the reference's accept / reject / converge rules as written; decide_legacy() and solve6_emul(...,
double_shift=j) are the deliberately wrong variants the CPU tests use to show the rules and bounds have teeth.
"""
import math
from fractions import Fraction

import numpy as np

U = 2.0 ** -53  # unit roundoff of fp64
N = 6


def gamma(k):
    return k * U / (1 - k * U)


# ---------------------------------------------------------------------------------------------------------------------
# the solve
def shifted(H, lam):
    """fl(H + lam I): the matrix solve6 factors (its diagonal shift is one fp64 add per entry)."""
    A = np.array(H, np.float64).reshape(6, 6).copy()
    for i in range(6):
        A[i, i] = A[i, i] + np.float64(lam)
    return A


def _frac(M):
    return [[Fraction(float(x)) for x in row] for row in np.asarray(M, np.float64).reshape(6, 6)]


def _gauss(A, rhs_cols):
    """Exact Gauss-Jordan on a list-of-lists Fraction matrix; None when singular."""
    n = len(A)
    M = [A[i][:] + [c[i] for c in rhs_cols] for i in range(n)]
    for k in range(n):
        p = next((i for i in range(k, n) if M[i][k] != 0), None)
        if p is None:
            return None
        M[k], M[p] = M[p], M[k]
        piv = M[k][k]
        M[k] = [x / piv for x in M[k]]
        for i in range(n):
            if i != k and M[i][k] != 0:
                f = M[i][k]
                M[i] = [x - f * y for x, y in zip(M[i], M[k])]
    return [[M[i][n + j] for i in range(n)] for j in range(len(rhs_cols))]


def solve_exact(H, b, lam):
    """The exact rational solution d of fl(H + lam I) d = -b (a list of 6 Fractions), None when that matrix is singular
    or not finite."""
    A = shifted(H, lam)
    if not (np.isfinite(A).all() and np.isfinite(b).all()):
        return None
    sol = _gauss(_frac(A), [[-Fraction(float(x)) for x in b]])
    return None if sol is None else sol[0]


def inverse_exact(A):
    """Exact inverse of a finite fp64 matrix (list of rows of Fractions), None when singular."""
    I = [[Fraction(int(i == j)) for i in range(6)] for j in range(6)]
    cols = _gauss(_frac(A), I)
    return None if cols is None else [[cols[j][i] for j in range(6)] for i in range(6)]


def solve6_emul(H, b, lam, double_shift=None):
    """solve6 replayed in fp64 (no FMA).  double_shift=j: the deliberately wrong variant that adds lam to diagonal entry j
    twice."""
    H = np.asarray(H, np.float64).reshape(6, 6)
    L = np.zeros((6, 6))
    D = np.zeros(6)
    for j in range(6):
        dj = H[j, j] + lam
        if j == double_shift:
            dj = dj + lam
        for k in range(j):
            dj -= L[j, k] * L[j, k] * D[k]
        D[j] = dj
        for i in range(j + 1, 6):
            v = H[i, j]
            for k in range(j):
                v -= L[i, k] * L[j, k] * D[k]
            L[i, j] = v / dj if dj != 0.0 else 0.0
    y = np.zeros(6)
    for i in range(6):
        s = -b[i]
        for k in range(i):
            s -= L[i, k] * y[k]
        y[i] = s
    y = np.array([y[i] / D[i] if D[i] != 0.0 else 0.0 for i in range(6)])
    x = np.zeros(6)
    for i in range(5, -1, -1):
        s = y[i]
        for k in range(i + 1, 6):
            s -= L[k, i] * x[k]
        x[i] = s
    return x


def solve_bound(H, b, lam, d_hat):
    """Componentwise bound on |d_hat - d| for the d_hat solve6 computes, d the exact solution of (H + lam I) d = -b -- of
    the matrix with the shift rounded (solve_exact) or not.  inf where no bound holds (A = fl(H + lam I) singular, not
    finite or not positive definite: solve6 is unpivoted and needs positive pivots).

    Derivation (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Lemma 8.4 / Thm 10.3 / §11.1), n = 6,
    A = fl(H + lam I), every operation of solve6 rounded once (an FMA the compiler contracts rounds fewer times, which only
    shrinks each theta below):
      factorization  d_j = a_jj - sum_{k<j} (l_jk * l_jk) * d_k   and   l_ij = (a_ij - sum_{k<j} (l_ik * l_jk) * d_k) / d_j.
                     solve6 recomputes each term as L*L*D with TWO multiplies (not l_ik * w_jk with w = D l stored), so a
                     term carries two roundings, the chain of at most n - 1 subtractions n - 1 more and the division one:
                     A + dA1 = L^ D^ L^T with |dA1| <= gamma_{n+2} |L^||D^||L^T|.
      substitutions  (L^ + dL1) y = -b, |dL1| <= gamma_{n-1} |L^|; (D^ + dD) z = y, |dD| <= u |D^|;
                     (L^T + dL2) x = z, |dL2| <= gamma_{n-1} |L^T|; the product of the three perturbed factors is
                     L^ D^ L^T + dE with |dE| <= gamma_{2n-1} |L^||D^||L^T|.
      together       (A + dA) d_hat = -b with |dA| <= (gamma_{n+2} + gamma_{2n-1}) |L^||D^||L^T| <= c gamma_{3n+1} |L^||D^||L^T|,
                     c = 1 for this formulation.
      |L^||D^||L^T|  with positive pivots (A positive definite) every row of L^ D^{1/2} has squared norm
                     sum_k l_ik^2 d_k <= a_ii / (1 - gamma_{n+2}) (the diagonal equation above, all terms positive), so by
                     Cauchy-Schwarz (|L^||D^||L^T|)_ij <= sqrt(a_ii a_jj) / (1 - gamma_{n+2}).
      the shift      fl(h_jj + lam) = (h_jj + lam)(1 + delta), |delta| <= u: a further u |a_jj| on the diagonal of dA when d
                     is the solution of the unrounded matrix.
      forward        A (d_hat - d) = -dA d_hat exactly, so |d_hat - d| <= |A^-1| |dA| |d_hat| with A^-1 exact (Fractions).
    The float evaluation of the final products is inflated by 1e-12 relative, far above its own rounding."""
    A = shifted(H, lam)
    d_hat = np.asarray(d_hat, np.float64)
    inf = np.full(6, np.inf)
    if not (np.isfinite(A).all() and np.isfinite(d_hat).all()):
        return inf
    Ai = inverse_exact(A)
    if Ai is None:
        return inf
    diag = np.diag(A)
    if (diag <= 0).any():
        return inf
    # positive definite <=> every exact pivot is positive (exact LDL^T of A)
    F = _frac(A)
    for j in range(6):
        if F[j][j] <= 0:
            return inf
        for i in range(j + 1, 6):
            f = F[i][j] / F[j][j]
            for k in range(j, 6):
                F[i][k] -= f * F[j][k]
    s = np.sqrt(diag)
    E = (gamma(3 * N + 1) / (1 - gamma(N + 2))) * np.outer(s, s) + np.diag(U * np.abs(diag))
    absAi = np.array([[abs(float(x)) for x in row] for row in Ai])
    return absAi @ (E @ np.abs(d_hat)) * (1 + 1e-12)


# ---------------------------------------------------------------------------------------------------------------------
# so3_exp
def theta_sq(w):
    """so3_exp_matrix's branch variable, w0*w0 + w1*w1 + w2*w2 in fp64 (left to right)."""
    w = np.asarray(w, np.float64)
    return (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]


def so3_exp_ref(w):
    """so3_exp (so3.hpp:99-118) and Quaternion::toRotationMatrix evaluated in longdouble, on the branch the fp64 theta^2
    selects (theta^2 < 1e-10: the quartic Taylor expansion the reference uses; the two branches agree to ~1e-30 there)."""
    small = theta_sq(w) < 1e-10
    w = np.asarray(w, np.float64).astype(np.longdouble)
    th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2]
    if small:
        imag = np.longdouble(0.5) - th2 / 48 + th2 * th2 / 3840
        real = np.longdouble(1) - th2 / 8 + th2 * th2 / 384
    else:
        th = np.sqrt(th2)
        imag, real = np.sin(th / 2) / th, np.cos(th / 2)
    qw, qx, qy, qz = real, imag * w[0], imag * w[1], imag * w[2]
    return np.array([[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qw * qz), 2 * (qx * qz + qw * qy)],
                     [2 * (qx * qy + qw * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qw * qx)],
                     [2 * (qx * qz - qw * qy), 2 * (qy * qz + qw * qx), 1 - 2 * (qx * qx + qy * qy)]], np.longdouble)


def so3_bound(w):
    """Bound on every entry of |so3_exp_matrix(w) - so3_exp_ref(w)|.  theta^2 carries gamma_3, sqrt one rounding more,
    CUDA's sin / cos at most 2 ulp (CUDA C Programming Guide, double-precision functions) plus the argument's error
    (<= theta u ... 2 theta u absolute), the division one rounding: every quaternion component (|q| = 1) is off by at most
    (8 + 2 theta) u; each matrix entry is 1 or a sum of two doubled products of components, (4 + 2) roundings more:
    (64 + 16 theta) u covers it with room.  The Taylor branch (theta < 1e-5) is a few roundings of numbers <= 1."""
    th = math.sqrt(max(float(theta_sq(w)), 0.0))
    return (64 + 16 * th) * U


# ---------------------------------------------------------------------------------------------------------------------
# rho
def rho_ref(y0, yi, d, lam, b):
    """-> (rho, err): rho = (y0 - yi) / d.(lam d - b) exact (a Fraction, or a float inf / nan where the exact denominator
    is 0) for the given fp64 inputs, and a bound err on |rho_hat - rho| for lm_update's fp64 evaluation (inf where the
    denominator's sign is not certain).  The numerator is one subtraction (u relative); the denominator six terms of a
    multiply, a subtract and a multiply, summed from 0 (gamma_9 of sum |d_i| (|lam d_i| + |b_i|)); the quotient one
    rounding more."""
    vals = [y0, yi, lam] + list(d) + list(b)
    if not all(math.isfinite(float(v)) for v in vals):
        return float("nan"), float("inf")
    num = Fraction(float(y0)) - Fraction(float(yi))
    L = Fraction(float(lam))
    den = sum(Fraction(float(di)) * (L * Fraction(float(di)) - Fraction(float(bi))) for di, bi in zip(d, b))
    S = sum(abs(float(di)) * (abs(float(lam) * float(di)) + abs(float(bi))) for di, bi in zip(d, b))
    Ed = gamma(9) * S * (1 + 1e-12)
    if den == 0:
        if num == 0:
            return float("nan"), float("inf")
        return (float("inf") if num > 0 else float("-inf")), float("inf")
    rho = num / den
    if abs(float(den)) <= Ed:
        return rho, float("inf")
    # |num_hat - num| <= u |num|; |den_hat - den| <= Ed; then one rounding of the quotient
    an, ad = abs(float(num)), abs(float(den))
    err = (an * (1 + U) / (ad - Ed) - an / ad) + U * an / ad + U * an * (1 + U) / (ad - Ed)
    return rho, err * (1 + 1e-9)


# ---------------------------------------------------------------------------------------------------------------------
# the rules
def is_converged(dR, dt, rotation_eps, transformation_eps):
    """is_converged (lsq_registration_impl.hpp:117-127) as written: max((1.0 / eps) * |x|) < 1 over R - I and t; the
    maximum of a block holding a NaN is NaN (the reference's maxCoeff of an all-NaN block is NaN; the engine extends that
    to any NaN), and NaN < 1 is false."""
    dR = np.asarray(dR, np.float64).reshape(3, 3)
    dt = np.asarray(dt, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        r = (1.0 / rotation_eps) * np.abs(dR - np.eye(3))
        t = (1.0 / transformation_eps) * np.abs(dt)
    if np.isnan(r).any() or np.isnan(t).any():
        return False
    return bool(max(r.max(), t.max()) < 1)


def init_lambda(H, factor):
    """lm_init_lambda_factor * |diag H|.maxCoeff() (:165-167); a NaN on the diagonal gives NaN."""
    dg = np.abs(np.diag(np.asarray(H, np.float64).reshape(6, 6)))
    return factor * (float("nan") if np.isnan(dg).any() else float(dg.max()))


def lambda_accept(lam, rho):
    """lm_lambda_ * max(1 / 3, 1 - pow(2 rho - 1, 3)) (:201), pow correctly rounded (the device computes x * x * x)."""
    with np.errstate(over="ignore", invalid="ignore"):
        x = 2 * np.float64(rho) - 1
        f = 1 - np.power(x, 3.0)
    f = float(f)
    return lam * (f if f > 1.0 / 3.0 else 1.0 / 3.0)  # std::max(1/3, f): 1/3 unless f > 1/3 (NaN gives 1/3)


# |lambda_device - lambda_accept| <= LAMBDA_ULPS ulp after an accept: x*x*x is two roundings where pow is one, 1 - x^3 is
# kept only when >= 1/3 (x^3 <= 2/3), so its error relative to the kept value is <= 3 * (3u * 2/3) = 6u, and the final
# product one more: 7u relative, at most 7 ulp (1 ulp >= u relative).  Rejections are bit-exact (nu * lambda, 2 * nu).
LAMBDA_ULPS = 8


def decide(case, rho, dR, dt, converged_fn=None):
    """The reference's decision for one trial (step_lm :176-205 and computeTransformation :101-111), as written:
    rho < 0 rejects (so +0, -0 and NaN accept); a rejection whose delta is_converged ends the solve converged (2); lambda
    *= nu, nu *= 2 after a rejection, and lm_max_iterations trials at most (3: "lm not converged!!"); an accept moves x0,
    lambda *= max(1/3, 1 - (2 rho - 1)^3) and the solve ends converged when is_converged(delta), or at max_iterations.
    case: lambda, nu, inner_it, outer_it, params (rotation_eps, transformation_eps, lm_max_iterations, max_iterations).
    -> dict(decision, lambda, nu, inner_it, outer_it, converged, lm_failed, done)"""
    p = case["params"]
    conv = converged_fn or is_converged
    lam, nu, inner, outer = case["lambda"], case.get("nu", 2.0), case.get("inner_it", 0), case.get("outer_it", 0)
    out = dict(converged=0, lm_failed=0, done=False)
    if rho < 0:
        if conv(dR, dt, p.rotation_eps, p.transformation_eps):
            return dict(out, decision=2, converged=1, done=True, **{"lambda": lam}, nu=nu, inner_it=inner, outer_it=outer)
        lam, nu, inner = nu * lam, 2 * nu, inner + 1
        if inner >= p.lm_max_iterations:
            return dict(out, decision=3, lm_failed=1, done=True, **{"lambda": lam}, nu=nu, inner_it=inner, outer_it=outer)
        return dict(out, decision=0, **{"lambda": lam}, nu=nu, inner_it=inner, outer_it=outer)
    lam = lambda_accept(lam, rho)
    if conv(dR, dt, p.rotation_eps, p.transformation_eps):
        return dict(out, decision=1, converged=1, done=True, **{"lambda": lam}, nu=nu, inner_it=inner, outer_it=outer)
    outer += 1
    return dict(out, decision=1, done=outer >= p.max_iterations, **{"lambda": lam}, nu=nu, inner_it=inner, outer_it=outer)


def start(case):
    """What step_lm does after linearize (:163-169): lambda init when lambda < 0, nu = 2, and a first trial only when
    lm_max_iterations > 0 (otherwise it returns false: lm_failed, not converged).  -> dict(lambda, nu, trial, lm_failed)"""
    p = case["params"]
    lam = case["lambda"]
    if lam < 0:
        lam = init_lambda(case["H"], p.lm_init_lambda_factor)
    trial = p.lm_max_iterations > 0
    return dict(nu=2.0, trial=trial, lm_failed=0 if trial else 1, **{"lambda": lam})


def is_converged_legacy(dR, dt, rotation_eps, transformation_eps):
    """The form the engine used before: |x| / eps, and fmax drops NaN."""
    dR = np.asarray(dR, np.float64).reshape(3, 3)
    m = 0.0
    with np.errstate(invalid="ignore"):
        for v in list((np.abs(dR - np.eye(3)) / rotation_eps).ravel()) + list(np.abs(np.asarray(dt, np.float64)) / transformation_eps):
            m = m if math.isnan(v) else max(m, float(v))
    return m < 1


def decide_legacy(case, rho, dR, dt):
    """decide() with the engine's former convergence test (division, NaN dropped): a deliberately wrong variant."""
    return decide(case, rho, dR, dt, converged_fn=is_converged_legacy)


def start_legacy(case):
    """start() as the engine had it: a trial even when lm_max_iterations <= 0, lambda init dropping NaN."""
    p = case["params"]
    lam = case["lambda"]
    if lam < 0:
        dg = np.abs(np.diag(np.asarray(case["H"], np.float64).reshape(6, 6)))
        lam = p.lm_init_lambda_factor * max([0.0] + [float(x) for x in dg if not math.isnan(x)])
    return dict(nu=2.0, trial=True, lm_failed=0, **{"lambda": lam})


# ---------------------------------------------------------------------------------------------------------------------
# cases
def spd(rng, kappa, rank=6, scale=1e4):
    """A symmetric positive (semi)definite 6x6 with eigenvalues log-spaced from scale down to scale / kappa (the last
    6 - rank exactly 0 before rounding)."""
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    ev = scale * np.logspace(0, -np.log10(kappa), 6)
    ev[rank:] = 0.0
    H = (Q * ev) @ Q.T
    return (H + H.T) / 2


def cluster_pair(n=4000, cluster=20, seed=0):
    """Random points in a 20 m box plus `cluster` copies of one point in both clouds: under regularization NONE their
    covariances are exactly 0, so C_t + R C_s R^T is singular and its inverse NaN."""
    rng = np.random.default_rng(seed)
    src = rng.uniform(-10, 10, (n, 3)).astype(np.float32)
    dst = (src + rng.normal(0, 0.02, src.shape)).astype(np.float32)
    c = np.array([[1.25, -2.5, 0.75]], np.float32)
    return np.vstack([src, np.repeat(c, cluster, 0)]), np.vstack([dst, np.repeat(c, cluster, 0)])
