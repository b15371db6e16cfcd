"""tests/lm_ref.py, the exact restatement of the LM controller, checked on the CPU: its solve against numpy / scipy from
kappa 1 to 1e12, its crafted cases reaching the edges they claim, its bounds and rules tight enough to refuse the wrong
variants, and tests/lm_trials.py and the oracle following the same rules."""
import math

import numpy as np
import pytest
import scipy.linalg

import lm_ref
import lm_trials

KAPPAS = [1.0, 1e2, 1e4, 1e6, 1e8, 1e10, 1e12]
# eps values where (1 / eps) * eps and eps / eps round differently (the first three) and the deployment's / facade's own
BOUNDARY_EPS = [1e-5, 1e-9, 0.022460905827680535]
SAFE_EPS = [0.01, 2e-3, 5e-4, 1e-3, 1e-6, 1e-8, 0.1]


class Prm:
    def __init__(self, **kv):
        self.max_iterations, self.lm_max_iterations = 32, 10
        self.transformation_eps, self.rotation_eps, self.lm_init_lambda_factor = 0.01, 2e-3, 1e-9
        self.__dict__.update(kv)


def _fl(d):
    return np.array([float(x) for x in d])


@pytest.mark.parametrize("kappa", KAPPAS)
def test_exact_solve_against_numpy_and_scipy(kappa):
    rng = np.random.default_rng(int(np.log10(kappa)) + 7)
    for _ in range(4):
        H = lm_ref.spd(rng, kappa)
        b = rng.normal(size=6) * 1e3
        for lam in (0.0, 1e-9 * np.abs(np.diag(H)).max()):
            A = lm_ref.shifted(H, lam)
            d = _fl(lm_ref.solve_exact(H, b, lam))
            cond = np.linalg.cond(A)
            for other in (np.linalg.solve(A, -b), scipy.linalg.solve(A, -b, assume_a="pos")):
                assert np.abs(other - d).max() <= 1e-14 * cond * np.abs(d).max() + 1e-300
            # the exact solution satisfies its system exactly (checked in fractions)
            Af = lm_ref._frac(A)
            dx = lm_ref.solve_exact(H, b, lam)
            for i in range(6):
                assert sum(Af[i][j] * dx[j] for j in range(6)) == -lm_ref.Fraction(float(b[i]))


@pytest.mark.parametrize("kappa", KAPPAS)
def test_solve6_replay_within_bound(kappa):
    rng = np.random.default_rng(100 + int(np.log10(kappa)))
    for _ in range(6):
        H = lm_ref.spd(rng, kappa)
        b = rng.normal(size=6) * 1e3
        lam = 1e-9 * np.abs(np.diag(H)).max()
        d_hat = lm_ref.solve6_emul(H, b, lam)
        bound = lm_ref.solve_bound(H, b, lam, d_hat)
        err = np.abs(d_hat - _fl(lm_ref.solve_exact(H, b, lam)))
        assert np.isfinite(bound).all() and (err <= bound).all(), (err, bound)


def test_wrong_solve_fails_the_bound():
    """lambda added twice to one diagonal entry: outside the bound on every kappa >= 1e8 case."""
    rng = np.random.default_rng(5)
    for kappa in (1e8, 1e10, 1e12):
        for _ in range(4):
            H = lm_ref.spd(rng, kappa)
            b = rng.normal(size=6) * 1e3
            lam = 1e-9 * np.abs(np.diag(H)).max()
            d = _fl(lm_ref.solve_exact(H, b, lam))
            j = int(np.argmax(np.abs(d)))
            bad = lm_ref.solve6_emul(H, b, lam, double_shift=j)
            assert (np.abs(bad - d) > lm_ref.solve_bound(H, b, lam, bad)).any(), kappa


def test_rank_deficient_and_zero():
    rng = np.random.default_rng(9)
    for rank in (3, 4, 5):
        H = lm_ref.spd(rng, 1e3, rank=rank)
        b = rng.normal(size=6)
        lam = 1e-9 * np.abs(np.diag(H)).max()
        d_hat = lm_ref.solve6_emul(H, b, lam)
        assert (np.abs(d_hat - _fl(lm_ref.solve_exact(H, b, lam))) <= lm_ref.solve_bound(H, b, lam, d_hat)).all()
    # the all-zero H with lambda = 0: singular, no exact solution; solve6's zero-pivot guard gives d = 0
    assert lm_ref.solve_exact(np.zeros((6, 6)), np.zeros(6), 0.0) is None
    assert not np.any(lm_ref.solve6_emul(np.zeros((6, 6)), np.zeros(6), 0.0))
    assert np.isinf(lm_ref.solve_bound(np.zeros((6, 6)), np.zeros(6), 0.0, np.zeros(6))).all()


def _theta_sq_at(target):
    """w = (w0, w1, 0) whose fp64 theta^2 is exactly target."""
    w0 = math.sqrt(target)
    while w0 * w0 > target:
        w0 = np.nextafter(w0, 0)
    rem = target - w0 * w0
    if rem == 0:
        return np.array([w0, 0.0, 0.0])
    w1 = math.sqrt(rem)
    for k in range(-64, 65):
        w = np.array([w0, w1 * (1 + k * 2.0 ** -52), 0.0])
        if lm_ref.theta_sq(w) == target:
            return w
    raise AssertionError("no w with theta^2 == %r" % target)


def test_so3_exp_edges():
    T = 1e-10
    for target, small in ((np.nextafter(T, 0), True), (T, False), (np.nextafter(T, 1), False)):
        w = _theta_sq_at(target)
        assert lm_ref.theta_sq(w) == target
        R = lm_ref.so3_exp_ref(w)
        assert np.abs(lm_trials.so3_exp(w) - R.astype(np.float64)).max() <= lm_ref.so3_bound(w)
        # both branches agree far below the bound at the switch
        th = math.sqrt(target)
        assert abs(float(np.cos(np.longdouble(th) / 2)) - (1 - target / 8 + target * target / 384)) < 1e-25
        assert (lm_ref.theta_sq(w) < 1e-10) == small
    rng = np.random.default_rng(3)
    for mag in (1e-9, 1e-6, 1e-3, 0.1, 1.0, 3.0, 10.0, 100.0, 1e3):
        for _ in range(20):
            w = rng.normal(size=3)
            w *= mag / np.linalg.norm(w)
            err = np.abs(lm_trials.so3_exp(w) - lm_ref.so3_exp_ref(w).astype(np.float64)).max()
            assert err <= lm_ref.so3_bound(w), (mag, err)


def _device_rho(y0, yi, d, lam, b):
    """lm_update's fp64 evaluation of rho (no FMA)."""
    den = 0.0
    for i in range(6):
        den += d[i] * (lam * d[i] - b[i])
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.float64(y0 - yi) / np.float64(den)


def _case(**kv):
    c = dict(params=Prm(), nu=2.0, inner_it=0, outer_it=0, **{"lambda": 1e-3})
    c.update(kv)
    return c


def test_rho_edges_and_decisions():
    I3, t0 = np.eye(3), np.array([1.0, 0, 0])  # a delta far from converged
    b = np.array([1.0, -2, 3, 0.5, 0, 1])
    d = np.array([0.1, 0.2, -0.1, 0.3, 0.0, 0.2])
    lam = 1e-3
    cases = {"+0": (5.0, 5.0, d, b), "-0": (5.0, 5.0, d, -1e6 * b), "+inf": (5.0, 4.0, np.zeros(6), b),
             "-inf": (4.0, 5.0, np.zeros(6), b), "nan": (5.0, 5.0, np.zeros(6), b)}
    want = {"+0": (0.0, False), "-0": (0.0, True), "+inf": (np.inf, False), "-inf": (-np.inf, True)}
    for name, (y0, yi, dd, bb) in cases.items():
        rho = _device_rho(y0, yi, dd, lam, bb)
        if name == "nan":
            assert np.isnan(rho)
        else:
            assert rho == want[name][0] and np.signbit(rho) == want[name][1], name
        exact, err = lm_ref.rho_ref(y0, yi, dd, lam, bb)
        assert (name in ("+0", "-0")) == (exact == 0)
        got = lm_ref.decide(_case(), rho, I3, t0)
        assert got["decision"] == (0 if name == "-inf" else 1), name
    # an ordinary rho within its bound
    rng = np.random.default_rng(1)
    for _ in range(50):
        dd, bb = rng.normal(size=6), rng.normal(size=6)
        y0, yi = abs(rng.normal()) * 10, abs(rng.normal()) * 10
        exact, err = lm_ref.rho_ref(y0, yi, dd, lam, bb)
        assert abs(float(exact) - _device_rho(y0, yi, dd, lam, bb)) <= err


def test_lambda_rule_across_one_third():
    """1 - x^3 crosses 1/3 at x^3 = 2/3: the device's x*x*x form stays within LAMBDA_ULPS of pow on both sides."""
    x0 = (2.0 / 3.0) ** (1.0 / 3.0)
    rho0 = (x0 + 1) / 2
    lam = 0.7
    sides = set()
    for k in range(-3000, 3001, 7):
        rho = rho0 + k * 2.0 ** -52
        x = 2 * rho - 1
        dev = lam * max(1.0 / 3.0, 1 - x * x * x)
        ref = lm_ref.lambda_accept(lam, rho)
        assert abs(dev - ref) <= lm_ref.LAMBDA_ULPS * np.spacing(ref)
        sides.add(ref == lam * (1.0 / 3.0))
    assert sides == {True, False}
    for rho in (0.0, -0.0, 0.25, 0.5, 1.0, 7.0, 1e300, np.inf, np.nan):
        x = np.float64(2 * rho - 1)
        with np.errstate(over="ignore", invalid="ignore"):
            dev = lam * max(1.0 / 3.0, float(1 - x * x * x))
        assert abs(dev - lm_ref.lambda_accept(lam, rho)) <= lm_ref.LAMBDA_ULPS * np.spacing(dev), rho


@pytest.mark.parametrize("eps", BOUNDARY_EPS)
def test_eps_boundary_reciprocal_form(eps):
    """|t| = eps exactly: the reference's (1.0 / eps) * |t| is just below 1 (converged), |t| / eps is 1 (not)."""
    assert (1.0 / eps) * eps < 1.0 and eps / eps == 1.0
    dt = np.array([0.0, eps, 0.0])
    dR = np.eye(3)
    assert lm_ref.is_converged(dR, dt, 1.0, eps)
    assert not lm_ref.is_converged_legacy(dR, dt, 1.0, eps)
    D = np.eye(4)
    D[:3, 3] = dt
    assert lm_trials.is_converged(D, 1.0, eps)
    # rotation block, same eps
    dR2 = np.eye(3)
    dR2[0, 1] = eps
    assert lm_ref.is_converged(dR2, np.zeros(3), eps, 1.0) and not lm_ref.is_converged_legacy(dR2, np.zeros(3), eps, 1.0)
    # a rejected trial with that delta ends the solve converged (2) under the reference's form, not under the former one
    c = _case(params=Prm(transformation_eps=eps, rotation_eps=1.0))
    assert lm_ref.decide(c, -1.0, dR, dt)["decision"] == 2
    assert lm_ref.decide_legacy(c, -1.0, dR, dt)["decision"] == 0


@pytest.mark.parametrize("eps", SAFE_EPS)
def test_default_eps_never_reach_the_boundary(eps):
    """Within 2e5 ulp of eps, both forms give the same answer for the deployment's and the facade's epsilons."""
    k = np.arange(-200000, 200001, dtype=np.float64)
    x = eps + k * np.spacing(eps)
    assert np.array_equal((1.0 / eps) * x < 1, x / eps < 1)


def test_nan_step_is_not_converged():
    nanR, nant = np.full((3, 3), np.nan), np.full(3, np.nan)
    for dR, dt in ((nanR, nant), (np.eye(3), np.array([np.nan, 0, 0])), (nanR, np.zeros(3))):
        assert not lm_ref.is_converged(dR, dt, 2e-3, 0.01)
        D = np.eye(4)
        D[:3, :3], D[:3, 3] = dR, dt
        assert not lm_trials.is_converged(D, 2e-3, 0.01)
    assert lm_ref.is_converged_legacy(nanR, nant, 2e-3, 0.01)
    # rho = NaN accepts; the all-NaN step then does not end the solve
    got = lm_ref.decide(_case(), float("nan"), nanR, nant)
    assert got["decision"] == 1 and not got["converged"] and got["outer_it"] == 1
    assert lm_ref.decide_legacy(_case(), float("nan"), nanR, nant)["converged"] == 1
    # a NaN on the diagonal of H makes the initial lambda NaN
    H = np.eye(6)
    H[2, 2] = np.nan
    assert math.isnan(lm_ref.init_lambda(H, 1e-9)) and lm_ref.start_legacy(_case(H=H, **{"lambda": -1.0}))["lambda"] == 1e-9


def test_caps():
    c = _case(params=Prm(lm_max_iterations=0), H=np.eye(6), **{"lambda": -1.0})
    assert lm_ref.start(c) == dict(nu=2.0, trial=False, lm_failed=1, **{"lambda": 1e-9})
    assert lm_ref.start_legacy(c)["trial"]
    far = (np.eye(3), np.array([1.0, 0, 0]))
    one = _case(params=Prm(lm_max_iterations=1))
    got = lm_ref.decide(one, -1.0, *far)
    assert (got["decision"], got["lm_failed"], got["lambda"], got["nu"]) == (3, 1, 2e-3, 4.0)
    got = lm_ref.decide(_case(inner_it=8, nu=512.0), -1.0, *far)
    assert (got["decision"], got["inner_it"], got["nu"]) == (0, 9, 1024.0) and got["lambda"] == 512.0 * 1e-3
    assert lm_ref.decide(_case(inner_it=9), -1.0, *far)["decision"] == 3
    got = lm_ref.decide(_case(outer_it=31), 0.5, *far)
    assert got["decision"] == 1 and got["done"] and not got["converged"]


def test_oracle_follows_the_rules(oracle):
    src, dst = lm_ref.cluster_pair()
    prm = oracle.GicpParams.default()
    prm.lm_max_iterations = 0
    g = np.eye(4)
    g[0, 3] = 0.3
    o = oracle.gicp_align(src, dst, params=prm, guess=g)
    assert (o["converged"], o["iterations"], o["n_linearize"], o["n_error"], o["lm_failed"]) == (False, 0, 1, 0, True)
    assert np.array_equal(o["T"], g)
    # NONE with identical-point clusters: H is NaN from the first linearize, so lambda is NaN and no step converges
    prm = oracle.GicpParams.default()
    prm.regularization = 0
    prm.max_iterations = 6
    o = oracle.gicp_align(src, dst, params=prm)
    assert (o["converged"], o["iterations"], o["n_linearize"], o["n_error"], o["lm_failed"]) == (False, 5, 6, 6, False)
    assert np.isnan(o["T"][:3]).all()
