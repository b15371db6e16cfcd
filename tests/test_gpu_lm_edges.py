"""The device LM controller (csrc/gicp.cu: solve6, so3_exp_matrix, lm_prepare_trial, lm_update, delta_converged) against
the exact restatement of tests/lm_ref.py, through b200reg_lm_step_tap (the product's own controller on crafted states),
through traced solves of degenerate scenes, and end to end against the oracle on the edges where the reference's rules
and a careless restatement of them part: |x| = eps, a NaN step, lm_max_iterations = 0."""
import math
from fractions import Fraction

import numpy as np
import pytest

import lm_ref

KAPPAS = [1.0, 1e2, 1e4, 1e6, 1e8, 1e10, 1e12]
BOUNDARY_EPS = [1e-5, 1e-9, 0.022460905827680535]
U = lm_ref.U


def _prm(**kv):
    import b200reg
    p = b200reg.default_params()
    for k, v in kv.items():
        setattr(p, k, v)
    return p


def _check_trial_prep(c, o):
    """The prepared trial of one tap output against the restatement: d within solve_bound of the exact solve, dR within
    so3_bound of so3_exp_ref(d), dt = d[3:], and the trial pose = dR x0 up to its own rounding.  -> |d - d_exact| / bound"""
    d = o["d"]
    ex = lm_ref.solve_exact(c["H"], c["b"], c["lambda"])
    ratio = 0.0
    if ex is not None:
        bound = lm_ref.solve_bound(c["H"], c["b"], c["lambda"], d)
        err = np.abs(d - np.array([float(x) for x in ex]))
        assert np.isfinite(bound).all() and (err <= bound).all(), (err, bound)
        ratio = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1), 0)))
    assert np.abs(o["dR"] - lm_ref.so3_exp_ref(d[:3]).astype(np.float64)).max() <= lm_ref.so3_bound(d[:3])
    assert np.array_equal(o["dt"], d[3:])
    R0, t0 = np.asarray(c.get("R", np.eye(3))), np.asarray(c.get("t", np.zeros(3)))
    dRl = o["dR"].astype(np.longdouble)
    Rt = dRl @ R0.astype(np.longdouble)
    tt = dRl @ t0.astype(np.longdouble) + o["dt"].astype(np.longdouble)
    assert np.abs(o["Rt"] - Rt.astype(np.float64)).max() <= 8 * U
    assert (np.abs(o["tt"] - tt.astype(np.float64)) <= 8 * U * (np.abs(t0).sum() + np.abs(o["dt"]) + 1e-300)).all()
    return ratio


def _solve_cases(seed=0):
    rng = np.random.default_rng(seed)
    cases = []
    for kappa in KAPPAS:
        for _ in range(3):
            H = lm_ref.spd(rng, kappa)
            b = rng.normal(size=6) * 1e3
            for lam in (1e-9 * np.abs(np.diag(H)).max(), 1e-3 * np.abs(np.diag(H)).max()):
                cases.append(dict(H=H, b=b, y0=10.0, yi=9.0, mode="trial", **{"lambda": lam}, kappa=kappa))
        H = lm_ref.spd(rng, kappa)  # lambda = 0: H itself, kappa as stated
        cases.append(dict(H=H, b=rng.normal(size=6), y0=10.0, yi=9.0, mode="trial", **{"lambda": 0.0}, kappa=kappa))
    for rank in (3, 4, 5):  # exactly rank-deficient, lambda > 0
        H = lm_ref.spd(rng, 1e3, rank=rank)
        cases.append(dict(H=H, b=rng.normal(size=6), y0=10.0, yi=9.0, mode="trial", **{"lambda": 1e-9 * np.abs(np.diag(H)).max()}, kappa=np.inf))
    # a step in a weak direction large enough for theta up to ~1e3 rad
    H = np.diag([1e-6, 1e4, 1e4, 1e4, 1e4, 1e4])
    cases.append(dict(H=H, b=np.array([-1e-3, 0, 0, 0, 0, 0]), y0=10.0, yi=9.0, mode="trial", **{"lambda": 0.0}, kappa=1e10))
    R0 = lm_ref.so3_exp_ref(np.array([0.3, -0.2, 0.1])).astype(np.float64)
    for c in cases[::4]:
        c["R"], c["t"] = R0, np.array([3.0, -4.0, 0.5])
    return cases


@pytest.mark.gpu
def test_tap_solves_within_bound(ctx):
    cases = _solve_cases()
    out = ctx.lm_step_tap(cases)
    worst = {}
    for c, o in zip(cases, out):
        assert o["has_trial"] == 1
        r = _check_trial_prep(c, o)
        worst[c["kappa"]] = max(worst.get(c["kappa"], 0.0), r)
    big = [c for c in cases if np.abs(np.array([float(x) for x in (lm_ref.solve_exact(c["H"], c["b"], c["lambda"]) or [0])])).max() > 100]
    assert big, "some case steps far into a weak direction"
    print("solve6 |d - d_exact| / bound, worst per kappa:", {k: "%.3g" % v for k, v in sorted(worst.items())})
    # the all-zero H with lambda = 0: the zero-pivot guard gives the zero step
    o = ctx.lm_step_tap([dict(H=np.zeros((6, 6)), b=np.zeros(6), y0=0.0, yi=0.0, mode="trial", **{"lambda": 0.0})])[0]
    assert not np.any(o["d"]) and np.array_equal(o["dR"], np.eye(3))


def _decision_cases():
    """(case, note) covering every decision path with certain answers: H = I and lambda = 0 make d = -b exactly, and
    dR = I exactly when the rotation part of b is 0."""
    I6 = np.eye(6)
    far = np.array([0.0, 0.0, 0.0, -1.0, 0.0, 0.0])  # d = (0, 0, 0, 1, 0, 0): not converged
    near = np.array([0.0, 0.0, 0.0, -1e-4, 0.0, 0.0])  # converged under the defaults
    rot = np.array([-0.05, 0.02, 0.0, -0.2, 0.1, 0.0])
    out = []
    add = lambda note, **kv: out.append((dict(dict(H=I6, b=far, y0=10.0, yi=9.0, mode="trial", nu=2.0, **{"lambda": 0.0}), **kv), note))
    add("accept", yi=9.0)
    add("accept converged", b=near, yi=9.0)
    add("accept at max_iterations", outer_it=31, yi=9.0)
    add("reject", yi=11.0, **{"lambda": 0.5})
    add("reject converged", b=near, yi=11.0, **{"lambda": 0.5})
    add("reject, last trial", yi=11.0, inner_it=9, nu=512.0, **{"lambda": 0.5})
    add("reject, lm_max_iterations 1", yi=11.0, params=_prm(lm_max_iterations=1))
    add("rho +0", yi=10.0)
    add("rho -0", yi=10.0, H=-I6)  # an indefinite system: d.(lam d - b) < 0 and y0 - yi = +0
    add("rotation step", b=rot, yi=9.5, **{"lambda": 1e-3})
    add("rotation step rejected", b=rot, yi=10.5, **{"lambda": 1e-3})
    for eps in BOUNDARY_EPS:
        b = np.array([0.0, 0.0, 0.0, 0.0, -eps, 0.0])
        p = _prm(transformation_eps=eps, rotation_eps=1.0)
        add("eps boundary accept", b=b, yi=9.0, params=p)
        add("eps boundary reject", b=b, yi=11.0, params=p)
    nanH = np.full((6, 6), np.nan)
    infH = I6.copy()
    infH[0, 0] = np.inf
    add("NaN H", H=nanH, yi=np.nan, **{"lambda": 1e-3})
    add("NaN b", b=np.full(6, np.nan), yi=9.0)
    add("NaN yi", yi=np.nan)
    add("NaN yi, converged step", b=near, yi=np.nan)
    add("inf H", H=infH, yi=9.0)
    add("inf b", b=np.array([0, 0, 0, -np.inf, 0, 0.0]), yi=9.0)
    add("inf yi", yi=np.inf)
    add("-inf yi", yi=-np.inf)
    return out


def _expect(c, o):
    """decide() on the device's own step and rho."""
    rec = o["record"]
    return lm_ref.decide(dict(c, params=c.get("params") or _prm()), float(rec["rho"]), o["dR"], o["dt"])


@pytest.mark.gpu
def test_tap_decisions_follow_the_reference_rules(ctx):
    cases = _decision_cases()
    out = ctx.lm_step_tap([c for c, _ in cases])
    seen = set()
    for (c, note), o in zip(cases, out):
        rec = o["record"]
        want = _expect(c, o)
        assert rec["decision"] == want["decision"], note
        assert (o["converged"], o["lm_failed"]) == (want["converged"], want["lm_failed"]), note
        assert o["outer_it"] == want["outer_it"] and o["nu"] == want["nu"], note
        assert rec["lambda"] == c["lambda"] and rec["nu"] == c["nu"] and rec["trial"] == c.get("inner_it", 0), note
        if want["decision"] == 1:  # x*x*x against pow
            lam, ref = o["lambda"], want["lambda"]
            assert (lam == ref) or abs(lam - ref) <= lm_ref.LAMBDA_ULPS * np.spacing(abs(ref)) or (math.isnan(lam) and math.isnan(ref)), note
            assert np.array_equal(o["R"], o["Rt"], equal_nan=True) and np.array_equal(o["t"], o["tt"], equal_nan=True)
        else:  # rejections are bit-exact
            assert np.array_equal(np.float64(o["lambda"]), np.float64(want["lambda"])), note
            assert np.array_equal(o["R"], np.asarray(c.get("R", np.eye(3)))), note
        phase = 2 if want["done"] else (1 if want["decision"] == 0 else 0)
        assert o["phase"] == phase, note
        # rho: where the inputs are finite, within its bound of the exact value for the device's step
        exact, err = lm_ref.rho_ref(c["y0"], c["yi"], rec["d"], c["lambda"], c["b"])
        if math.isfinite(err):
            assert abs(float(exact) - rec["rho"]) <= err, note
        seen.add(int(rec["decision"]))
    assert seen == {0, 1, 2, 3}
    by = {note: (c, o) for (c, note), o in zip(cases, out)}
    # the crafted cases reach the edges they claim
    assert by["rho +0"][1]["record"]["rho"] == 0 and not np.signbit(by["rho +0"][1]["record"]["rho"])
    assert math.isnan(by["NaN H"][1]["record"]["rho"]) and np.isnan(by["NaN H"][1]["dR"]).all()
    assert by["NaN H"][1]["record"]["decision"] == 1 and by["NaN H"][1]["converged"] == 0  # a NaN step is not converged
    assert by["rho -0"][1]["record"]["rho"] == 0 and np.signbit(by["rho -0"][1]["record"]["rho"])
    # |t| = eps exactly: converged under (1.0 / eps) * |t|
    eps_out = [(c, o) for (c, note), o in zip(cases, out) if note.startswith("eps boundary")]
    assert len(eps_out) == 2 * len(BOUNDARY_EPS)
    for c, o in eps_out:
        assert o["dt"][1] == c["params"].transformation_eps and np.array_equal(o["dR"], np.eye(3))
        assert o["converged"] == 1 and o["record"]["decision"] in (1, 2)


@pytest.mark.gpu
def test_tap_lambda_rule_across_one_third(ctx):
    """lambda after an accept, x*x*x on the device against pow, on both sides of 1 - x^3 = 1/3."""
    I6 = np.eye(6)
    b = np.array([0.0, 0.0, 0.0, -1.0, 0.0, 0.0])
    x0 = (2.0 / 3.0) ** (1.0 / 3.0)
    d = 1.0 / 1.7  # H = I, lambda = 0.7: d = -b / 1.7 and d.(lambda d - b) = d (0.7 d + 1)
    denom = d * (0.7 * d + 1.0)
    cases = []
    for k in range(-40, 41):
        rho = (x0 + 1) / 2 + k * 1e-3
        cases.append(dict(H=I6, b=b, y0=10.0, yi=10.0 - rho * denom, mode="trial", nu=2.0, **{"lambda": 0.7}))
    out = ctx.lm_step_tap(cases)
    sides = set()
    for c, o in zip(cases, out):
        rho = float(o["record"]["rho"])
        ref = lm_ref.lambda_accept(0.7, rho)
        assert o["record"]["decision"] == 1
        assert abs(o["lambda"] - ref) <= lm_ref.LAMBDA_ULPS * np.spacing(ref)
        sides.add(ref == 0.7 / 3.0)
    assert sides == {True, False}


@pytest.mark.gpu
def test_tap_linearize_mode(ctx):
    rng = np.random.default_rng(4)
    H = lm_ref.spd(rng, 1e6)
    b = rng.normal(size=6)
    Hn = H.copy()
    Hn[3, 3] = np.nan
    cases = [dict(H=H, b=b, y0=3.0, mode="linearize", **{"lambda": -1.0}),
             dict(H=H, b=b, y0=3.0, mode="linearize", **{"lambda": 0.25}, nu=64.0, inner_it=5),
             dict(H=Hn, b=b, y0=3.0, mode="linearize", **{"lambda": -1.0}),
             dict(H=H, b=b, y0=3.0, mode="linearize", **{"lambda": -1.0}, params=_prm(lm_max_iterations=0)),
             dict(H=H, b=b, y0=3.0, mode="linearize", **{"lambda": -1.0}, params=_prm(lm_max_iterations=-3)),
             dict(H=H, b=b, y0=3.0, mode="linearize", **{"lambda": -1.0}, params=_prm(lm_max_iterations=1))]
    out = ctx.lm_step_tap(cases)
    for c, o in zip(cases, out):
        st = lm_ref.start(dict(c, params=c.get("params") or _prm()))
        lam = o["lambda"]
        assert (lam == st["lambda"]) or (math.isnan(lam) and math.isnan(st["lambda"]))
        assert o["nu"] == 2.0 and o["inner_it"] == 0
        assert o["has_trial"] == int(st["trial"]) and o["lm_failed"] == st["lm_failed"]
        if st["trial"]:
            assert o["phase"] == 1
            if not math.isnan(lam):
                _check_trial_prep(dict(c, **{"lambda": lam}), o)
        else:  # no trial: finished, not converged, x0 untouched
            assert o["phase"] == 2 and o["converged"] == 0 and np.array_equal(o["R"], np.eye(3))
    assert out[0]["lambda"] == 1e-9 * np.abs(np.diag(H)).max()
    assert math.isnan(out[2]["lambda"])


# ---------------------------------------------------------------------------------------------------------------------
# traced solves
def _traced(ctx, src, dst, prm, guess=None):
    cs, ct = ctx.create_clouds([src, dst])
    ctx.set_lm_trace(True)
    try:
        res = ctx.gicp_align([cs], [ct], params=prm, guesses=None if guess is None else [guess])[0]
        tr = ctx.lm_trace()[0]
    except Exception:
        cs.destroy(); ct.destroy()
        raise
    finally:
        ctx.set_lm_trace(False)
    return cs, ct, res, tr


def _lin_poses(tr, guess):
    """The pose of each record's linearization: the guess, then x0 after the previous record."""
    g = np.eye(4) if guess is None else np.asarray(guess, np.float64)
    poses = []
    for k in range(len(tr)):
        P = np.eye(4)
        P[:3] = g[:3] if k == 0 else tr["T"][k - 1]
        poses.append(P)
    return poses


def _case_of(rec, lin, pose, prm):
    return dict(H=lin["H"], b=lin["b"], y0=lin["err"], yi=float(rec["yi"]), R=pose[:3, :3], t=pose[:3, 3], nu=float(rec["nu"]),
                outer_it=int(rec["outer"]), inner_it=int(rec["trial"]), params=prm, mode="trial", **{"lambda": float(rec["lambda"])})


@pytest.mark.gpu
def test_tap_is_the_solves_controller(ctx, synth):
    """Every trial of traced solves, bit for bit: linearize reproduces y0, the tap reproduces d, rho, the decision and
    lambda / nu, compute_error at the tap's trial pose reproduces yi."""
    s, d, _ = synth.make_pair(1104, 5000, 5000)
    runs = [(s, d, synth.se3(yaw=0.8, t=(1.0, 0.0, 0.0)), _prm()), (s, d, None, _prm(lm_max_iterations=1)),
            (*synth.make_pair(1001, 5000, 6000)[:2], None, _prm())]
    n = 0
    for src, dst, guess, prm in runs:
        cs, ct, res, tr = _traced(ctx, src, dst, prm, guess)
        try:
            poses = _lin_poses(tr, guess)
            lins = {}
            cases = []
            for k, rec in enumerate(tr):
                key = int(rec["outer"])
                if key not in lins:
                    lins[key] = ctx.linearize(cs, ct, poses[k], prm.max_corr_dist)
                lin = lins[key]
                assert np.float64(lin["err"]).tobytes() == np.float64(rec["y0"]).tobytes()
                cases.append(_case_of(rec, lin, poses[k], prm))
            out = ctx.lm_step_tap(cases)
            for k, (rec, c, o) in enumerate(zip(tr, cases, out)):
                assert o["d"].tobytes() == rec["d"].tobytes(), k
                assert o["record"].tobytes() == rec.tobytes(), k
                if k + 1 < len(tr) and tr[k + 1]["outer"] == rec["outer"]:
                    assert np.float64(o["lambda"]) == tr[k + 1]["lambda"] and o["nu"] == tr[k + 1]["nu"]
                T = np.eye(4)
                T[:3, :3], T[:3, 3] = o["Rt"], o["tt"]
                yi = ctx.compute_error(cs, ct, poses[k], T, prm.max_corr_dist)
                assert np.float64(yi).tobytes() == np.float64(rec["yi"]).tobytes(), k
                n += 1
        finally:
            cs.destroy(); ct.destroy()
    assert n >= 10


def _ground(rng, n, T=None, noise=0.02):
    p = np.column_stack([rng.uniform(-40, 40, n), rng.uniform(-40, 40, n), rng.normal(0, noise, n)])
    return _place(p, T)


def _corridor(rng, n, T=None, noise=0.01):
    k = n // 3
    x = rng.uniform(-30, 30, n)
    wall = np.column_stack([x[:2 * k], np.where(np.arange(2 * k) < k, -2.0, 2.0) + rng.normal(0, noise, 2 * k), rng.uniform(0, 3, 2 * k)])
    floor = np.column_stack([x[2 * k:], rng.uniform(-2, 2, n - 2 * k), rng.normal(0, noise, n - 2 * k)])
    return _place(np.vstack([wall, floor]), T)


def _place(p, T):
    if T is not None:
        p = p @ T[:3, :3].T + T[:3, 3]
    return p.astype(np.float32)


def _scene_stats(ctx, name, src, dst, prm, guess=None):
    """Traced solve of one scene: every trial's d against the exact solve of its own system, every certifiable decision
    against decide().  -> dict of the reported numbers"""
    cs, ct, res, tr = _traced(ctx, src, dst, prm, guess)
    try:
        assert len(tr) == res["n_error"] > 0
        poses = _lin_poses(tr, guess)
        lins = {}
        kappa, worst, uncertified, nan_trials, no_bound = 0.0, 0.0, 0, 0, 0
        for k, rec in enumerate(tr):
            key = int(rec["outer"])
            if key not in lins:
                lins[key] = ctx.linearize(cs, ct, poses[k], prm.max_corr_dist)
            lin = lins[key]
            H, b, lam, d = lin["H"], lin["b"], float(rec["lambda"]), rec["d"]
            if not (np.isfinite(H).all() and np.isfinite(b).all() and math.isfinite(lam)):
                nan_trials += 1
                uncertified += 1
                continue
            A = lm_ref.shifted(H, lam)
            kappa = max(kappa, float(np.linalg.cond(A)))
            ex = lm_ref.solve_exact(H, b, lam)
            bound = lm_ref.solve_bound(H, b, lam, d)
            if ex is None or not np.isfinite(bound).all():  # singular or not positive definite: no bound to hold it to
                no_bound += 1
                uncertified += 1
                continue
            err = np.abs(d - np.array([float(x) for x in ex]))
            assert (err <= bound).all(), (name, k, err, bound)
            worst = max(worst, float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1), 0))))
            # the decision, where the restatement is certain of it
            rho, rerr = lm_ref.rho_ref(lin["err"], float(rec["yi"]), d, lam, b)
            sign_certain = isinstance(rho, Fraction) and (rho == 0 or abs(float(rho)) > rerr)
            Rref = lm_ref.so3_exp_ref(d[:3]).astype(np.float64)
            m = lm_ref.so3_bound(d[:3])
            vals = list((1.0 / prm.rotation_eps) * np.abs(Rref - np.eye(3)).ravel()) + list((1.0 / prm.transformation_eps) * np.abs(d[3:]))
            marg = [(1.0 / prm.rotation_eps) * m] * 9 + [0.0] * 3
            conv_certain = all(v + e < 1 for v, e in zip(vals, marg)) or any(v - e >= 1 for v, e in zip(vals, marg))
            if not (sign_certain and conv_certain):
                uncertified += 1
                continue
            c = dict(nu=float(rec["nu"]), inner_it=int(rec["trial"]), outer_it=int(rec["outer"]), params=prm, **{"lambda": lam})
            want = lm_ref.decide(c, float(rho) if rho != 0 else 0.0, Rref, d[3:])
            assert rec["decision"] == want["decision"], (name, k)
        return dict(scene=name, trials=len(tr), kappa=kappa, worst_err_over_bound=worst, uncertified=uncertified,
                    nan_trials=nan_trials, no_bound=no_bound, converged=res["converged"], iterations=res["iterations"])
    finally:
        cs.destroy(); ct.destroy()


@pytest.mark.gpu
def test_degenerate_scenes(ctx, synth):
    rng = np.random.default_rng(11)
    off = synth.se3(yaw=0.05, roll=0.02, t=(1.0, 0.6, 0.2))
    s100, d100, _ = synth.make_pair(1000, 100000)
    a_s, a_d, a_T = synth.make_pair(1001, 5000, 6000)
    # PLANE keeps some in-plane information (its covariances are (1, 1, 1e-3) in the surface frame); NONE on surfaces with
    # 10 um of noise leaves x, y and yaw of the plane (the corridor's axis) nearly unobservable
    scenes = [("ground plane", _ground(rng, 30000, off), _ground(rng, 30000), _prm()),
              ("corridor", _corridor(rng, 30000, off), _corridor(rng, 30000), _prm()),
              ("ground plane, NONE", _ground(rng, 30000, off, 1e-5), _ground(rng, 30000, None, 1e-5), _prm(regularization=0)),
              ("corridor, NONE", _corridor(rng, 30000, off, 1e-5), _corridor(rng, 30000, None, 1e-5), _prm(regularization=0)),
              ("raw 100k, NONE", s100, d100, _prm(regularization=0)),
              ("already aligned", a_s, a_d, _prm())]
    stats = []
    for name, src, dst, prm in scenes:
        stats.append(_scene_stats(ctx, name, src, dst, prm, a_T if name == "already aligned" else None))
    for s in stats:
        print("LM scene %(scene)s: trials %(trials)d, largest kappa %(kappa).3g, largest |d - d_exact| / bound "
              "%(worst_err_over_bound).3g, uncertified decisions %(uncertified)d (non-finite systems %(nan_trials)d, not positive "
              "definite %(no_bound)d), "
              "converged %(converged)s after %(iterations)d" % s)
    assert min(s["kappa"] for s in stats[2:4]) > 1e7, "the plane and the corridor under NONE are degenerate"


# ---------------------------------------------------------------------------------------------------------------------
# the findings, end to end against the oracle
def _both(ctx, oracle, src, dst, guess=None, **kv):
    from oracle.oracle import GicpParams
    prm = _prm(**kv)
    oprm = GicpParams.default()
    for k, v in kv.items():
        setattr(oprm, k, v)
    cs, ct = ctx.create_clouds([src, dst])
    try:
        ctx.set_lm_trace(True)
        r = ctx.gicp_align([cs], [ct], params=prm, guesses=None if guess is None else [guess])[0]
        tr = ctx.lm_trace()[0]
    finally:
        ctx.set_lm_trace(False)
        cs.destroy(); ct.destroy()
    o = oracle.gicp_align(src, dst, params=oprm, guess=guess)
    keys = ("converged", "iterations", "n_linearize", "n_error", "lm_failed")
    assert tuple(bool(r[k]) if k in ("converged", "lm_failed") else r[k] for k in keys) == tuple(o[k] for k in keys)
    return r, o, tr


@pytest.mark.gpu
def test_zero_lm_iterations_runs_no_trial(ctx, oracle, synth):
    src, dst, _ = synth.make_pair(1001, 5000, 6000)
    g = synth.se3(yaw=0.05, t=(0.3, 0.0, 0.0))
    r, o, tr = _both(ctx, oracle, src, dst, g, lm_max_iterations=0)
    assert (r["converged"], r["iterations"], r["n_linearize"], r["n_error"], r["lm_failed"]) == (False, 0, 1, 0, True)
    assert len(tr) == 0 and np.array_equal(r["T"], g)


@pytest.mark.gpu
def test_none_clusters_nan_step(ctx, oracle):
    """regularization NONE with identical-point clusters in both clouds: C_t + R C_s R^T = 0, its inverse and H are NaN,
    lambda is NaN, and no step is ever converged: the solve runs to max_iterations like the reference's."""
    src, dst = lm_ref.cluster_pair()
    r, o, tr = _both(ctx, oracle, src, dst, regularization=0, max_iterations=6)
    assert (r["converged"], r["iterations"], r["n_linearize"], r["lm_failed"]) == (False, 5, 6, False)
    assert np.isnan(tr["d"]).all() and (tr["decision"] == 1).all() and np.isnan(tr["lambda"]).all()


@pytest.mark.gpu
def test_eps_boundary_and_nan_through_the_tap(ctx):
    """One certain case per finding, through the product's controller (the reverted forms fail each)."""
    I6 = np.eye(6)
    cases = []
    for eps in BOUNDARY_EPS:
        cases.append(dict(H=I6, b=np.array([0, 0, 0, -eps, 0, 0.0]), y0=10.0, yi=11.0, mode="trial", **{"lambda": 0.0},
                          params=_prm(transformation_eps=eps, rotation_eps=1.0)))
    cases.append(dict(H=np.full((6, 6), np.nan), b=np.ones(6), y0=10.0, yi=np.nan, mode="trial", **{"lambda": 1e-3}))
    cases.append(dict(H=I6, b=np.ones(6), y0=10.0, mode="linearize", **{"lambda": -1.0}, params=_prm(lm_max_iterations=0)))
    out = ctx.lm_step_tap(cases)
    for o in out[:len(BOUNDARY_EPS)]:
        assert o["record"]["decision"] == 2 and o["converged"] == 1  # rejected, but (1.0 / eps) * eps < 1
    nan = out[len(BOUNDARY_EPS)]
    assert nan["record"]["decision"] == 1 and nan["converged"] == 0 and nan["phase"] == 0
    zero = out[-1]
    assert zero["has_trial"] == 0 and zero["lm_failed"] == 1 and zero["converged"] == 0 and zero["phase"] == 2
