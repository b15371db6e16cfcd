"""Per-trial trace of the CPU oracle's Levenberg-Marquardt solve, in the records of b200reg_lm_trial.

The oracle's solve (orc_gicp_align) reports one 64-double record per OUTER iteration: the pose at linearization, H, b, y0,
lambda after the step, the number of trials and the outcome.  Each trial of step_lm (lsq_registration_impl.hpp:170-205) is
then fixed by these: it is solved from H, b and the lambda in force, and its error is the oracle's own compute_error at the
trial pose with the correspondences of that linearization.  replay() restates those trials one by one, decides each by the
reference's rules, and refuses (AssertionError) a replay whose decisions, trial counts or lambdas differ from what the
oracle reported, so its records are the oracle's trials.
"""
import numpy as np

TRIAL_FIELDS = ("outer", "trial", "decision", "y0", "yi", "rho", "lambda", "nu", "d", "T")


def so3_exp(w):
    """so3_exp (so3.hpp:99-118) and Quaternion::toRotationMatrix, in the order the solvers evaluate them."""
    th2 = float(w @ w)
    if th2 < 1e-10:
        imag = 0.5 - 1.0 / 48.0 * th2 + 1.0 / 3840.0 * th2 * th2
        real = 1.0 - 1.0 / 8.0 * th2 + 1.0 / 384.0 * th2 * th2
    else:
        th = np.sqrt(th2)
        imag, real = np.sin(0.5 * th) / th, np.cos(0.5 * th)
    qw, qx, qy, qz = real, imag * w[0], imag * w[1], imag * w[2]
    tx, ty, tz = 2 * qx, 2 * qy, 2 * qz
    twx, twy, twz = tx * qw, ty * qw, tz * qw
    txx, txy, txz = tx * qx, ty * qx, tz * qx
    tyy, tyz, tzz = ty * qy, tz * qy, tz * qz
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1 - (txx + tyy)]])


def is_converged(delta, rotation_eps, transformation_eps):
    """LsqRegistration::is_converged (lsq_registration_impl.hpp:117-127): (1.0 / eps) * |x| as the reference writes it; a
    NaN anywhere in delta is not converged."""
    r = 1.0 / rotation_eps * np.abs(delta[:3, :3] - np.eye(3))
    t = 1.0 / transformation_eps * np.abs(delta[:3, 3])
    if np.isnan(r).any() or np.isnan(t).any():
        return False
    return max(r.max(), t.max()) < 1


def replay(oracle, src, tgt, params=None, guess=None):
    """-> (list of trial dicts with TRIAL_FIELDS, the oracle's gicp_align result with its per-outer "trace")."""
    prm = params or oracle.GicpParams.default()
    o = oracle.gicp_align(src, tgt, params=prm, guess=guess, want_trace=True)
    cov_s = oracle.covariances(src, prm.k_correspondences)
    cov_t = oracle.covariances(tgt, prm.k_correspondences)
    recs = []
    lam = None
    for it, row in enumerate(o["trace"]):
        x0 = row[:16].reshape(4, 4)
        H, b, y0 = row[16:52].reshape(6, 6), row[52:58], row[58]
        n_trials, outcome = int(row[60]), int(row[61])
        if lam is None:  # lm_lambda_ < 0 at the first step_lm of the solve (:165-167)
            lam = prm.lm_init_lambda_factor * np.abs(np.diag(H)).max()
        nu = 2.0
        if prm.lm_max_iterations <= 0:  # step_lm runs no trial and returns false: "lm not converged!!"
            assert (n_trials, outcome) == (0, 0) and it == len(o["trace"]) - 1, ("no trial", it, n_trials, outcome)
            break
        for i in range(prm.lm_max_iterations):
            d = np.linalg.solve(H + lam * np.eye(6), -b)
            delta = np.eye(4)
            delta[:3, :3] = so3_exp(d[:3])
            delta[:3, 3] = d[3:]
            xi = delta @ x0
            yi = oracle.compute_error(src, tgt, cov_s, cov_t, x0, xi, prm.max_corr_dist)
            rho = (y0 - yi) / (d @ (lam * d - b))
            if not rho < 0:  # rho < 0 rejects; anything else, 0 included, accepts (:191)
                decision = 1
            elif is_converged(delta, prm.rotation_eps, prm.transformation_eps):
                decision = 2
            else:
                decision = 3 if i == prm.lm_max_iterations - 1 else 0
            recs.append(dict(outer=it, trial=i, decision=decision, y0=y0, yi=yi, rho=rho, **{"lambda": lam}, nu=nu, d=d,
                             T=(xi if decision == 1 else x0)[:3].copy()))
            if decision == 1:
                lam = lam * max(1.0 / 3.0, 1 - (2 * rho - 1) ** 3)
                break
            if decision == 2:
                break
            lam, nu = nu * lam, 2 * nu
        # the oracle's own account of this outer iteration
        assert i + 1 == n_trials, ("trials", it, i + 1, n_trials)
        assert {1: 1, 2: 2, 3: 0}[decision] == outcome, ("outcome", it, decision, outcome)
        assert abs(lam - row[59]) <= 1e-6 * abs(row[59]), ("lambda after the step", it, lam, row[59])
        lam = row[59]
    assert len(recs) == o["n_error"]
    return recs, o
