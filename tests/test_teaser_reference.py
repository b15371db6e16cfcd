"""The oracle's TEASER++ solve against the fp64 restatement in teaser_ref.py, on crafted sets that reach every edge of the
solve and on random sets; and each crafted set shown to pin the rule it is meant to reach."""
import math

import numpy as np
import pytest

import teaser_ref as tr

CASES = tr.crafted_cases()


def oracle_params(oracle, prm):
    p = oracle.QuatroParams.default()
    p.noise_bound, p.rot_gnc_factor, p.rot_cost_thr, p.rot_max_iter = prm.noise_bound, prm.gnc_factor, prm.cost_thr, prm.max_iter
    return p


def oracle_solve(oracle, S, D, prm):
    n = len(S)
    corr = np.repeat(np.arange(n, dtype=np.int32)[:, None], 2, 1)
    return oracle.quatro_solve(np.asarray(S, np.float32).reshape(n, 3), np.asarray(D, np.float32).reshape(n, 3), corr,
                               oracle_params(oracle, prm))


def assert_same(o, ref, tol=1e-12):
    valid, clique, iters, T = ref
    assert o["valid"] == valid
    assert np.array_equal(o["clique"], clique)
    assert o["gnc_iters"] == iters
    assert np.abs(o["T"] - T).max() <= tol, np.abs(o["T"] - T).max()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_crafted_case_pins_its_rule(case):
    assert case.probe(case), case.reaches


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_equals_restatement_on_crafted_sets(oracle, case):
    assert_same(oracle_solve(oracle, case.S, case.D, case.prm), case.solve())


@pytest.mark.parametrize("seed", range(20))
def test_oracle_equals_restatement_on_random_sets(oracle, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(50, 601))
    S, D = tr.natural_set(n, 100 + seed, n_in=int(rng.integers(3, n // 2)), noise=float(rng.choice([0.02, 0.1, 0.25])),
                          yaw=float(rng.uniform(-math.pi, math.pi)))
    prm = tr.Params(noise_bound=0.3)
    ref = tr.solve(S, D, prm)
    assert ref[0] and len(ref[1]) >= 3
    assert_same(oracle_solve(oracle, S, D, prm), ref)


def test_empty_set_is_invalid(oracle):
    o = oracle.quatro_solve(np.zeros((1, 3), np.float32), np.zeros((1, 3), np.float32), np.zeros((0, 2), np.int32))
    assert_same(o, tr.solve(np.zeros((0, 3)), np.zeros((0, 3))))
    assert not o["valid"] and len(o["clique"]) == 0 and np.array_equal(o["T"], np.eye(4))


@pytest.mark.parametrize("seed", range(5))
def test_closed_form_kabsch_equals_svd(seed):
    """The closed-form yaw of kabsch_yaw is the 2-D Kabsch rotation V diag(1, det) U^T of H = sum w x y^T."""
    rng = np.random.default_rng(seed)
    X = rng.normal(0, 5, (30, 2))
    Y = X @ np.array([[math.cos(1.1), math.sin(1.1)], [-math.sin(1.1), math.cos(1.1)]]) + rng.normal(0, 2, (30, 2))
    W = rng.uniform(0, 1, 30)
    cs, sn, h = tr.kabsch_yaw(X.tolist(), Y.tolist(), W.tolist())
    U, _, Vt = np.linalg.svd(np.array(h).reshape(2, 2))
    R = Vt.T @ np.diag([1, np.linalg.det(Vt.T @ U.T)]) @ U.T
    assert np.abs(R - [[cs, -sn], [sn, cs]]).max() < 1e-12
