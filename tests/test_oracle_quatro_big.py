"""The oracle's TEASER++ solve on a correspondence set larger than 8192, against a numpy restatement of its graph steps:
TIM graph, core numbers by one-at-a-time peeling, the (core desc, degree desc, index asc) order and the greedy clique
grown from every start (largest first, lowest rank on ties)."""
import numpy as np

from teaser_ref import _greedy_clique_numpy
from test_gpu_quatro_big import synthetic_set


def test_oracle_solve_beyond_8192_matches_numpy(oracle, synth):
    n = 9000
    S, D, Texp = synthetic_set(n, seed=n)
    o = oracle.quatro_solve(S, D, np.repeat(np.arange(n, dtype=np.int32)[:, None], 2, 1))
    clique = _greedy_clique_numpy(S[:, :3].astype(np.float64), D[:, :3].astype(np.float64))
    assert np.array_equal(o["clique"], clique)
    assert o["valid"] and len(clique) >= 300
    rot, tr = synth.se3_error(o["T"], Texp)
    assert rot < 1e-2 and tr < 0.1
