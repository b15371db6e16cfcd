"""The oracle's per-trial LM trace (tests/lm_trials.py) against the oracle's own per-outer trace: same y0, number of trials,
outcome and lambda after each step; accepted trials move x0 to the next linearization's pose."""
import os

import numpy as np

import lm_trials

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gicp_oracle_3k.npz")


def _check_against_outer_trace(recs, o):
    tr = o["trace"]
    assert len(recs) == o["n_error"] and len({r["outer"] for r in recs}) == o["n_linearize"] == len(tr)
    for it, row in enumerate(tr):
        mine = [r for r in recs if r["outer"] == it]
        assert [r["trial"] for r in mine] == list(range(int(row[60])))
        assert all(r["y0"] == row[58] for r in mine)
        assert all(r["decision"] == 0 for r in mine[:-1])
        assert {1: 1, 2: 2, 0: 3}[int(row[61])] == mine[-1]["decision"]
        assert mine[0]["nu"] == 2.0 and all(b["nu"] == 2 * a["nu"] for a, b in zip(mine, mine[1:]))
        if it > 0:
            assert mine[0]["lambda"] == tr[it - 1, 59]  # lambda carries over from the previous outer iteration
            prev = [r for r in recs if r["outer"] == it - 1][-1]
            assert prev["decision"] == 1 and np.abs(prev["T"] - row[:16].reshape(4, 4)[:3]).max() < 1e-12
    assert np.abs(recs[-1]["T"] - o["T"][:3]).max() < 1e-12


def test_trials_of_the_golden_pair(oracle):
    g = np.load(GOLDEN)
    recs, o = lm_trials.replay(oracle, g["src"], g["dst"])
    # the committed trace, up to the summation order of the oracle's threaded sums
    assert np.abs(o["trace"] - g["trace"]).max() <= 1e-9 * np.abs(g["trace"]).max() and o["n_error"] == int(g["n_error"])
    _check_against_outer_trace(recs, o)


def test_trials_with_rejections(oracle, synth):
    """Started 0.8 rad off, the first outer iteration rejects five trials; lm_max_iterations = 1 turns the first rejection
    into "lm not converged!!" (3), and with epsilons of 10 it counts as converged (2)."""
    src, dst, _ = synth.make_pair(1104, 5000, 5000)
    guess = synth.se3(yaw=0.8, t=(1.0, 0.0, 0.0))
    seen = set()
    for kv in ({}, dict(lm_max_iterations=1), dict(transformation_eps=10.0, rotation_eps=10.0)):
        prm = oracle.GicpParams.default()
        for k, v in kv.items():
            setattr(prm, k, v)
        recs, o = lm_trials.replay(oracle, src, dst, params=prm, guess=guess)
        _check_against_outer_trace(recs, o)
        assert (recs[-1]["decision"] == 3) == o["lm_failed"]
        seen.update(r["decision"] for r in recs)
    assert seen == {0, 1, 2, 3}
