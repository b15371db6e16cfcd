"""The fp32 restatement of the feature matcher (tests/match_ref.py) against the CPU oracle's optimizedMatching /
advancedMatching, its fp64 certificate, and the margin of k_feat_nn's projected lower bound measured on the crafted
extremes of the descriptor domain."""
import numpy as np
import pytest

import match_ref as M

CASES = M.crafted_cases() + M.size_cases()[::5]


def _points(rng, n):
    return rng.uniform(-20, 20, (n, 3)).astype(np.float32)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_match_ref_equals_oracle(oracle, case):
    rng = np.random.default_rng(1)
    src, dst = _points(rng, len(case.fi)), _points(rng, len(case.fj))
    for thr in case.thrs:
        p = oracle.QuatroParams.default()
        p.distance_threshold = thr
        r = M.match_ref(case.fi, case.fj, thr)
        _, mutual = oracle.match(src, dst, case.fi, case.fj, p)  # fi = src (ni >= nj): no swap
        assert np.array_equal(r["mutual"], mutual), thr
    keep = oracle.match_advanced(src, dst, case.fi, case.fj, tuple_test=False)
    ra = M.match_ref(case.fi, case.fj, advanced=True)
    m = ra["mutual"]
    assert np.array_equal(m[np.lexsort((m[:, 1], m[:, 0]))], keep)  # the oracle lists them sorted by (src, dst)


def test_gate_cases_are_what_they_claim():
    case = next(c for c in M.crafted_cases() if c.name == "gate")
    r = M.match_ref(case.fi, case.fj, advanced=True)
    d = set(r["dis"][r["nn"] >= 0].tolist())
    assert {0.0, 16.0, 16.0 + 2.0 ** -19, 16.0 + 2.0 ** -18, 16.0 + 3 * 2.0 ** -19} <= d, sorted(d)
    assert np.float32(16.0 + 2.0 ** -19) == np.nextafter(np.float32(16), np.float32(17))
    assert M.thr2_of(4.0) == 16 and M.thr2_of(float(np.nextafter(np.float32(4), np.float32(5)))) == np.float32(16.0 + 2.0 ** -18)
    assert np.isinf(M.thr2_of(1e20))
    four, below, above, zero, huge, nan = [int((M.match_ref(case.fi, case.fj, t)["nn"] >= 0).sum()) for t in case.thrs]
    # thr 4: d2 = 16 kept, 16 + 2^-19 (the next float) dropped; the next thr squares to 16 + 2^-18 (rounded); the thr
    # below 4 squares below 16 and keeps the d2 = 0 records only, as thr = 0 does
    assert huge == nan == int((r["nn"] >= 0).sum()) > above > four > below == zero > 0


def test_crafted_ties_cover_both_sweep_directions():
    above = below = 0
    for c in M.crafted_cases():
        if c.name.startswith("tie_lattice"):
            a, b = M.tie_coverage(c.fj, c.fi)
            above, below = above + a, below + b
    print("\nforward queries whose lowest-index tie lies in a later-visited tile: %d above s_t0, %d below" % (above, below))
    assert above > 0 and below > 0


def test_reverse_ties_cover_both_sweep_directions():
    """The reverse search runs over fi's sorted blocks (every row of fi, only the rows some j reached search)."""
    above = below = 0
    for c in M.crafted_cases():
        if "tie_lattice" in c.name:
            r = M.match_ref(c.fi, c.fj)
            a, b = M.tie_coverage(c.fi, c.fj, searched=r["rnn"] >= 0)
            above, below = above + a, below + b
    print("\nreverse queries likewise: %d above, %d below" % (above, below))
    assert above > 0 and below > 0


def test_crafted_set_reaches_the_filter_margin():
    """The near-tight case puts winners and their exact-tie members inside filt_bound's allowance, in both directions:
    there a filter without its margin (or with a smaller one) could drop them, so the GPU comparison on this case tests
    the margin.  And the emulated filter never exceeds the allowance on them."""
    c = next(c for c in M.crafted_cases() if c.name == "projected_tight_and_extremes")
    r = M.match_ref(c.fi, c.fj, advanced=True)
    fwd = M.bound_approach(c.fj, c.fi)
    rev = M.bound_approach(c.fi[r["rnn"] >= 0], c.fj)
    print("\nnear-tight case: sqrt(filt_lb) - sqrt(d2) of winners and tie members, forward: %d of %d within 4e-3, closest "
          "%.3e; reverse: %d of %d, closest %.3e" % ((fwd > -4e-3).sum(), len(fwd), fwd.max(), (rev > -4e-3).sum(), len(rev),
                                                    rev.max()))
    assert (fwd > -4e-3).sum() >= 50 and (rev > -4e-3).sum() >= 20
    assert fwd.max() > -1e-4 and rev.max() > -1e-4
    assert np.all(fwd <= 4e-3) and np.all(rev <= 4e-3)
    # an anchor at |a - mu| = 220.5 among the queries whose winner is near-tight
    x = np.linalg.norm(c.fj.astype(np.float64) - M.FB_MU.astype(np.float64), axis=1)
    assert abs(x.max() - M.max_centered_norm()) < 1e-9


def test_fp64_certificate_on_crafted_cases():
    for c in M.crafted_cases()[:4]:
        r = M.match_ref(c.fi, c.fj, advanced=True)
        cert = M.certify_fp64(c.fj, c.fi, M.usable(c.fi), r["nn"].astype(np.int64))
        assert cert["differ"] == 0, (c.name, cert)  # integer bins: every d2 is exact


def test_filter_margin_on_extremes():
    """sqrt(filt_lb) - sqrt(d2) <= filt_bound's allowance (1e-5 relative + 4e-3) for every pair with d2 > 0 of crafted
    extremes: one-hot blocks (|a - mu| = 220.5 at the smallest mu), the near-tight pairs of projected_tight (residuals
    parallel: filt_lb = d2 up to rounding), and random descriptors."""
    xmax = M.max_centered_norm()
    assert abs(xmax - 220.5) < 0.01
    excess = M.derived_excess(xmax)
    print("\nmax |a - mu| %.3f; derived worst-case excess of sqrt(filt_lb) over the true bound %.3e (allowance 4e-3)"
          % (xmax, excess))
    assert excess < 4e-3
    rng = np.random.default_rng(3)
    fi, fj = M.projected_tight(rng)
    F = np.concatenate([M.one_hot_extremes(), fi, fj, M.random_desc(rng, 300, conc=0.3)])
    P = M.filter_coords(F)
    x = np.linalg.norm(F.astype(np.float64) - M.FB_MU.astype(np.float64), axis=1)
    assert x.max() <= xmax + 1e-6 and x.max() > 220.0
    worst, room_min = -np.inf, np.inf
    for a in range(0, len(F), 256):
        q = np.arange(a, min(a + 256, len(F)))
        lb = M.filt_lb(P[q][:, None, :], P[None, :, :]).astype(np.float64)
        d2 = np.stack([M.d2_fp32(np.repeat(F[k:k + 1], len(F), 0), F) for k in q]).astype(np.float64)
        off = d2 > 0  # a record paired with itself (or a copy) is not a test of the bound
        ex = np.where(off, np.sqrt(lb) - np.sqrt(d2), -np.inf)
        room = np.where(off, M.filt_margin(d2) - ex, np.inf)
        worst = max(worst, float(ex.max()))
        room_min = min(room_min, float(room.min()))
    print("crafted extremes and near-tight pairs (%d records, pairs with d2 > 0): closest approach sqrt(filt_lb) - sqrt(d2) "
          "%.3e, least room left in the margin %.3e" % (len(F), worst, room_min))
    assert room_min > 0
    assert worst > -1e-4  # the set holds near-tight pairs: the room measured is that of the margin, not of loose pairs
