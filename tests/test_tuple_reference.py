"""optimizedMatching's tuple test (matcher.cc:461-538) restated in numpy fp32, and what it says about two of its edges:

* normalizePoints' mean.  The reference (and the oracle) sum the points in fp32 in original order; k_cloud_sum sums in
  fp64 and casts the mean to fp32.  Kilometres from the map origin the two means differ by centimetres.  The restated
  loop is run under both means on pairs shifted by (3000, -2000, 50) m: every normalised length moves (the max radius
  that divides them moves), but no trial of the tuple test changes its verdict, so the device keeps its fp64 mean.
* tuple_scale == 0: the tuple block is the only writer of corres_, so optimizedMatching keeps nothing and the stage is
  invalid with the identity; advancedMatching keeps every cross-checked pair.
"""
import numpy as np
import pytest

SHIFT = np.array([3000.0, -2000.0, 50.0])
SEEDS = range(2000, 2020)


def _splitmix64(x):
    x = x + np.uint64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def _draw(seed, t, k, n):
    """The counter-based generator that replaces rand() (oracle_quatro.cpp `draw`, quatro.cu `draw`)."""
    with np.errstate(over="ignore"):
        return (_splitmix64(np.uint64(seed) ^ _splitmix64(t * np.uint64(4) + np.uint64(k))) % np.uint64(n)).astype(np.int64)


def mean_fp32_running(P):
    """Matcher::normalizePoints' mean: an fp32 running sum in original order, divided by n in fp32."""
    acc = np.zeros(3, np.float32)
    for p in np.asarray(P, np.float32)[:, :3]:
        acc = acc + p
    return acc / np.float32(len(P))


def mean_fp64(P):
    """k_cloud_sum's mean: the fp64 sum over n, cast to fp32."""
    return (np.asarray(P, np.float32)[:, :3].astype(np.float64).sum(0) / len(P)).astype(np.float32)


def normalize(clouds, means):
    pc = [(np.asarray(P, np.float32)[:, :3] - m).astype(np.float32) for P, m in zip(clouds, means)]
    scale = max(np.sqrt((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2]).max() for c in pc)
    return [c / scale for c in pc] if scale != np.float32(1) else pc


def tuple_trials(pc_i, pc_j, mutual, tuple_scale, seed=1):
    """Every trial's verdict (vectorised; each is independent) -> (pass (trials,), r0, r1, r2)."""
    n = len(mutual)
    t = np.arange(100 * n, dtype=np.uint64)
    r0, r1, r2 = (_draw(seed, t, k, n) for k in range(3))
    I, J = mutual[:, 0], mutual[:, 1]
    ts = np.float32(tuple_scale)

    def ln(pc, a, b):
        d = pc[a] - pc[b]
        return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    li0, lj0 = ln(pc_i, I[r0], I[r1]), ln(pc_j, J[r0], J[r1])
    li1, li2, lj1, lj2 = ln(pc_i, I[r1], I[r2]), ln(pc_i, I[r2], I[r0]), ln(pc_j, J[r1], J[r2]), ln(pc_j, J[r2], J[r0])
    ok = ~((li0 * ts > lj0) | (lj0 > li0 / ts))
    ok &= (li1 * ts < lj1) & (lj1 < li1 / ts) & (li2 * ts < lj2) & (lj2 < li2 / ts)
    return ok, r0, r1, r2, li0


def tuple_select(ok, r0, r1, r2, n, max_corres):
    """The serial loop: members of passing trials in insertion order, stop once more than max_corres are kept."""
    inc = np.zeros(n, bool)
    out = []
    for k in np.flatnonzero(ok):
        for r in (r0[k], r1[k], r2[k]):
            if not inc[r]:
                inc[r] = True
                out.append(r)
        if len(out) > max_corres:
            break
    return np.array(out, np.int64)


@pytest.fixture(scope="module")
def far_pairs(oracle, synth):
    out = []
    for seed in SEEDS:
        src, dst, _ = synth.make_pair(seed, 8000, 9000, mode="quatro")
        src, dst = src.copy(), dst.copy()
        for a in (src, dst):
            a[:, :3] = (a[:, :3].astype(np.float64) + SHIFT).astype(np.float32)
        fs, fd = oracle.fpfh(src)[2], oracle.fpfh(dst)[2]
        corr, mutual = oracle.match(src, dst, fs, fd)
        out.append((seed, src, dst, corr, mutual))
    return out


def test_far_from_origin_the_mean_flips_no_tuple_trial(far_pairs):
    gaps, moved, flips, margin = [], [], 0, np.inf
    for seed, src, dst, corr, mutual in far_pairs:
        clouds = [dst, src]  # fi = the larger cloud (matcher.cc:364-369): dst has 9000 points
        pa = normalize(clouds, [mean_fp32_running(P) for P in clouds])
        pb = normalize(clouds, [mean_fp64(P) for P in clouds])
        oka, r0, r1, r2, la = tuple_trials(pa[0], pa[1], mutual, 0.95)
        okb, _, _, _, lb = tuple_trials(pb[0], pb[1], mutual, 0.95)
        # the restated loop under the reference's mean IS the oracle's matcher
        sel = tuple_select(oka, r0, r1, r2, len(mutual), 200)
        assert np.array_equal(mutual[sel][:, ::-1], corr), seed
        flips += int((oka != okb).sum())
        gaps.append(max(float(np.abs(mean_fp32_running(P).astype(np.float64) - mean_fp64(P)).max()) for P in clouds))
        moved.append(float((la != lb).mean()))
    # measured over the 20 pairs: mean gaps of 4.4 mm to 18.8 mm; 98.3 % to 99.9 % of the first-edge lengths differ in
    # their last bits; no verdict flips (the ratios move by fp32 rounding only; the closest lies ~2e-6 from its bound)
    assert max(gaps) > 1e-2 and min(moved) > 0.95
    assert flips == 0


def test_tuple_scale_zero_keeps_nothing_in_optimized_matching(oracle, synth):
    src, dst, _ = synth.make_pair(2000, 8000, 9000, mode="quatro")
    fs, fd = oracle.fpfh(src)[2], oracle.fpfh(dst)[2]
    p = oracle.QuatroParams.default()
    p.tuple_scale = 0.0
    corr, mutual = oracle.match(src, dst, fs, fd, p)
    assert len(mutual) > 100 and len(corr) == 0
    q = oracle.quatro_align(src, dst, p)
    assert not q["valid"] and q["n_corr"] == 0 and np.array_equal(q["T"], np.eye(4))


def test_tuple_scale_zero_keeps_everything_in_advanced_matching(oracle, synth):
    src, dst, _ = synth.make_pair(2000, 8000, 9000, mode="quatro")
    fs, fd = oracle.fpfh(src)[2], oracle.fpfh(dst)[2]
    p = oracle.QuatroParams.default()
    p.tuple_scale = 0.0
    keep = oracle.match_advanced(src, dst, fs, fd, p)
    assert np.array_equal(keep, oracle.match_advanced(src, dst, fs, fd, tuple_test=False))
    assert len(keep) > len(oracle.match_advanced(src, dst, fs, fd)) > 0
