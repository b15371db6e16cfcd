"""optimizedMatching's tuple test at caps above 509: the oracle's matcher equals the serial restatement of
test_tuple_reference.py at max_corres 1000 (the loop stops at the cap) and 8189 (every passing trial is kept), and keeps
at most max_corres + 3 correspondences."""
import numpy as np
import pytest

from test_tuple_reference import mean_fp32_running, normalize, tuple_select, tuple_trials


@pytest.fixture(scope="module")
def pair_50k(oracle, synth):
    """2912 mutual matches: a 0.8 tuple test keeps 2748 of them, a 0.99 one 1629."""
    src, dst, _ = synth.make_pair(2004, 50000, 50000, mode="quatro")
    fs, fd = oracle.fpfh(src)[2], oracle.fpfh(dst)[2]
    return src, dst, fs, fd


@pytest.mark.parametrize("tuple_scale", [0.8, 0.99])
@pytest.mark.parametrize("max_corres", [1000, 8189])
def test_oracle_match_equals_serial_restatement(oracle, pair_50k, max_corres, tuple_scale):
    src, dst, fs, fd = pair_50k
    p = oracle.QuatroParams.default()
    p.max_corres, p.tuple_scale = max_corres, tuple_scale
    corr, mutual = oracle.match(src, dst, fs, fd, p)
    swapped = len(dst) > len(src)  # fi = the larger cloud (matcher.cc:364-369); equal sizes: fi = src
    clouds = [dst, src] if swapped else [src, dst]
    pc = normalize(clouds, [mean_fp32_running(P) for P in clouds])
    ok, r0, r1, r2, _ = tuple_trials(pc[0], pc[1], mutual, tuple_scale, seed=p.seed)
    sel = tuple_select(ok, r0, r1, r2, len(mutual), max_corres)
    want = mutual[sel][:, ::-1] if swapped else mutual[sel]
    assert np.array_equal(corr, want)
    assert len(corr) <= max_corres + 3
    if max_corres == 1000:
        assert max_corres < len(corr)  # the loop stopped at the cap
    else:
        assert len(corr) == len(np.unique(np.r_[r0[ok], r1[ok], r2[ok]]))  # nothing stopped it
