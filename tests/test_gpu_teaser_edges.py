"""The three device paths of the TEASER++ solve -- k_teaser_solve (shared memory, optimizedMatching's sets of at most 512),
the k_big_* chain for advancedMatching's sets up to 8192 ("global") and beyond ("wide") -- on the crafted edge sets of
teaser_ref.py and on sets at the shared solver's capacity, against the oracle and the fp64 restatement; and the tuple test
end to end, where its key buffer and the shared solver run full, and at tuple_scale == 0."""
import numpy as np
import pytest

import teaser_ref as tr

pytestmark = pytest.mark.gpu
CASES = tr.crafted_cases()
SHARED_CAP = 512


def device_params(native, prm):
    p = native.default_quatro_params()
    p.noise_bound, p.rot_gnc_factor, p.rot_cost_thr, p.rot_max_iter = prm.noise_bound, prm.gnc_factor, prm.cost_thr, prm.max_iter
    return p


def oracle_params(oracle, prm):
    p = oracle.QuatroParams.default()
    p.noise_bound, p.rot_gnc_factor, p.rot_cost_thr, p.rot_max_iter = prm.noise_bound, prm.gnc_factor, prm.cost_thr, prm.max_iter
    return p


def check_every_path(ctx, native, oracle, S, D, prm):
    n = len(S)
    o = oracle.quatro_solve(S, D, np.repeat(np.arange(n, dtype=np.int32)[:, None], 2, 1), oracle_params(oracle, prm))
    paths = (["shared"] if n <= SHARED_CAP else []) + ["global", "wide"]
    got = {p: ctx.quatro_solve_tap(S, D, device_params(native, prm), path=p) for p in paths}
    for p, g in got.items():
        assert g["valid"] == o["valid"], p
        assert np.array_equal(g["clique"], o["clique"]), p
        assert g["clique_size"] == len(o["clique"]), p
        assert g["gnc_iterations"] == o["gnc_iters"], p
        assert np.abs(g["T"] - o["T"]).max() < 1e-9, (p, np.abs(g["T"] - o["T"]).max())
    first = got[paths[0]]
    for p, g in got.items():
        assert np.array_equal(g["clique"], first["clique"]) and g["gnc_iterations"] == first["gnc_iterations"], p
        assert np.abs(g["T"] - first["T"]).max() < 1e-12, (p, np.abs(g["T"] - first["T"]).max())
    return got, o


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_crafted_set_on_every_path(ctx, native, oracle, case):
    got, o = check_every_path(ctx, native, oracle, case.S, case.D, case.prm)
    valid, clique, iters, T = case.solve()
    assert o["valid"] == valid and np.array_equal(o["clique"], clique) and o["gnc_iters"] == iters
    if not valid:
        for g in got.values():
            assert np.array_equal(g["T"], np.eye(4))


@pytest.mark.parametrize("n", [2, 37, 256, 500, 512])
def test_random_sets_on_every_path(ctx, native, oracle, n):
    S, D = tr.natural_set(n, 7000 + n, noise=0.1, yaw=-2.5)
    got, _ = check_every_path(ctx, native, oracle, S, D, tr.Params(noise_bound=0.3))
    if n == SHARED_CAP:
        assert got["shared"]["valid"] and got["shared"]["clique_size"] >= n // 3


def test_shared_tap_rejects_513(ctx, native):
    S, D = tr.natural_set(SHARED_CAP + 1, 1)
    with pytest.raises(native.B200RegError):
        ctx.quatro_solve_tap(S, D, path="shared")


def _stage(ctx, srcs, dsts, prm):
    cl = ctx.create_clouds(srcs + dsts)
    try:
        infos = ctx.quatro_align(cl[:len(srcs)], cl[len(srcs):], params=prm, want_corr=True)
        feats = [ctx.get_fpfh(c)[1] for c in cl]
    finally:
        for c in cl:
            c.destroy()
    return infos, feats[:len(srcs)], feats[len(srcs):]


def _oracle_match_params(oracle, prm):
    p = oracle.QuatroParams.default()
    p.max_corres, p.tuple_scale, p.seed = prm.max_corres, prm.tuple_scale, prm.seed
    return p


@pytest.fixture(scope="module")
def pairs(synth):
    """Mixed sizes: the last pair is large enough that 509 correspondences survive even a 0.99 tuple test."""
    return [synth.make_pair(2000, 8000, 9000, mode="quatro")[:2], synth.make_pair(2005, 3000, 2500, mode="quatro")[:2],
            synth.make_pair(2004, 20000, 20000, mode="quatro")[:2], synth.make_pair(2004, 50000, 50000, mode="quatro")[:2]]


@pytest.mark.parametrize("max_corres,tuple_scale", [(1, 0.8), (1, 0.99), (509, 0.8), (509, 0.99)])
def test_tuple_test_and_solver_end_to_end(ctx, native, oracle, pairs, max_corres, tuple_scale):
    """Every pair in one batched call (several k_teaser_solve blocks per launch): the device correspondences equal
    oracle.match on the device's descriptors, order included, and the solve equals the oracle's; each pair alone gives
    the same bytes."""
    prm = native.default_quatro_params()
    prm.max_corres, prm.tuple_scale = max_corres, tuple_scale
    srcs, dsts = [p[0] for p in pairs], [p[1] for p in pairs]
    infos, fs, fd = _stage(ctx, srcs, dsts, prm)
    for k, info in enumerate(infos):
        corr, mutual = oracle.match(srcs[k], dsts[k], fs[k], fd[k], _oracle_match_params(oracle, prm))
        assert info["n_mutual"] == len(mutual), k
        assert np.array_equal(info["corr"], corr), k
        assert len(corr) <= max_corres + 3
        o = oracle.quatro_solve(srcs[k], dsts[k], corr)
        assert info["valid"] == o["valid"] and info["clique_size"] == len(o["clique"]), k
        assert info["gnc_iterations"] == o["gnc_iters"], k
        assert np.abs(info["T"] - o["T"]).max() < 1e-9, k
        alone = _stage(ctx, [srcs[k]], [dsts[k]], prm)[0][0]
        assert alone["T"].tobytes() == info["T"].tobytes() and np.array_equal(alone["corr"], info["corr"]), k
    if max_corres == 509:
        assert 510 <= infos[-1]["n_corr"] <= 512  # k_tuple_select's keys and the shared solver's slots run full
        assert len({i["n_corr"] for i in infos}) >= 3, "the batch is meant to mix set sizes"


def test_tuple_scale_zero(ctx, native, oracle, pairs):
    """optimizedMatching keeps nothing (invalid, identity; the shared solver sees n = 0); advancedMatching keeps every
    cross-checked pair."""
    src, dst = pairs[0]
    prm = native.default_quatro_params()
    prm.tuple_scale = 0.0
    (info,), (fs,), (fd,) = _stage(ctx, [src], [dst], prm)
    corr, mutual = oracle.match(src, dst, fs, fd, _oracle_match_params(oracle, prm))
    assert len(corr) == 0 and info["n_corr"] == 0 and info["n_mutual"] == len(mutual) > 100
    assert not info["valid"] and info["clique_size"] == 0 and np.array_equal(info["T"], np.eye(4))
    prm.use_optimized_matching = 0
    (info,), (fs,), (fd,) = _stage(ctx, [src], [dst], prm)
    keep = oracle.match_advanced(src, dst, fs, fd, _oracle_match_params(oracle, prm))
    assert np.array_equal(keep, oracle.match_advanced(src, dst, fs, fd, tuple_test=False))
    assert np.array_equal(info["corr"], keep) and info["n_corr"] == len(keep) > 0
    o = oracle.quatro_solve(src, dst, keep)
    assert info["valid"] == o["valid"] and info["gnc_iterations"] == o["gnc_iters"]
    assert np.abs(info["T"] - o["T"]).max() < 1e-9


def test_far_from_origin_matcher_equals_oracle(ctx, native, oracle, synth):
    """Pairs 3.6 km from the map origin: the device's fp64 mean differs from the reference's fp32 running sum by
    centimetres, and the correspondences still equal the oracle's (see test_tuple_reference.py)."""
    shift = np.array([3000.0, -2000.0, 50.0])
    src, dst, _ = synth.make_pair(2005, 8000, 9000, mode="quatro")
    src, dst = src.copy(), dst.copy()
    for a in (src, dst):
        a[:, :3] = (a[:, :3].astype(np.float64) + shift).astype(np.float32)
    prm = native.default_quatro_params()
    (info,), (fs,), (fd,) = _stage(ctx, [src], [dst], prm)
    corr, mutual = oracle.match(src, dst, fs, fd)
    assert info["n_mutual"] == len(mutual) and np.array_equal(info["corr"], corr) and len(corr) > 0
