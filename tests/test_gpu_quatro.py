"""GPU parity tests for the Quatro half: each stage isolated against the CPU oracle, then end to end.

The reference stage is nondeterministic (time-seeded rand(), racy TBB), so the bar is the oracle with a
fixed counter-based generator; the end-to-end bar is the SE(3) AFTER the Nano-GICP refinement
(SURVEY.md §8c iii): 1e-4 rad / 1e-3 m.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROT_TOL, TRANS_TOL = 1e-4, 1e-3


@pytest.fixture(scope="module")
def qpair(synth):
    return synth.make_pair(2000, 8000, 9000, mode="quatro")


def test_normals_and_fpfh_match_oracle(ctx, oracle, qpair):
    src, dst, _ = qpair
    cl, = ctx.create_clouds([dst])
    ctx.fpfh([cl], 0.9, 1.5)
    gn, gf = ctx.get_fpfh(cl)
    on, osp, of = oracle.fpfh(dst, 0.9, 1.5)
    assert np.array_equal(np.isnan(gn[:, 0]), np.isnan(on[:, 0]))
    ok = ~np.isnan(on[:, 0])
    # same flip rule on both sides: normals agree including sign, up to fp64 eigen-solver round-off; a handful of
    # near-isotropic neighbourhoods (two equal small eigenvalues) are ill-conditioned
    dots = np.einsum("ij,ij->i", gn[ok], on[ok])
    assert np.quantile(dots, 0.01) > 1 - 1e-6
    assert (dots > 0.999).mean() > 0.995
    # FPFH, stage-isolated (SURVEY §8(c)(iii): <= 1e-3 abs per bin): the GPU's OWN normals through the oracle's SPFH/FPFH.
    # What is left is the fp32 summation order (tree-walk order vs the oracle's sorted order): EVERY bin of EVERY point
    # within 1e-3 (profiles/diag_fpfh.py measures the deviation).
    _, of2 = oracle.fpfh_from_normals(dst, np.where(np.isnan(gn), np.nan, gn), 1.5)
    err2 = np.abs(gf - of2).max(1)
    assert err2.max() < 1e-3, np.quantile(err2, [0.5, 0.9, 0.99, 1.0])
    # complete pipelines (each side with its own normals): identical to 1e-3 per bin except where a fp64 eigen-solver
    # round-off flips a float normal in an ill-conditioned (near-isotropic / collinear) neighbourhood; such a point changes
    # the SPFH of everything within the FPFH radius and through it the FPFH within twice the radius -- nowhere else.
    err = np.abs(gf - of).max(1)
    assert np.quantile(err, 0.98) < 1e-3, np.quantile(err, [0.5, 0.98, 0.999, 1.0])
    bad_n = np.flatnonzero(~ok | (gn != on).any(1))  # any float difference of a normal can move a pair feature across a bin edge
    off = np.flatnonzero(err > 1e-3)
    if len(off):
        assert len(bad_n) > 0
        d = np.linalg.norm(dst[off, None, :3] - dst[None, bad_n, :3], axis=2).min(1)
        assert d.max() <= 2 * 1.5 + 1e-3, "an FPFH deviation away from any differing normal"
    # structure: each 11-bin block sums to 100 (or the descriptor is all zero)
    sums = gf.reshape(-1, 3, 11).sum(2)
    nz = np.abs(gf).sum(1) > 0
    assert np.allclose(sums[nz], 100.0, atol=2e-2)
    cl.destroy()


def _gpu_stage(ctx, src, dst, prm=None):
    cs, cd = ctx.create_clouds([src, dst])
    info = ctx.quatro_align([cs], [cd], params=prm, want_corr=True)[0]
    _, fs = ctx.get_fpfh(cs)
    _, fd = ctx.get_fpfh(cd)
    cs.destroy(); cd.destroy()
    return info, fs, fd


def test_matching_equals_oracle_on_same_descriptors(ctx, oracle, qpair):
    src, dst, _ = qpair
    info, fs, fd = _gpu_stage(ctx, src, dst)
    corr, mutual = oracle.match(src, dst, fs, fd)  # the GPU's descriptors through the CPU matcher
    assert info["n_mutual"] == len(mutual)
    assert info["n_corr"] == len(corr)
    assert np.array_equal(info["corr"], corr), "final correspondences (order included) must equal the oracle's"
    assert 0 < len(corr) <= 203


def test_matching_swapped_clouds(ctx, oracle, qpair):
    """dst larger than src: fi/fj swap (matcher.cc:364-369); output pairs stay (src, dst)."""
    src, dst, _ = qpair
    assert len(dst) > len(src)
    info, fs, fd = _gpu_stage(ctx, dst, src)  # now the FIRST cloud is the larger one: no swap
    corr, _ = oracle.match(dst, src, fs, fd)
    assert np.array_equal(info["corr"], corr)


def test_solver_equals_oracle_on_same_correspondences(ctx, oracle, synth, qpair):
    src, dst, Texp = qpair
    info, _, _ = _gpu_stage(ctx, src, dst)
    o = oracle.quatro_solve(src, dst, info["corr"])
    assert info["valid"] == o["valid"]
    assert info["clique_size"] == len(o["clique"])
    assert info["gnc_iterations"] == o["gnc_iters"]
    assert np.abs(info["T"] - o["T"]).max() < 1e-9
    # yaw-only rotation (SURVEY A.8 viii)
    assert info["T"][2, 2] == 1.0 and info["T"][0, 2] == 0.0 and info["T"][2, 0] == 0.0
    rot, tr = synth.se3_error(info["T"], Texp)
    assert rot < 0.06 and tr < 3.5  # coarse stage only: GICP absorbs the rest


def _adv_params(native):
    prm = native.default_quatro_params()
    prm.use_optimized_matching = 0
    return prm


@pytest.mark.parametrize("case", ["small", "small_swapped", "beyond_512", "thousands"])
def test_advanced_matching_and_big_solver_equal_oracle(ctx, oracle, synth, native, qpair, case):
    """Matcher::advancedMatching (matcher.cc:118-356) + the global-memory TEASER++ solve: the final correspondence
    list is bit-identical to the oracle's on the same descriptors (below and above the 512-entry shared-memory
    solver's capacity), clique size / GNC iterations equal, T to 1e-9."""
    if case == "small":
        src, dst, Texp = qpair
    elif case == "small_swapped":
        dst, src, Texp = qpair  # first cloud smaller: fi/fj swap inside the matcher (matcher.cc:125-130)
        Texp = np.linalg.inv(Texp)
    elif case == "beyond_512":
        src, dst, Texp = synth.make_pair(2002, 100000, 100000, mode="quatro", voxel=0.2)
    else:
        src, dst, Texp = synth.make_pair(2003, 100000, 100000, mode="quatro", voxel=0.1)
    info, fs, fd = _gpu_stage(ctx, src, dst, _adv_params(native))
    corr = oracle.match_advanced(src, dst, fs, fd)
    assert info["n_corr"] == len(corr)
    assert np.array_equal(info["corr"], corr)
    if case == "beyond_512":
        assert len(corr) > 512
    if case == "thousands":
        assert len(corr) > 1500
    assert np.all(np.diff(corr[:, 0].astype(np.int64) * (1 << 32) + corr[:, 1]) > 0), "sorted, unique (matcher.cc:353-355)"
    o = oracle.quatro_solve(src, dst, corr)
    assert info["valid"] == o["valid"]
    assert info["clique_size"] == len(o["clique"])
    assert info["gnc_iterations"] == o["gnc_iters"]
    assert np.abs(info["T"] - o["T"]).max() < 1e-9
    rot, tr = synth.se3_error(info["T"], Texp)
    assert rot < 0.06 and tr < 3.5


def test_advanced_matching_batch_and_loop_closure(ctx, synth, native):
    """advancedMatching through the batched entry points: batch == single, and coarse-to-fine lands on the truth."""
    pairs = [synth.make_pair(2010 + i, 30000, 30000, mode="quatro", voxel=0.3) for i in range(3)]
    prm = _adv_params(native)
    res, qi = ctx.loop_closure([p[0] for p in pairs], [p[1] for p in pairs], qparams=prm)
    for i, (s, d, T) in enumerate(pairs):
        r1, q1 = ctx.loop_closure([s], [d], qparams=prm)
        assert np.array_equal(res[i]["T"], r1[0]["T"]) and qi[i]["n_corr"] == q1[0]["n_corr"]
        assert qi[i]["valid"] and res[i]["converged"]
        rot, tr = synth.se3_error(res[i]["T"], T)
        assert rot < 5e-3 and tr < 5e-2, (i, rot, tr)


def test_coarse_to_fine_matches_oracle(ctx, oracle, synth):
    """LoopClosure::coarseToFineAlignment.  Two statements:
    (a) fine stage on the SAME coarse transform agrees with the oracle to the parity bar (1e-4 rad / 1e-3 m);
    (b) the two complete pipelines (each with its own Quatro stage, whose descriptors differ by fp32 summation
        order) land within Nano-GICP's own stopping tolerance of each other and on the ground truth."""
    for seed in (2000, 2002):
        src, dst, Texp = synth.make_pair(seed, 8000, 8000, mode="quatro")
        res, qi = ctx.loop_closure([src], [dst])
        r, q = res[0], qi[0]
        assert q["valid"]
        o_same = oracle.coarse_to_fine(src, dst, quatro_T=q["T"])
        rot, tr = synth.se3_error(r["T"], o_same["T"])
        assert rot < ROT_TOL and tr < TRANS_TOL, (seed, rot, tr)
        assert r["converged"] == o_same["converged"] and r["n_linearize"] == o_same["gicp"]["n_linearize"]
        assert abs(r["fitness"] - o_same["fitness"]) < 1e-5 * max(o_same["fitness"], 1e-3)
        o = oracle.coarse_to_fine(src, dst)
        assert o["quatro"]["valid"]
        rot, tr = synth.se3_error(q["T"], o["quatro"]["T"])
        assert rot < 0.05 and tr < 1.5, ("coarse stages", rot, tr)
        rot, tr = synth.se3_error(r["T"], o["T"])
        assert rot < 2e-3 and tr < 1e-2, ("pipelines", rot, tr)  # rotation_eps 2e-3 / transformation_eps 1e-2
        rot, tr = synth.se3_error(r["T"], Texp)
        assert rot < 5e-3 and tr < 5e-2


def test_quatro_batch_equals_single_and_invalid_pairs(ctx, synth):
    pairs = [synth.make_pair(2100 + i, 5000 + 400 * i, 6000 - 300 * i, mode="quatro") for i in range(3)]
    # an unrelated pair of tiny random blobs: no correspondences -> invalid, Identity (quatro_module.cc:63-66)
    rng = np.random.default_rng(0)
    blob_a = rng.normal(0, 20, (300, 4)).astype(np.float32)
    blob_b = rng.normal(0, 20, (280, 4)).astype(np.float32)
    srcs = [p[0] for p in pairs] + [blob_a]
    dsts = [p[1] for p in pairs] + [blob_b]
    res, qi = ctx.loop_closure(srcs, dsts)
    res2, qi2 = ctx.loop_closure(srcs, dsts)
    for i in range(4):
        single, qs = ctx.loop_closure([srcs[i]], [dsts[i]])
        assert np.array_equal(res[i]["T"], single[0]["T"]) and np.array_equal(res[i]["T"], res2[i]["T"])
        assert qi[i]["n_corr"] == qs[0]["n_corr"] == qi2[i]["n_corr"]
    assert not qi[3]["valid"] and np.array_equal(qi[3]["T"], np.eye(4)) and not res[3]["valid"]


def test_isolated_points_normals_descriptors_and_matching(ctx, oracle, synth):
    """Points with fewer than 3 neighbours inside the normal radius (isolated returns): NaN normal, all-zero descriptor on
    both sides, and they take no part in the matching (the deliberate definition stated in DESIGN §6 / oracle_quatro.cpp --
    PCL would bin NaN-normal neighbours into bin 0 and FLANN would still match all-zero descriptors)."""
    src, dst, _ = synth.make_pair(2001, 6000, 6500, mode="quatro")
    lone = np.array([[200.0 + 10 * i, -150.0, 40.0, 0.5] for i in range(6)], np.float32)  # far from everything, 10 m apart
    dst2 = np.concatenate([dst[:3000], lone, dst[3000:]]).astype(np.float32)
    cl, = ctx.create_clouds([dst2])
    ctx.fpfh([cl], 0.9, 1.5)
    gn, gf = ctx.get_fpfh(cl)
    on, _, of = oracle.fpfh(dst2, 0.9, 1.5)
    idx = np.arange(3000, 3006)
    assert np.isnan(gn[idx]).all() and np.isnan(on[idx]).all()
    assert (gf[idx] == 0).all() and (of[idx] == 0).all()
    assert np.array_equal(np.isnan(gn[:, 0]), np.isnan(on[:, 0]))
    assert np.array_equal(np.abs(gf).sum(1) == 0, np.abs(of).sum(1) == 0)
    cl.destroy()
    # the matcher on the GPU's descriptors: same mutual set and correspondences as the oracle, no isolated point in either
    info, fs, fd = _gpu_stage(ctx, src, dst2)
    corr, mutual = oracle.match(src, dst2, fs, fd)
    assert info["n_mutual"] == len(mutual) and np.array_equal(info["corr"], corr)
    assert not np.isin(corr[:, 1], idx).any()


@pytest.mark.parametrize("mode", ["optimized", "advanced"])
def test_matching_with_runs_of_identical_descriptors(ctx, oracle, native, mode):
    """Noise-free planes: thousands of points share ONE bitwise-identical descriptor (runs far longer than a 64-record
    tile, runs cut by tile borders), next to a few hundred distinct ones.  The matcher collapses such runs to one base
    record that answers with the run's lowest original index (k_fgather); the correspondences must still equal the
    oracle's brute-force matcher on the same descriptors, order included."""
    rng = np.random.default_rng(5)

    def scene(shift):
        g = np.stack(np.meshgrid(np.arange(70) * 0.3, np.arange(70) * 0.3, indexing="ij"), -1).reshape(-1, 2)
        floor = np.c_[g, np.zeros(len(g))]
        wall = np.c_[g[:, 0], np.full(len(g), 21.0), g[:, 1] * 0.5 + 0.3]
        blob = rng.uniform(0, 1, (400, 3)) * [6.0, 6.0, 3.0] + [5.0, 8.0, 0.3]
        pts = np.concatenate([floor, wall, blob]) + shift
        return np.c_[pts, np.zeros(len(pts))].astype(np.float32)
    src = scene(np.array([-10.0, -12.0, -1.5]))
    dst = scene(np.array([-10.4, -11.7, -1.5]))[::-1].copy()  # other order: the lowest-index rule is exercised
    prm = native.default_quatro_params()
    prm.use_optimized_matching = 1 if mode == "optimized" else 0
    info, fs, fd = _gpu_stage(ctx, src, dst, prm)
    u = np.unique(fd[(fd != 0).any(1)], axis=0)
    assert (fd != 0).any(1).sum() - len(u) > 2000, "the scene is meant to produce long runs of identical descriptors"
    if mode == "optimized":
        corr, mutual = oracle.match(src, dst, fs, fd)
        assert info["n_mutual"] == len(mutual)
    else:
        corr = oracle.match_advanced(src, dst, fs, fd)
    assert info["n_corr"] == len(corr)
    assert np.array_equal(info["corr"], corr)
