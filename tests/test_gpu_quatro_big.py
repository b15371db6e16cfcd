"""advancedMatching sets larger than B200REG_ADV_CORR_CAPACITY (8192): solved on the device, equal to the CPU oracle.

Synthetic sets of n correspondences (a known rigid motion on some, random pairs on the rest) go through the solve tap
on both solver paths; one sub-map pair whose surviving set exceeds 8192 goes through the whole Quatro stage, the C ABI
contract and coarse-to-fine.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ADV_CAP = 8192


def synthetic_set(n, seed=0, n_in=300):
    """n correspondences: n_in inliers (dst = yaw-rotated, shifted src plus 2 cm of noise), the rest random pairs in a
    120 x 120 x 12 m box.  Returns (src (n, 4), dst (n, 4), T_expected) as float32 records."""
    rng = np.random.default_rng(seed)
    S = rng.uniform([-60, -60, -3], [60, 60, 9], (n, 3))
    D = rng.uniform([-60, -60, -3], [60, 60, 9], (n, 3))
    yaw = 0.3
    R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    t = np.array([4.0, -2.5, 0.4])
    inl = rng.choice(n, n_in, replace=False)
    D[inl] = S[inl] @ R.T + t + rng.uniform(-0.02, 0.02, (n_in, 3))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    pad = np.zeros((n, 1))
    return np.c_[S, pad].astype(np.float32), np.c_[D, pad].astype(np.float32), T


def _pose_at(synth, sarc, half=100.0, r=1.8):
    """The keyframe poses of synth.make_sequence: laps of a two-lane street with U-turns at both ends."""
    lap = 4 * half + 2 * np.pi * r
    u = sarc % lap
    if u < 2 * half:
        x, y, yaw = -half + u, -r, 0.0
    elif u < 2 * half + np.pi * r:
        a = (u - 2 * half) / r
        x, y, yaw = half + r * np.sin(a), -r * np.cos(a), a
    elif u < 4 * half + np.pi * r:
        x, y, yaw = half - (u - 2 * half - np.pi * r), r, np.pi
    else:
        a = (u - 4 * half - np.pi * r) / r
        x, y, yaw = -half - r * np.sin(a), r * np.cos(a), np.pi + a
    return synth.se3(yaw=yaw, t=(x, y, 1.73))


def make_submap_pair(seed=7, k0=40, leaf=0.2):
    """enable_submap_matching sub-maps of 11 keyframes (+-5) at the same place one lap apart, voxelised at `leaf`, both
    at their true poses, so registration must return the identity.  Returns (src, dst, I).  At leaf 0.2 m about 9000
    correspondences survive advancedMatching (0.3 m gives about 4700).  Displacing the source by even 1.5 deg / 0.7 m
    drops that to about 3800: normals are flipped towards the origin, so the descriptors change with the pose."""
    from b200reg import synth
    lap_kf = int(round((400 + 2 * np.pi * 1.8) / 0.8))

    def submap(kc):
        poses = [_pose_at(synth, k * 0.8) for k in range(kc - 5, kc + 6)]
        pts = [synth.to_map_frame(synth.scan(seed, 7919 * seed + k, P, 30000), P) for k, P in zip(range(kc - 5, kc + 6), poses)]
        return synth.voxelize(np.concatenate(pts), leaf)
    return submap(k0 + lap_kf), submap(k0), np.eye(4)


def _adv_params(native):
    prm = native.default_quatro_params()
    prm.use_optimized_matching = 0
    return prm


def _corr_of(n):
    return np.repeat(np.arange(n, dtype=np.int32)[:, None], 2, 1)


@pytest.mark.parametrize("n", [6000, 8192, 8193, 12000, 24000])
def test_solver_equals_oracle_at_scale(ctx, oracle, synth, n):
    S, D, Texp = synthetic_set(n, seed=n)
    g = ctx.quatro_solve_tap(S, D, wide=n > ADV_CAP)
    o = oracle.quatro_solve(S, D, _corr_of(n))
    assert g["valid"] == o["valid"] and g["valid"]
    assert np.array_equal(g["clique"], o["clique"])
    assert g["clique_size"] == len(o["clique"]) >= 300
    assert g["gnc_iterations"] == o["gnc_iters"]
    assert np.abs(g["T"] - o["T"]).max() < 1e-9
    rot, tr = synth.se3_error(g["T"], Texp)
    assert rot < 1e-2 and tr < 0.1
    if n <= ADV_CAP:  # both solver paths: the same bytes
        w = ctx.quatro_solve_tap(S, D, wide=True)
        assert w["T"].tobytes() == g["T"].tobytes()
        assert np.array_equal(w["clique"], g["clique"])
        assert (w["valid"], w["gnc_iterations"]) == (g["valid"], g["gnc_iterations"])


def test_solver_tap_rejects_bad_sizes(ctx, native):
    S, D, _ = synthetic_set(ADV_CAP + 1)
    with pytest.raises(native.B200RegError):
        ctx.quatro_solve_tap(S, D, wide=False)


@pytest.fixture(scope="module")
def big_pair():
    return make_submap_pair()


@pytest.fixture(scope="module")
def big_stage(ctx, native, big_pair):
    src, dst, _ = big_pair
    cs, cd = ctx.create_clouds([src, dst])
    info = ctx.quatro_align([cs], [cd], params=_adv_params(native), want_corr=True)[0]
    _, fs = ctx.get_fpfh(cs)
    _, fd = ctx.get_fpfh(cd)
    cs.destroy(); cd.destroy()
    return info, fs, fd


def test_end_to_end_beyond_the_cap_equals_oracle(oracle, synth, big_pair, big_stage):
    src, dst, Texp = big_pair
    info, fs, fd = big_stage
    corr = oracle.match_advanced(src, dst, fs, fd)
    assert len(corr) > ADV_CAP
    assert info["n_corr"] == len(corr)
    assert np.array_equal(info["corr"], corr)
    o = oracle.quatro_solve(src, dst, corr)
    assert info["valid"] == o["valid"] and info["valid"]
    assert info["clique_size"] == len(o["clique"])
    assert info["gnc_iterations"] == o["gnc_iters"]
    assert np.abs(info["T"] - o["T"]).max() < 1e-9
    rot, tr = synth.se3_error(info["T"], Texp)
    assert rot < 0.06 and tr < 3.5


def test_loop_closure_beyond_the_cap_lands_on_the_truth(ctx, synth, native, big_pair, big_stage):
    src, dst, Texp = big_pair
    (r,), (q,) = ctx.loop_closure([src], [dst], qparams=_adv_params(native))
    assert q["n_corr"] == big_stage[0]["n_corr"] > ADV_CAP
    assert q["valid"] and r["converged"]
    rot, tr = synth.se3_error(r["T"], Texp)
    assert rot < 5e-3 and tr < 5e-2, (rot, tr)


def _align(native, ctx, clouds_s, clouds_d, prm, corr_fixed=False, ex=None):
    """Raw C calls: b200reg_quatro_align (corr_fixed: with a count x 8192-pair buffer) or, with ex = capacity,
    b200reg_quatro_align_ex.  Returns (rc, infos, offsets, corr)."""
    cnt = len(clouds_s)
    sa = (C.c_void_p * cnt)(*[c.h for c in clouds_s])
    da = (C.c_void_p * cnt)(*[c.h for c in clouds_d])
    info = (native.QuatroInfo * cnt)()
    if ex is None:
        buf = np.zeros((cnt, ADV_CAP, 2), np.int32) if corr_fixed else None
        rc = native.lib().b200reg_quatro_align(ctx.h, cnt, sa, da, C.byref(prm), info,
                                               None if buf is None else buf.ctypes.data_as(C.c_void_p))
        return rc, [i.as_dict() for i in info], None, buf
    offsets = np.full(cnt + 1, -7, np.int64)
    corr = np.full((max(ex, 1), 2), -7, np.int32)
    rc = native.lib().b200reg_quatro_align_ex(ctx.h, cnt, sa, da, C.byref(prm), info, offsets.ctypes.data_as(C.c_void_p),
                                              C.c_size_t(ex), corr.ctypes.data_as(C.c_void_p))
    return rc, [i.as_dict() for i in info], offsets, corr


def test_abi_contract_beyond_the_cap(ctx, native, big_pair, big_stage):
    src, dst, _ = big_pair
    info0 = big_stage[0]
    n = info0["n_corr"]
    prm = _adv_params(native)
    cs, cd = ctx.create_clouds([src, dst])
    try:
        rc, _, _, _ = _align(native, ctx, [cs], [cd], prm, corr_fixed=True)
        assert rc == native.ESTATE  # the fixed-stride buffer cannot hold the set
        rc, (i_null,), _, _ = _align(native, ctx, [cs], [cd], prm)
        assert rc == 0 and i_null["n_corr"] == n
        rc, (i_ex,), off, corr = _align(native, ctx, [cs], [cd], prm, ex=n)
        assert rc == 0 and list(off) == [0, n]
        assert i_null["T"].tobytes() == i_ex["T"].tobytes() == info0["T"].tobytes()
        assert np.array_equal(corr, info0["corr"])
        rc, _, off, corr = _align(native, ctx, [cs], [cd], prm, ex=n - 1)
        assert rc == native.ESTATE and list(off) == [0, n]
        assert (corr == -7).all(), "nothing but the offsets is written when the capacity is too small"
    finally:
        cs.destroy(); cd.destroy()


def test_batch_mixing_small_and_large_sets(ctx, synth, native, big_pair, big_stage):
    """Pairs below and above the cap in one call: each pair's answer equals solving it alone; repeated calls agree."""
    small = [synth.make_pair(2010 + i, 30000, 30000, mode="quatro", voxel=0.3)[:2] for i in range(2)]
    srcs = [small[0][0], big_pair[0], small[1][0], big_pair[1]]
    dsts = [small[0][1], big_pair[1], small[1][1], big_pair[0]]  # the last pair is the large one swapped
    prm = _adv_params(native)
    cl = ctx.create_clouds(srcs + dsts)
    cs, cd = cl[:4], cl[4:]
    try:
        runs = [ctx.quatro_align(cs, cd, params=prm, want_corr=True) for _ in range(2)]
        alone = [ctx.quatro_align([cs[i]], [cd[i]], params=prm, want_corr=True)[0] for i in range(4)]
    finally:
        for c in cl:
            c.destroy()
    assert runs[0][1]["n_corr"] > ADV_CAP and runs[0][3]["n_corr"] > ADV_CAP
    assert runs[0][0]["n_corr"] <= ADV_CAP and runs[0][2]["n_corr"] <= ADV_CAP
    back = runs[0][3]["corr"][:, ::-1]  # (src, dst) of the unswapped pair, sorted again
    assert np.array_equal(back[np.lexsort((back[:, 1], back[:, 0]))], big_stage[0]["corr"])
    for i in range(4):
        for run in runs:
            a, b = run[i], alone[i]
            assert a["T"].tobytes() == b["T"].tobytes(), i
            assert np.array_equal(a["corr"], b["corr"]), i
            assert (a["valid"], a["n_corr"], a["clique_size"], a["gnc_iterations"]) == \
                   (b["valid"], b["n_corr"], b["clique_size"], b["gnc_iterations"]), i
