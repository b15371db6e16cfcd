"""optimizedMatching with max_corres above 509 (up to 8189 = B200REG_ADV_CORR_CAPACITY - 3).

The tuple test keeps at most max_corres + 3 correspondences.  Sets of at most 512 are solved by k_teaser_solve in shared
memory as before; larger ones by the global-memory chain of advancedMatching, all such pairs of a call in one batch.
Every answer is compared with the CPU oracle on the device's own descriptors, and each pair of a batch with the same
pair solved alone.

Pairs: a small synthetic pair (its set stays below 512 at any cap), a 50k x 50k synthetic pair (2912 mutual matches;
2748 survive a 0.8 tuple test, 1629 a 0.99 one) and the 0.2 m sub-map pair of test_gpu_quatro_big.py (about 14 830
mutual matches; a 0.8 tuple test passes more than 8189 of them, a 0.99 one about 2200).  Counts are the oracle's on its
own descriptors; the device's differ by a few.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_quatro_big import make_submap_pair

pytestmark = pytest.mark.gpu
SHARED_CAP = 512         # B200REG_CORR_CAPACITY: k_teaser_solve's largest set, corr_out's stride
OPT_MAX = 8189           # B200REG_ADV_CORR_CAPACITY - 3
EINVAL, ECUDA, ESTATE = -1, -2, -4


@pytest.fixture(scope="module")
def small(synth):
    return synth.make_pair(2005, 3000, 2500, mode="quatro")[:2]


@pytest.fixture(scope="module")
def p50k(synth):
    return synth.make_pair(2004, 50000, 50000, mode="quatro")[:2]


@pytest.fixture(scope="module")
def submap():
    return make_submap_pair(leaf=0.2)[:2]


def _params(native, max_corres, tuple_scale=0.95):
    prm = native.default_quatro_params()
    prm.max_corres, prm.tuple_scale = max_corres, tuple_scale
    return prm


def _oracle_params(oracle, prm):
    p = oracle.QuatroParams.default()
    p.max_corres, p.tuple_scale, p.seed = prm.max_corres, prm.tuple_scale, prm.seed
    return p


def _stage(ctx, srcs, dsts, prm):
    """One batched call (correspondences as CSR through b200reg_quatro_align_ex) and the device descriptors."""
    cl = ctx.create_clouds(srcs + dsts)
    try:
        infos = ctx.quatro_align(cl[:len(srcs)], cl[len(srcs):], params=prm, want_corr=True)
        feats = [ctx.get_fpfh(c)[1] for c in cl]
    finally:
        for c in cl:
            c.destroy()
    return infos, feats[:len(srcs)], feats[len(srcs):]


def _same(a, b):
    return (a["T"].tobytes() == b["T"].tobytes() and np.array_equal(a["corr"], b["corr"])
            and (a["valid"], a["n_mutual"], a["n_corr"], a["clique_size"], a["gnc_iterations"])
            == (b["valid"], b["n_mutual"], b["n_corr"], b["clique_size"], b["gnc_iterations"]))


@pytest.mark.parametrize("tuple_scale", [0.8, 0.99])
@pytest.mark.parametrize("max_corres", [510, 1000, 2000, OPT_MAX])
def test_large_sets_equal_oracle(ctx, native, oracle, small, p50k, submap, max_corres, tuple_scale):
    """Every pair of one batched call: correspondences equal oracle.match on the device's descriptors, order included;
    the solve equals oracle.quatro_solve; the pair alone gives the same bytes."""
    prm = _params(native, max_corres, tuple_scale)
    pairs = [small, p50k] + ([submap] if max_corres >= 2000 else [])
    srcs, dsts = [p[0] for p in pairs], [p[1] for p in pairs]
    infos, fs, fd = _stage(ctx, srcs, dsts, prm)
    for k, info in enumerate(infos):
        corr, mutual = oracle.match(srcs[k], dsts[k], fs[k], fd[k], _oracle_params(oracle, prm))
        assert info["n_mutual"] == len(mutual), k
        assert info["n_corr"] == len(corr) <= max_corres + 3, k
        assert np.array_equal(info["corr"], corr), k
        o = oracle.quatro_solve(srcs[k], dsts[k], corr)
        assert info["valid"] == o["valid"] and info["clique_size"] == len(o["clique"]), k
        assert info["gnc_iterations"] == o["gnc_iters"], k
        assert np.abs(info["T"] - o["T"]).max() < 1e-9, (k, np.abs(info["T"] - o["T"]).max())
        alone = _stage(ctx, [srcs[k]], [dsts[k]], prm)[0][0]
        assert _same(alone, info), k
    n = [i["n_corr"] for i in infos]
    # from 1000 on the batch mixes both solvers (at 510 these pairs keep 511 or 512: test_first_set_beyond_the_shared_solver
    # has a 513), and the sets the large path gets are the ones the cap asks for
    assert n[0] <= SHARED_CAP
    if max_corres >= 1000:
        assert n[1] > SHARED_CAP
    if max_corres < 2000 or (max_corres == 2000 and tuple_scale == 0.8):
        assert max_corres < n[1] <= max_corres + 3  # the 50k pair is cut at the cap
    if max_corres == 2000:
        assert max(n) > 2000
    if max_corres == OPT_MAX and tuple_scale == 0.8:
        assert 8190 <= n[2] <= 8192  # the sort and the batched solver run full
    if max_corres == OPT_MAX and tuple_scale == 0.99:
        assert n[2] > 2000


def test_first_set_beyond_the_shared_solver(ctx, native, oracle, synth):
    """At max_corres 510 the last trial can add three new correspondences: a set of 513, the smallest one the shared
    solver cannot hold, goes to the global-memory chain and equals the oracle.  The tuple test's seed is scanned (20k
    pair, tuple_scale 0.8) for the first such set."""
    src, dst = synth.make_pair(2004, 20000, 20000, mode="quatro")[:2]
    prm = _params(native, 510, 0.8)
    cs, cd = ctx.create_clouds([src, dst])
    try:
        for seed in range(1, 400):
            prm.seed = seed
            if ctx.quatro_align([cs], [cd], params=prm)[0]["n_corr"] == SHARED_CAP + 1:
                break
        info = ctx.quatro_align([cs], [cd], params=prm, want_corr=True)[0]
        fs, fd = ctx.get_fpfh(cs)[1], ctx.get_fpfh(cd)[1]
    finally:
        cs.destroy(); cd.destroy()
    corr, _ = oracle.match(src, dst, fs, fd, _oracle_params(oracle, prm))
    assert info["n_corr"] == len(corr) == SHARED_CAP + 1
    assert np.array_equal(info["corr"], corr)
    o = oracle.quatro_solve(src, dst, corr)
    assert info["valid"] == o["valid"] and info["clique_size"] == len(o["clique"])
    assert info["gnc_iterations"] == o["gnc_iters"]
    assert np.abs(info["T"] - o["T"]).max() < 1e-9


def test_mixed_batch_each_pair_as_alone(ctx, native, synth, small, p50k):
    """Sets of at most 512 and larger ones in one call, in both clouds' orders, repeated: each pair gets its single-call
    bytes."""
    mid = synth.make_pair(2004, 20000, 20000, mode="quatro")[:2]
    pairs = [p50k, small, (p50k[1], p50k[0]), mid, small]
    srcs, dsts = [p[0] for p in pairs], [p[1] for p in pairs]
    prm = _params(native, 1000)
    runs = [_stage(ctx, srcs, dsts, prm)[0] for _ in range(2)]
    alone = [_stage(ctx, [s], [d], prm)[0][0] for s, d in zip(srcs, dsts)]
    n = [i["n_corr"] for i in runs[0]]
    assert n[0] > SHARED_CAP and n[2] > SHARED_CAP and n[1] <= SHARED_CAP
    for run in runs:
        for k in range(len(pairs)):
            assert _same(run[k], alone[k]), k


def _align_raw(native, ctx, cs, cd, prm, fixed=False):
    """b200reg_quatro_align with corr_out NULL, or (fixed) a count x B200REG_CORR_CAPACITY-pair buffer."""
    cnt = len(cs)
    sa = (C.c_void_p * cnt)(*[c.h for c in cs])
    da = (C.c_void_p * cnt)(*[c.h for c in cd])
    info = (native.QuatroInfo * cnt)()
    buf = np.full((cnt, SHARED_CAP, 2), -7, np.int32) if fixed else None
    rc = native.lib().b200reg_quatro_align(ctx.h, cnt, sa, da, C.byref(prm), info,
                                           None if buf is None else buf.ctypes.data_as(C.c_void_p))
    return rc, [i.as_dict() for i in info], buf


def _align_ex(native, ctx, cs, cd, prm, capacity):
    cnt = len(cs)
    sa = (C.c_void_p * cnt)(*[c.h for c in cs])
    da = (C.c_void_p * cnt)(*[c.h for c in cd])
    info = (native.QuatroInfo * cnt)()
    offsets = np.full(cnt + 1, -7, np.int64)
    corr = np.full((max(capacity, 1), 2), -7, np.int32)
    rc = native.lib().b200reg_quatro_align_ex(ctx.h, cnt, sa, da, C.byref(prm), info, offsets.ctypes.data_as(C.c_void_p),
                                              C.c_size_t(capacity), corr.ctypes.data_as(C.c_void_p))
    return rc, [i.as_dict() for i in info], offsets, corr


def test_abi_edges(ctx, native, oracle, small, p50k):
    """8189 is taken and 8190 refused; a fixed-stride corr_out refuses a set beyond 512 naming the pair and the count
    and still serves smaller sets; _ex returns any count as CSR, equal to the oracle."""
    cl = ctx.create_clouds([small[0], p50k[0], small[1], p50k[1]])
    cs, cd = cl[:2], cl[2:]
    try:
        assert _align_raw(native, ctx, cs, cd, _params(native, OPT_MAX))[0] == 0
        for bad in (OPT_MAX + 1, 10000, 0):
            assert _align_raw(native, ctx, cs, cd, _params(native, bad))[0] == EINVAL, bad
        assert "1..8189" in native.lib().b200reg_last_error().decode()
        prm = _params(native, 1000)
        rc, infos, _ = _align_raw(native, ctx, cs, cd, prm)
        assert rc == 0 and infos[0]["n_corr"] <= SHARED_CAP < infos[1]["n_corr"]
        n1 = infos[1]["n_corr"]
        rc, _, _ = _align_raw(native, ctx, cs, cd, prm, fixed=True)
        assert rc == ESTATE
        msg = native.lib().b200reg_last_error().decode()
        assert "pair 1" in msg and str(n1) in msg, msg
        # the same stride serves the pair whose set fits, with the bytes of the CSR call
        rc, (i_fix,), buf = _align_raw(native, ctx, cs[:1], cd[:1], prm, fixed=True)
        total = sum(i["n_corr"] for i in infos)
        rc_ex, i_ex, off, corr = _align_ex(native, ctx, cs, cd, prm, total)
        assert rc == 0 and rc_ex == 0
        assert list(off) == [0, infos[0]["n_corr"], total]
        assert np.array_equal(buf[0][:i_fix["n_corr"]], corr[:off[1]])
        assert i_fix["T"].tobytes() == i_ex[0]["T"].tobytes() == infos[0]["T"].tobytes()
        assert i_ex[1]["T"].tobytes() == infos[1]["T"].tobytes()
        fs, fd = ctx.get_fpfh(cs[1])[1], ctx.get_fpfh(cd[1])[1]
        oc, _ = oracle.match(p50k[0], p50k[1], fs, fd, _oracle_params(oracle, prm))
        assert np.array_equal(corr[off[1]:off[2]], oc)
        rc, _, off2, corr2 = _align_ex(native, ctx, cs, cd, prm, total - 1)
        assert rc == ESTATE and list(off2) == list(off) and (corr2 == -7).all()
    finally:
        for c in cl:
            c.destroy()


def test_launch_counts(ctx, native, small, p50k):
    """Up to 509 the call launches what it launched before (509 = 200 for one pair); above it, a call with a set beyond
    512 adds one gather and the five kernels of the batched solve, once for the whole batch."""
    cl = ctx.create_clouds([small[0], p50k[0], small[1], p50k[1]])
    cs, cd = cl[:2], cl[2:]

    def launches(prm, s, d):
        before = ctx.launch_count
        rc, infos, _ = _align_raw(native, ctx, s, d, prm)
        assert rc == 0
        return ctx.launch_count - before, infos
    try:
        ctx.fpfh(cl)  # descriptors first: the counts below are the matcher's and the solver's only
        base, _ = launches(_params(native, 200), cs[1:], cd[1:])
        assert launches(_params(native, 509), cs[1:], cd[1:])[0] == base
        l_small, i_small = launches(_params(native, 1000), cs[:1], cd[:1])
        assert i_small[0]["n_corr"] <= SHARED_CAP and l_small == base
        l_big, i_big = launches(_params(native, 1000), cs[1:], cd[1:])
        assert i_big[0]["n_corr"] > SHARED_CAP and l_big == base + 6
        l_two, _ = launches(_params(native, 1000), [cs[1], cs[1]], [cd[1], cd[1]])
        assert l_two == base + 6
    finally:
        for c in cl:
            c.destroy()


def test_loop_closure_at_2000_coarse_stage_equals_quatro_align(ctx, native, p50k):
    """b200reg_loop_closure passes max_corres through: its coarse stage equals b200reg_quatro_align on the same clouds."""
    src, dst = p50k
    prm = _params(native, 2000)
    (q_al,) = _stage(ctx, [src], [dst], prm)[0]
    _, (q_lc,) = ctx.loop_closure([src], [dst], qparams=prm)
    assert q_al["n_corr"] > SHARED_CAP and q_al["valid"]
    for key in ("valid", "n_mutual", "n_corr", "clique_size", "gnc_iterations"):
        assert q_lc[key] == q_al[key], key
    assert np.asarray(q_lc["T"]).tobytes() == q_al["T"].tobytes()


def test_perform_loop_closure_at_2000_coarse_stage_equals_quatro_align(ctx, native, p50k):
    """b200reg_perform_loop_closure (keyframe store, voxel_res 0.05): its coarse stage equals b200reg_quatro_align on
    the clouds the store assembles for the same pair."""
    import b200reg
    src, dst = p50k
    cfg = b200reg.default_loop_config()
    cfg.voxel_res = 0.05
    cfg.quatro.max_corres = 2000
    kf = ctx.keyframes()
    try:
        kf.add(dst, np.eye(4), 0.0)
        kf.add(src, np.eye(4), 100.0)
        q, closest = np.array([1], np.int32), np.array([0], np.int32)
        _, (q_pl,) = kf.perform_loop_closure(q, closest, cfg)
        cs, cd = kf.assemble(q, closest, cfg, n_keyframes=q + 1)
        try:
            rc, (q_al,), _ = _align_raw(native, ctx, cs, cd, cfg.quatro)
        finally:
            for c in cs + cd:
                c.destroy()
    finally:
        kf.destroy()
    assert rc == 0 and q_al["n_corr"] > SHARED_CAP and q_al["valid"]
    for key in ("valid", "n_mutual", "n_corr", "clique_size", "gnc_iterations"):
        assert q_pl[key] == q_al[key], key
    assert np.asarray(q_pl["T"]).tobytes() == np.asarray(q_al["T"]).tobytes()
