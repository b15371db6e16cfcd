"""The feature matcher alone (b200reg_match_tap: k_load_records, k_fcode, the radix sort, k_fgather, k_feat_nn both ways,
k_first_hit, k_mutual) against the exact fp32 restatement of tests/match_ref.py, on nn, dis (bits, where nn >= 0), rnn and
the mutual list in its order, in optimizedMatching's and advancedMatching's modes: device FPFH of raw and voxelised scans
(100k points), and crafted descriptors at the kernel's edges (exact ties across tiles, near-tight projected bounds,
one-hot extremes, the gate, identical runs across tiles and sort-key collisions, unusable rows, partial tiles and blocks)."""
import time

import numpy as np
import pytest

import match_ref as M

pytestmark = pytest.mark.gpu


def check(got, want, name=""):
    assert np.array_equal(got["nn"], want["nn"]), (name, np.flatnonzero(got["nn"] != want["nn"])[:8])
    on = want["nn"] >= 0
    assert np.array_equal(got["dis"][on].view(np.uint32), want["dis"][on].view(np.uint32)), name
    assert np.array_equal(got["rnn"], want["rnn"]), (name, np.flatnonzero(got["rnn"] != want["rnn"])[:8])
    assert np.array_equal(got["mutual"], want["mutual"]), name


def run_both_modes(ctx, fi, fj, thrs=(35.0,), backend="numpy", name=""):
    out = {}
    for thr in thrs:
        got = ctx.match_tap([(fi, fj)], distance_threshold=thr)[0]
        check(got, M.match_ref(fi, fj, thr, backend=backend), "%s thr=%r" % (name, thr))
        out[thr] = got
    got = ctx.match_tap([(fi, fj)], advanced=True)[0]
    ref = M.match_ref(fi, fj, advanced=True, backend=backend)
    check(got, ref, name + " advanced")
    out["advanced"] = got
    return out, ref


def test_torch_reference_equals_numpy_bitwise():
    """The torch backend (used at 100k x 100k) against numpy on a few hundred rows, ties included: a fused or flushed op
    would show here, not be blamed on the kernel."""
    rng = np.random.default_rng(11)
    fi, fj = M.tie_lattice(7, n_centres=3)
    fi = np.concatenate([fi[:300], M.random_desc(rng, 100), M.one_hot_extremes()[:100],
                         (M.random_desc(rng, 100) * np.float32(0.37)).astype(np.float32)])
    fj = np.concatenate([fj, fi[rng.choice(len(fi), 150)], M.random_desc(rng, 100)])
    for adv in (False, True):
        a = M.match_ref(fi, fj, 7.0, advanced=adv)
        b = M.match_ref(fi, fj, 7.0, advanced=adv, backend="torch")
        for k in ("nn", "rnn", "mutual"):
            assert np.array_equal(a[k], b[k]), k
        assert np.array_equal(a["dis"].view(np.uint32), b["dis"].view(np.uint32))


RAW = [("raw_2000", dict(pair_seed=2000, voxel=None)), ("voxel0.3_2000", dict(pair_seed=2000, voxel=0.3)),
       ("voxel0.1_2003", dict(pair_seed=2003, voxel=0.1))]


@pytest.mark.parametrize("name,kw", RAW, ids=[r[0] for r in RAW])
def test_raw_density_matches_reference(ctx, native, synth, name, kw):
    t = time.time()
    src, dst, _ = synth.make_pair(kw["pair_seed"], 100000, 100000, mode="quatro", voxel=kw["voxel"])
    cl = ctx.create_clouds([src, dst])
    try:
        ctx.fpfh(cl)
        fs, fd = ctx.get_fpfh(cl[0])[1], ctx.get_fpfh(cl[1])[1]
        infos = {}
        for adv in (0, 1):
            prm = native.default_quatro_params()
            prm.use_optimized_matching = 1 - adv
            infos[adv] = ctx.quatro_align([cl[0]], [cl[1]], params=prm)[0]
    finally:
        for c in cl:
            c.destroy()
    fi, fj = (fd, fs) if len(dst) > len(src) else (fs, fd)  # the matcher's roles: fi the larger cloud
    # first, the torch reference against numpy on a few hundred of these very rows (ties included): a fused or flushed op
    # would show here and not be blamed on the kernel
    rng = np.random.default_rng(0)
    si, sj = fi[rng.choice(len(fi), 400)], fj[rng.choice(len(fj), 300)]
    si = np.concatenate([si, sj[:50]])  # exact matches and duplicate rows
    for adv in (False, True):
        a, b = M.match_ref(si, sj, advanced=adv), M.match_ref(si, sj, advanced=adv, backend="torch")
        assert all(np.array_equal(a[k], b[k]) for k in ("nn", "rnn", "mutual"))
        assert np.array_equal(a["dis"].view(np.uint32), b["dis"].view(np.uint32))
    out, ref = run_both_modes(ctx, fi, fj, backend="torch", name=name)
    # the tap is the production matcher: the same mutual count as quatro_align on the same clouds
    assert len(out[35.0]["mutual"]) == infos[0]["n_mutual"]
    assert len(out["advanced"]["mutual"]) == infos[1]["n_mutual"]
    cert = M.certify_fp64(fj, fi, M.usable(fi), ref["nn"].astype(np.int64), backend="torch")
    print("\n%s: %d x %d descriptors, %d mutual (optimized), %d (advanced); fp64 layer: %d winners, %d fp32-only "
          "(fp32 winner is not the fp64 argmin), largest fp64 gap among them %.3e (relative %.3e), largest gap / allowed "
          "%.3f; %.1f s" % (name, len(fi), len(fj), len(out[35.0]["mutual"]), len(out["advanced"]["mutual"]), cert["n"],
                            cert["differ"], cert["max_gap"], cert["max_rel_gap"], cert["max_ratio"], time.time() - t))


CRAFTED = M.crafted_cases()


@pytest.mark.parametrize("case", CRAFTED, ids=[c.name for c in CRAFTED])
def test_crafted_edges(ctx, case):
    run_both_modes(ctx, case.fi, case.fj, case.thrs, name=case.name)


def test_gate_overflow_keeps_every_pair(ctx, native, oracle, synth):
    """distance_threshold = 1e20: its fp32 square overflows to +inf, and the reference's `dis > thr * thr` drops nothing.
    The tap keeps every pair of the crafted gate case, and b200reg_quatro_align keeps the same mutual set as the tap and
    the oracle on a scan pair."""
    case = next(c for c in CRAFTED if c.name == "gate")
    got = ctx.match_tap([(case.fi, case.fj)], distance_threshold=1e20)[0]
    assert (got["nn"] >= 0).all() and len(got["mutual"]) == len(case.fj)
    rng = np.random.default_rng(4)
    src = rng.uniform(-20, 20, (len(case.fi), 3)).astype(np.float32)
    p = oracle.QuatroParams.default()
    p.distance_threshold = 1e20
    _, mutual = oracle.match(src, src[:len(case.fj)], case.fi, case.fj, p)
    assert np.array_equal(got["mutual"], mutual)
    # the production path: a gate that drops pairs at 1e-3 keeps them all at 1e20
    src, dst, _ = synth.make_pair(2005, 3000, 2500, mode="quatro")
    cl = ctx.create_clouds([src, dst])
    try:
        n = {}
        for thr in (1e-3, 1e20):
            prm = native.default_quatro_params()
            prm.distance_threshold = thr
            n[thr] = ctx.quatro_align([cl[0]], [cl[1]], params=prm)[0]["n_mutual"]
        fs, fd = ctx.get_fpfh(cl[0])[1], ctx.get_fpfh(cl[1])[1]
    finally:
        for c in cl:
            c.destroy()
    tap = ctx.match_tap([(fs, fd)], distance_threshold=1e20)[0]  # src is the larger cloud: fi
    p.distance_threshold = 1e20
    _, mutual = oracle.match(src, dst, fs, fd, p)
    assert n[1e20] == len(tap["mutual"]) == len(mutual) > n[1e-3]


SIZES = M.size_cases()


@pytest.mark.parametrize("case", SIZES, ids=[c.name for c in SIZES])
def test_sizes_and_tile_counts(ctx, case):
    run_both_modes(ctx, case.fi, case.fj, name=case.name)


def test_batch_of_mixed_sizes_equals_each_pair_alone(ctx):
    cases = [c for c in CRAFTED + SIZES if c.name in ("tie_lattice_1", "gate", "unusable_mixed_and_whole_block",
                                                      "base_without_usable_rows", "n1_1", "n129_65", "tiles41", "tiles2")]
    assert len(cases) == 8
    for adv in (False, True):
        batch = ctx.match_tap([(c.fi, c.fj) for c in cases], advanced=adv)
        for c, b in zip(cases, batch):
            alone = ctx.match_tap([(c.fi, c.fj)], advanced=adv)[0]
            for k in ("nn", "dis", "rnn", "mutual"):
                assert alone[k].tobytes() == b[k].tobytes(), (c.name, k, adv)


def test_tap_rejects_a_larger_query_set(ctx, native):
    f = M.random_desc(np.random.default_rng(0), 10)
    with pytest.raises(native.B200RegError):
        ctx.match_tap([(f[:5], f)])
