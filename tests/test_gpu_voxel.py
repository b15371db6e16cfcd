"""The device pcl::VoxelGrid (k_voxel_keys -> 3 x 11-bit radix sort -> k_voxel_heads -> k_voxel_centroid) against the
oracle, bit for bit: the same voxel count, the same order and the same fp32 centroids.  Keyframes are stored with the
identity pose and assembled with enable_quatro=1, enable_submap_matching=0, so every job is one keyframe and the merged
cloud is the keyframe itself.  The inputs are the crafted clouds of voxel_cases.py, which test_oracle_crosschecks.py
pins to a numpy restatement of PCL (that test also records which of them reach keys above 2^28 or trip the guard)."""
import numpy as np
import pytest

import voxel_cases as vc

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _voxelize_on_device(ctx, clouds, leaf):
    """One assemble call over len(clouds) single-keyframe jobs -> the voxelised xyz of each, in voxel order."""
    import b200reg
    kf = ctx.keyframes()
    for k, c in enumerate(clouds):
        kf.add(c, np.eye(4), float(k))
    cfg = b200reg.default_loop_config()
    cfg.enable_quatro, cfg.enable_submap_matching, cfg.voxel_res = 1, 0, leaf
    idx = np.arange(len(clouds), dtype=np.int32)
    sc, dc = kf.assemble(idx, idx, cfg)
    out = []
    for s, d in zip(sc, dc):
        got = ctx.cloud_points(s)
        assert np.array_equal(_bits(got), _bits(ctx.cloud_points(d)))  # src and dst jobs of a pair are the same keyframe
        out.append(got)
    for c in sc + dc:
        c.destroy()
    kf.destroy()
    return out


def _assert_equals_oracle(oracle, got, cloud, leaf, name):
    want = oracle.voxelize(cloud, leaf)
    assert got.shape[0] == want.shape[0], (name, got.shape, want.shape)
    assert np.array_equal(_bits(got), _bits(want[:, :3])), name


@pytest.mark.parametrize("leaf", vc.SWEEP_LEAVES)
def test_leaf_sweep_on_sequence_keyframes(ctx, oracle, synth, leaf):
    """Keyframes 0 and 70 at 0.05 m have keys above 2^28: the third sort pass orders real digits."""
    seq = vc.sweep_sequence(synth)
    clouds = [seq["clouds"][k] + np.float32(0) for k in vc.SWEEP_KEYFRAMES]
    for k, c, got in zip(vc.SWEEP_KEYFRAMES, clouds, _voxelize_on_device(ctx, clouds, leaf)):
        _assert_equals_oracle(oracle, got, c, leaf, (k, leaf))


@pytest.mark.parametrize("leaf", (0.3, 0.1))
def test_cell_boundaries(ctx, oracle, leaf):
    c = vc.cell_boundaries(leaf, 11 if leaf == 0.3 else 12)
    got, = _voxelize_on_device(ctx, [c], leaf)
    _assert_equals_oracle(oracle, got, c, leaf, leaf)


def test_run_lengths(ctx, oracle):
    """One voxel of 5000 points; totals around the 1024-point chunks of k_voxel_heads and the 2048-key sort tiles."""
    clouds = [vc.one_voxel(13)] + [vc.run_total(n, 100 + n) for n in vc.RUN_TOTALS]
    got = _voxelize_on_device(ctx, clouds, 0.3)
    assert got[0].shape == (1, 3)
    for n, c, g in zip(("one_voxel",) + vc.RUN_TOTALS, clouds, got):
        _assert_equals_oracle(oracle, g, c, 0.3, n)


def test_every_point_its_own_voxel(ctx, oracle):
    c = vc.own_voxels(14)
    got, = _voxelize_on_device(ctx, [c], 1.0)
    assert got.shape == (len(c), 3)
    _assert_equals_oracle(oracle, got, c, 1.0, "own_voxels")


def test_overflow_guard(ctx, oracle):
    """trunc counts INT32_MAX - 1: voxelised (keys up to ~2^31); 2^31: the input comes back unchanged, in input order."""
    below, above = vc.guard_below(15), vc.guard_above(16)
    got_below, got_above = _voxelize_on_device(ctx, [below, above], 1.0)
    _assert_equals_oracle(oracle, got_below, below, 1.0, "guard_below")
    assert np.array_equal(_bits(got_above), _bits(above[:, :3]))
    _assert_equals_oracle(oracle, got_above, above, 1.0, "guard_above")


def test_index_above_int32_sorts_last(ctx, oracle):
    """The guard passes but indices of the upper z cell exceed INT32_MAX: the voxels come out in ascending order of the
    index as an unsigned 32-bit value, as PCL sorts it (the top corner's index also passes 2^32 and wraps to the front)."""
    c = vc.index_wrap(17)
    got, = _voxelize_on_device(ctx, [c], 1.0)
    _assert_equals_oracle(oracle, got, c, 1.0, "index_wrap")
    # at L = 1 the cell of a coordinate is its floor; here every voxel holds one point, so its centroid is that point
    min_b, max_b = np.floor(c[:, :3].min(0)).astype(np.int64), np.floor(c[:, :3].max(0)).astype(np.int64)
    div_b = max_b - min_b + 1
    ijk = np.floor(got).astype(np.int64) - min_b
    key = ijk[:, 0] + ijk[:, 1] * div_b[0] + ijk[:, 2] * div_b[0] * div_b[1]
    assert (key > vc.INT32_MAX).any() and (key >= 2 ** 32).any()
    assert (np.diff(key % 2 ** 32) > 0).all()


def test_ragged_batch(ctx, oracle, synth):
    """One call whose jobs differ in size by three orders of magnitude, one of which overflows the guard."""
    seq = vc.sweep_sequence(synth)
    clouds = [vc.run_total(1, 101), vc.guard_above(16), vc.own_voxels(14), vc.index_wrap(17), seq["clouds"][3] + np.float32(0),
              vc.run_total(2, 102), vc.guard_below(15), vc.one_voxel(13)]
    got = _voxelize_on_device(ctx, clouds, 1.0)
    assert np.array_equal(_bits(got[1]), _bits(clouds[1][:, :3]))
    for k, (c, g) in enumerate(zip(clouds, got)):
        _assert_equals_oracle(oracle, g, c, 1.0, k)
