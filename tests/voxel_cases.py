"""Crafted clouds for the pcl::VoxelGrid tests: the same inputs feed the numpy restatement of the oracle
(test_oracle_crosschecks.py, CPU) and the device voxel grid (test_gpu_voxel.py).  Every cloud is (n, 4) float32
(x, y, z, intensity) with no -0.0 coordinate: keyframes go through the identity transform on the device, and
1*(-0.0) + 0*y + 0*z + 0 is +0.0."""
import numpy as np

INT32_MAX = 2 ** 31 - 1
# keyframes of the test sequence used by the leaf sweep (at 0.05 m, 0 and 70 give voxel keys above 2^28)
SWEEP_KEYFRAMES = (0, 3, 70)
SWEEP_LEAVES = (0.05, 0.1, 0.3, 1.0, 2.5)
RUN_TOTALS = (1, 2, 1023, 1024, 1025, 2047, 2048, 2049)  # k_voxel_heads chunks of 1024 and their carry; sort tiles of 2048


def sweep_sequence(synth):
    return synth.make_sequence(7, 71, pts_per_keyframe=6000, spacing=3.0, speed=8.0)


def _cloud(xyz, seed):
    xyz = np.asarray(xyz, np.float32)
    rng = np.random.default_rng(seed)
    out = np.empty((len(xyz), 4), np.float32)
    out[:, :3] = xyz + np.float32(0)  # -0.0 + 0.0 = +0.0
    out[:, 3] = rng.uniform(0, 100, len(xyz)).astype(np.float32)
    return out


def _box(seed, n, lo, hi):
    """n points uniform in [lo, hi] (scalars or per axis); with n >= 2 the corners lo and hi are points, so that they
    are the fp32 bbox."""
    rng = np.random.default_rng(seed)
    lo, hi = np.broadcast_to(np.float32(lo), 3), np.broadcast_to(np.float32(hi), 3)
    xyz = np.clip(rng.uniform(lo, hi, (n, 3)).astype(np.float32), lo, hi)
    if n >= 2:
        xyz[0], xyz[1] = lo, hi
    rng.shuffle(xyz)
    return _cloud(xyz, seed)


def cell_boundaries(leaf, seed):
    """Coordinates k*L (fp32 product) and one nextafter either side, for both signs of k; the bbox minimum of every
    axis is the boundary value k_min*L itself.  1/L is inexact in fp32 for L = 0.1, 0.3: floor(v * (1/L)) then
    lands on either side of k, the same way on both sides of a correct comparison."""
    rng = np.random.default_rng(seed)
    v = np.arange(-12, 13).astype(np.float32) * np.float32(leaf)
    vals = np.concatenate([np.nextafter(v, np.float32(-np.inf)), v, np.nextafter(v, np.float32(np.inf))])
    vals = np.unique(vals[vals >= v[0]])
    xyz = rng.choice(vals, (3000, 3))
    xyz[:len(vals)] = vals[:, None]  # every value on every axis, v[0] included
    rng.shuffle(xyz)
    return _cloud(xyz, seed)


def one_voxel(seed, n=5000):
    return _box(seed, n, 0.31, 0.59)  # L = 0.3: floor(p / L) = 1 on every axis


def own_voxels(seed, n=3000):
    """L = 1: one point per occupied voxel, in shuffled order."""
    rng = np.random.default_rng(seed)
    cells = rng.choice(30 ** 3, n, replace=False)
    ijk = np.stack([cells % 30, cells // 30 % 30, cells // 900], 1) - 15
    return _cloud(ijk + rng.uniform(0.1, 0.9, (n, 3)), seed)


def run_total(n, seed):
    """n points in a 3 m cube: about 1000 voxels at L = 0.3, runs of every length."""
    return _box(seed, n, 0.05, 2.95)


# L = 1 below.  The guard multiplies trunc((max - min) / L) + 1 per axis; the index uses div_b = floor(max / L) -
# floor(min / L) + 1, which can be one larger.
def guard_below(seed, n=4000):
    """trunc counts 42966 x 49981 x 1 = INT32_MAX - 1: voxelised, keys up to ~2^31."""
    return _box(seed, n, (0.25, 0.25, 0.25), (42965.5, 49980.5, 0.75))


def guard_above(seed, n=4000):
    """trunc counts 32768 x 65536 x 1 = 2^31 > INT32_MAX: PCL returns the input unchanged."""
    return _box(seed, n, (0.25, 0.25, 0.25), (32767.5, 65535.5, 0.75))


def index_wrap(seed, n=4000):
    """trunc counts 46340 x 46340 x 1 = 2,147,395,600 pass the guard, but div_b = 46341 x 46341 x 2: every point in the
    upper z cell has an index >= 46341^2 = 2,147,488,281 > INT32_MAX.  PCL stores it as unsigned int and sorts those
    voxels after the lower layer; the top corner's index also passes 2^32 and wraps to 9265.  min_b is negative on
    x and y."""
    return _box(seed, n, (-19999.5, -19999.5, 0.5), (26340.25, 26340.25, 1.25))


def crafted():
    """(name, leaf, cloud) of every crafted case."""
    cases = [("boundaries_0.3", 0.3, cell_boundaries(0.3, 11)), ("boundaries_0.1", 0.1, cell_boundaries(0.1, 12)),
             ("one_voxel", 0.3, one_voxel(13)), ("own_voxels", 1.0, own_voxels(14))]
    cases += [("total_%d" % n, 0.3, run_total(n, 100 + n)) for n in RUN_TOTALS]
    cases += [("guard_below", 1.0, guard_below(15)), ("guard_above", 1.0, guard_above(16)), ("index_wrap", 1.0, index_wrap(17))]
    return cases
