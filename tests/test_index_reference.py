"""The index-build restatement (tests/index_ref.py) on the CPU: it agrees with a slow node-by-node Karras build, it
accepts a tap made from itself (with garbage in every record a collapsed leaf hides), and each deliberately wrong build
-- an unstable sort, a split off by one, a box that misses one point on one axis, leaves collapsed at LEAF + 1, numpy's
float -> int cast in place of cvt.rzi -- fails it."""
import numpy as np
import pytest

import index_ref as X


def make_tap(xyz, ref=None, tree=None, seed=0):
    """What b200reg_index_tap would return if the build were the restatement; unreachable records hold random bits."""
    ref = ref or X.build(xyz)
    n = len(ref["keys"])
    pts = np.zeros((n, 4), np.float32)
    pts[:, :3] = ref["pts"]
    pts[:, 3] = ref["order"].astype(np.int32).view(np.float32)
    tn = np.random.default_rng(seed).integers(0, 2 ** 32, (max(n - 1, 0), 4, 4), dtype=np.uint32).view(np.float32)
    tree = tree if tree is not None else X.expected_tree(ref["keys"], ref["pts"])
    if tree is not None:
        node, refs, lo, hi = tree[:4]
        tn[node, 0, :3], tn[node, 1, :3] = lo[:, 0], hi[:, 0]
        tn[node, 2, :3], tn[node, 3, :3] = lo[:, 1], hi[:, 1]
        tn[node, 0, 3] = refs[:, 0].astype(np.int32).view(np.float32)
        tn[node, 2, 3] = refs[:, 1].astype(np.int32).view(np.float32)
    return dict(keys=ref["keys"].copy(), orig=ref["order"].astype(np.int32), pts=pts, rank=ref["rank"].astype(np.int32),
                tnodes=tn, root_ref=0 if n > X.LEAF else int(X.leaf_ref(0, n)))


def clouds():
    rng = np.random.default_rng(5)
    out = {"n=%d" % n: rng.uniform(-5, 5, (n, 3)).astype(np.float32) for n in (1, 2, 8, 9, 17, 100, 777)}
    out["duplicates"] = np.repeat(rng.uniform(0, 1, (40, 3)).astype(np.float32), 7, axis=0)[rng.permutation(280)]
    g = np.arange(6, dtype=np.float32)
    out["lattice"] = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    nan = rng.uniform(0, 10, (300, 3)).astype(np.float32)
    nan[[0, 5, 6, 7, 100, 299]] = np.nan
    nan[[50, 51], 1] = np.nan
    out["nan"] = nan
    out["comb"] = X.comb_cloud(6)
    return out


@pytest.mark.parametrize("name", sorted(clouds()))
def test_restatement_accepts_itself(name):
    xyz = clouds()[name]
    depth = X.check(xyz, make_tap(xyz))
    assert depth <= X.depth_bound(len(xyz))


@pytest.mark.parametrize("name", ["n=9", "n=17", "n=100", "n=777", "duplicates", "lattice", "nan", "comb"])
def test_split_and_ranges_equal_slow_karras(name):
    """Without collapse every internal node of the top-down restatement has the range and split of Karras' per-node search."""
    ref = X.build(clouds()[name])
    slow = X.karras_slow(ref["keys"])
    node, refs, lo, hi, rng, depth = X.expected_tree(ref["keys"], ref["pts"], leaf=1)
    assert sorted(node.tolist()) == list(range(len(ref["keys"]) - 1))
    for i, r in zip(node.tolist(), rng.tolist()):
        first, last, g = slow[i]
        assert (r[0][0], r[1][1], r[0][1]) == (first, last, g), (name, i)


def test_comb_reaches_the_depth_bound():
    for m in (5, 6, 9, 12):  # 2^m > 30 extra points: n - 1 has m + 1 bits
        xyz = X.comb_cloud(m)
        ref = X.build(xyz)
        assert np.array_equal(ref["order"], np.arange(len(xyz)))  # keys 0, 1 (run), 2, 4, ..., 2^29, 2^30 - 1
        depth = X.expected_tree(ref["keys"], ref["pts"])[-1]
        assert depth == 28 + m == X.depth_bound(len(xyz)), (m, depth)
    assert X.DEPTH_BOUND == 53 <= X.MAX_STACK


def test_cvt_semantics():
    x = np.array([np.nan, np.inf, -np.inf, 2.0 ** 31, -2.0 ** 32, 1.9, -1.9, 1023.5, 3e9], np.float32)
    assert X.cvt_rzi(x).tolist() == [0, 2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1, -2 ** 31, 1, -1, 1023, 2 ** 31 - 1]


def _fails(xyz, tap):
    with pytest.raises(AssertionError):
        X.check(xyz, tap)


def test_unstable_sort_fails():
    xyz = clouds()["duplicates"]
    ref = X.build(xyz)
    keys = X.morton_keys(xyz)
    order = np.lexsort((-np.arange(len(keys)), keys))  # equal keys in descending index order
    bad = dict(ref, order=order, keys=keys[order], pts=xyz[order])
    bad["rank"] = np.argsort(order)
    _fails(xyz, make_tap(xyz, bad, X.expected_tree(bad["keys"], bad["pts"])))


def test_split_off_by_one_fails():
    xyz = clouds()["n=777"]
    ref = X.build(xyz)
    _fails(xyz, make_tap(xyz, ref, X.expected_tree(ref["keys"], ref["pts"], off_by=1)))


def test_box_missing_one_point_on_one_axis_fails():
    xyz = clouds()["n=777"]
    ref = X.build(xyz)
    node, refs, lo, hi, rng, depth = X.expected_tree(ref["keys"], ref["pts"])
    lo = lo.copy()
    f, l = rng[3, 1]
    x = np.sort(ref["pts"][f:l + 1, 1])
    assert x[0] < x[1]
    lo[3, 1, 1] = x[1]  # child 1 of the fourth record, y axis: its lowest point left out
    _fails(xyz, make_tap(xyz, ref, (node, refs, lo, hi, rng, depth)))


def test_collapse_at_leaf_plus_one_fails():
    xyz = clouds()["n=777"]
    ref = X.build(xyz)
    _fails(xyz, make_tap(xyz, ref, X.expected_tree(ref["keys"], ref["pts"], leaf=X.LEAF + 1)))


def test_numpy_cast_in_place_of_cvt_fails():
    """NaN alone gives key 0 either way (INT_MIN clamps to 0), and so does an infinite coordinate (ext = inf, scale = 0);
    a subnormal extent makes 1023 / ext = +inf, and (p - lo) * inf saturates to 1023 under cvt.rzi but becomes INT_MIN -> 0
    under numpy's cast."""
    xyz = np.zeros((40, 3), np.float32)
    xyz[1::2, 0] = np.float32(1e-42)
    xyz[0] = np.nan
    bad = X.build(xyz, cvt=X.cast_numpy)
    assert not np.array_equal(bad["keys"], X.build(xyz)["keys"])
    _fails(xyz, make_tap(xyz, bad, X.expected_tree(bad["keys"], bad["pts"])))
