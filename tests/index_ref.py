"""An exact numpy restatement of the spatial-index build (index_build.cu) and of the shared radix sort, no tolerances.

What b200reg_index_tap returns is held to it bit for bit:

* bounding box: NaN-ignoring fmin / fmax of every coordinate (+inf / -inf on an axis without a number);
* keys: ``ext = fmax(fmax(hi0 - lo0, hi1 - lo1), hi2 - lo2)`` and ``scale = ext > 0 ? 1023 / ext : 0`` in fp32 with IEEE
  division, ``q = clamp(cvt.rzi.s32.f32((p - lo) * scale), 0, 1023)`` (NaN -> 0, +-inf and out-of-range values saturate),
  key = expand10(q2) << 2 | expand10(q1) << 1 | expand10(q0);
* order: a stable sort of the keys gives the sorted points (w = original index bits) and rank;
* tree (over the records reachable from root_ref): Karras' split with the index tie-break
  ``delta(i, j) = clz(key_i ^ key_j)``, or ``32 + clz(i ^ j)`` for equal keys (= clz64 of (key << 32 | index));
  a child is a leaf exactly when its range holds <= LEAF points (the leaves partition [0, n) in order), an internal child
  of range [f, g] / [g + 1, l] is node g / g + 1; every child box is the fmin / fmax of its range's points per axis.  An
  axis without a number in the range is NaN for a one-point child (its box is the point) and (+inf, -inf) otherwise (a
  collapsed leaf starts its reduction at +-inf, and fmin / fmax never return NaN for a number);
* depth: the internal records on a root-to-leaf path.  delta strictly increases along a path; a reachable record spans
  >= LEAF + 1 points.  Distinct 30-bit keys give delta in [2, 31] (30 values); equal keys give 32 + clz(i ^ j) with
  8 <= i ^ j < 2^bitlen(n - 1), i.e. delta in [64 - bitlen(n - 1), 60].  So depth <= depth_bound(n) = 30 + bitlen(n - 1) - 3,
  53 at the largest cloud (2^26 points), within MAX_STACK = 64.  The comb of comb_cloud() reaches the bound exactly.

Records inside collapsed leaves are never written by the build and are excluded from every comparison.
"""
import numpy as np

LEAF = 8
MAX_STACK = 64
SORT_TILE = 2048
MAX_POINTS = 1 << 26  # clouds_create's cap


def bitlen(v):
    return int(v).bit_length()


def depth_bound(n):
    """Most internal records on a root-to-leaf path of an n-point cloud (module docstring)."""
    return 30 + max(0, bitlen(n - 1) - 3)


DEPTH_BOUND = depth_bound(MAX_POINTS)


def leaf_ref(start, count):
    return -1 - ((np.asarray(start, np.int64) << 4) | count)


# ---------------------------------------------------------------------------------------------------------------------
# keys and order
def bbox(xyz):
    p = np.asarray(xyz, np.float32)[:, :3]
    lo = np.fmin.reduce(p, axis=0, initial=np.inf).astype(np.float32)
    hi = np.fmax.reduce(p, axis=0, initial=-np.inf).astype(np.float32)
    return lo, hi


def cvt_rzi(x):
    """cvt.rzi.s32.f32: truncate; NaN -> 0; +-inf and out-of-range values saturate to the int32 range."""
    x = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        t = np.clip(np.trunc(np.where(np.isnan(x), 0.0, x)), -2.0 ** 31, 2.0 ** 31 - 1)
    return t.astype(np.int64)


def cast_numpy(x):
    """The wrong variant: numpy's float -> int32 cast (NaN and inf become INT_MIN on x86)."""
    with np.errstate(invalid="ignore"):
        return np.asarray(x, np.float32).astype(np.int32).astype(np.int64)


def expand10(v):
    v = np.asarray(v, np.uint32) & np.uint32(0x3FF)
    v = (v | (v << np.uint32(16))) & np.uint32(0x030000FF)
    v = (v | (v << np.uint32(8))) & np.uint32(0x0300F00F)
    v = (v | (v << np.uint32(4))) & np.uint32(0x030C30C3)
    v = (v | (v << np.uint32(2))) & np.uint32(0x09249249)
    return v


def interleave(q0, q1, q2):
    return (expand10(q2) << np.uint32(2)) | (expand10(q1) << np.uint32(1)) | expand10(q0)


def morton_keys(xyz, cvt=cvt_rzi):
    p = np.asarray(xyz, np.float32)[:, :3]
    lo, hi = bbox(p)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ext = np.fmax(np.fmax(hi[0] - lo[0], hi[1] - lo[1]), hi[2] - lo[2])
        scale = np.float32(1023.0) / ext if ext > 0 else np.float32(0.0)
        q = [np.clip(cvt((p[:, a] - lo[a]) * scale), 0, 1023) for a in range(3)]
    return interleave(*q)


def build(xyz, cvt=cvt_rzi, kind="stable"):
    """-> dict(keys (sorted), order (sorted position -> original index), rank, pts (n, 3) sorted) of the restatement."""
    p = np.ascontiguousarray(np.asarray(xyz, np.float32)[:, :3])
    keys = morton_keys(p, cvt)
    order = np.argsort(keys, kind=kind)
    rank = np.empty(len(p), np.int64)
    rank[order] = np.arange(len(p))
    return dict(keys=keys[order], order=order, rank=rank, pts=p[order])


# ---------------------------------------------------------------------------------------------------------------------
# the tree
def _clz32(v):
    v = np.asarray(v, np.int64)
    return np.where(v == 0, 32, 32 - np.frexp(v.astype(np.float64))[1])


def delta(keys, i, j):
    """Karras' delta with the index tie-break (index_build.cu: delta) for index arrays i, j inside [0, n)."""
    k = np.asarray(keys, np.int64)
    x = k[i] ^ k[j]
    return np.where(x != 0, _clz32(x), 32 + _clz32(np.asarray(i, np.int64) ^ np.asarray(j, np.int64)))


def split(keys, f, l, off_by=0):
    """Karras split of the ranges [f, l] (f < l): the last position g of the left child.  off_by: the wrong variant."""
    aug = (np.asarray(keys, np.uint64) << np.uint64(32)) | np.arange(len(keys), dtype=np.uint64)
    f = np.asarray(f, np.int64)
    l = np.asarray(l, np.int64)
    b = 63 - delta(keys, f, l)  # highest differing bit of the augmented keys
    thr = (aug[l] >> b.astype(np.uint64)) << b.astype(np.uint64)
    g = np.searchsorted(aug, thr, side="left").astype(np.int64) - 1
    return np.clip(g + off_by, f, l - 1) if off_by else g


def _range_box(s, f, l):
    """Per-axis fmin / fmax of the sorted points over the ranges [f, l], with the empty-axis rule of the build."""
    pts = np.concatenate([s, np.zeros((1, 3), np.float32)])
    idx = np.empty(2 * len(f), np.int64)
    idx[0::2], idx[1::2] = f, l + 1
    lo = np.fmin.reduceat(pts, idx, axis=0)[0::2]
    hi = np.fmax.reduceat(pts, idx, axis=0)[0::2]
    empty = np.isnan(lo) & ((l - f) > 0)[:, None]
    lo[empty], hi[empty] = np.inf, -np.inf
    return lo.astype(np.float32), hi.astype(np.float32)


def expected_tree(keys, pts, leaf=LEAF, off_by=0, box_fn=None):
    """The records the build must write: {node: (refs (2,), lo (2, 3), hi (2, 3))} as arrays over the reachable nodes,
    plus the depth.  -> (nodes (m,), refs (m, 2), lo (m, 2, 3), hi (m, 2, 3), ranges (m, 2, 2), depth)."""
    n = len(keys)
    box_fn = box_fn or _range_box
    if n <= leaf:
        return None
    out = {k: [] for k in ("node", "refs", "lo", "hi", "rng")}
    node, f, l = np.array([0]), np.array([0]), np.array([n - 1])
    depth = 0
    while len(node):
        depth += 1
        g = split(keys, f, l, off_by)
        cf = np.stack([f, g + 1], 1)
        cl = np.stack([g, l], 1)
        size = cl - cf + 1
        internal = size > leaf
        ids = np.stack([g, g + 1], 1)
        refs = np.where(internal, ids, leaf_ref(cf, np.minimum(size, 15)))
        lo, hi = box_fn(pts, cf.ravel(), cl.ravel())
        out["node"].append(node)
        out["refs"].append(refs)
        out["lo"].append(lo.reshape(-1, 2, 3))
        out["hi"].append(hi.reshape(-1, 2, 3))
        out["rng"].append(np.stack([cf, cl], 2))
        node, f, l = ids[internal], cf[internal], cl[internal]
    cat = {k: np.concatenate(v) for k, v in out.items()}
    return cat["node"], cat["refs"], cat["lo"], cat["hi"], cat["rng"], depth


def _same_f32(a, b):
    """== per element, NaN matching NaN (so +0 and -0 compare equal, as the build may give either)."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    return (a == b) | (np.isnan(a) & np.isnan(b))


def reachable(tnodes, root_ref):
    """Internal record indices reachable from root_ref (from the tap's records) and the depth -> (sorted ids, depth)."""
    refs = np.asarray(tnodes, np.float32)[:, [0, 2], 3].view(np.int32) if len(tnodes) else np.zeros((0, 2), np.int32)
    if root_ref < 0:
        return np.zeros(0, np.int64), 0
    seen, level, depth = [], np.array([root_ref]), 0
    while len(level):
        assert len(level) <= len(tnodes) and (level < len(tnodes)).all() and (level >= 0).all(), "a ref leaves the record array"
        depth += 1
        seen.append(level)
        r = refs[level].ravel()
        level = r[r >= 0].astype(np.int64)
        assert depth <= MAX_STACK + 1, "the records form a cycle or a path deeper than MAX_STACK"
    return np.sort(np.concatenate(seen)), depth


def check(xyz, tap, ref=None, tree=None):
    """Assert the tap of one cloud equals the restatement bit for bit; returns the tree depth."""
    p = np.ascontiguousarray(np.asarray(xyz, np.float32)[:, :3])
    n = len(p)
    ref = ref or build(p)
    assert np.array_equal(tap["keys"], ref["keys"]), ("keys", np.flatnonzero(tap["keys"] != ref["keys"])[:5])
    assert np.array_equal(tap["orig"], ref["order"]), ("order", np.flatnonzero(tap["orig"] != ref["order"])[:5])
    assert np.array_equal(tap["pts"][:, :3].view(np.uint32), ref["pts"].view(np.uint32)), "sorted points"
    assert np.array_equal(tap["rank"], ref["rank"]), "rank"
    if n <= LEAF:
        assert tap["root_ref"] == leaf_ref(0, n), ("root_ref", tap["root_ref"])
        return 0
    assert tap["root_ref"] == 0, ("root_ref", tap["root_ref"])
    tree = tree or expected_tree(ref["keys"], ref["pts"])
    node, refs, lo, hi, rng, depth = tree
    tn = np.asarray(tap["tnodes"], np.float32)
    got_refs = tn[node][:, [0, 2], 3].view(np.int32)
    bad = np.flatnonzero((got_refs != refs).any(1))
    assert len(bad) == 0, ("topology / leaf collapse", node[bad[:5]], got_refs[bad[:5]].tolist(), refs[bad[:5]].tolist())
    got_lo = tn[node][:, [0, 2], :3]
    got_hi = tn[node][:, [1, 3], :3]
    bad = np.flatnonzero(~(_same_f32(got_lo, lo) & _same_f32(got_hi, hi)).all((1, 2)))
    assert len(bad) == 0, ("boxes", node[bad[:3]], got_lo[bad[:3]].tolist(), lo[bad[:3]].tolist(), got_hi[bad[:3]].tolist(),
                           hi[bad[:3]].tolist())
    # the reachable set is exactly the expected one, and the leaves partition [0, n) in order
    ids, gdepth = reachable(tn, tap["root_ref"])
    assert np.array_equal(ids, np.sort(node)), "reachable records differ"
    leaves = rng.reshape(-1, 2)[refs.ravel() < 0]
    leaves = leaves[np.argsort(leaves[:, 0])]
    assert leaves[0, 0] == 0 and leaves[-1, 1] == n - 1 and (leaves[1:, 0] == leaves[:-1, 1] + 1).all(), "leaves"
    assert ((leaves[:, 1] - leaves[:, 0] + 1) <= LEAF).all()
    check_containment(ref["pts"], rng.reshape(-1, 2), got_lo.reshape(-1, 3), got_hi.reshape(-1, 3))
    assert gdepth == depth <= depth_bound(n) <= MAX_STACK, (gdepth, depth, depth_bound(n))
    return depth


def check_containment(pts, rng, lo, hi):
    """Every finite coordinate of a range lies inside the box of that range (so inside every ancestor's box)."""
    lo_r, hi_r = _range_box(pts, rng[:, 0], rng[:, 1])
    fin = np.isfinite(lo_r) & np.isfinite(hi_r)
    ok = ~fin | ((lo <= lo_r) & (hi_r <= hi))
    bad = np.flatnonzero(~ok.all(1))
    assert len(bad) == 0, ("a point lies outside its box", rng[bad[:3]].tolist())


# ---------------------------------------------------------------------------------------------------------------------
# a slow per-node Karras build (the restatement's own check on small clouds)
def karras_slow(keys, leaf=LEAF):
    """Node-by-node, as Karras 2012 states it: the direction, the range by doubling and binary search, the split by binary
    search, for every i in [0, n - 1).  -> {i: (first, last, split)}."""
    n = len(keys)

    def d(i, j):
        if j < 0 or j >= n:
            return -1
        x = int(keys[i]) ^ int(keys[j])
        return 32 - x.bit_length() if x else 32 + 32 - (i ^ j).bit_length()

    nodes = {}
    for i in range(n - 1):
        s = 1 if d(i, i + 1) - d(i, i - 1) >= 0 else -1
        dmin = d(i, i - s)
        lmax = 2
        while d(i, i + lmax * s) > dmin:
            lmax *= 2
        ln = 0
        t = lmax // 2
        while t >= 1:
            if d(i, i + (ln + t) * s) > dmin:
                ln += t
            t //= 2
        j = i + ln * s
        dn = d(i, j)
        sp = 0
        t = ln
        while True:
            t = (t + 1) // 2
            if d(i, i + (sp + t) * s) > dn:
                sp += t
            if t <= 1:
                break
        g = i + sp * s + min(s, 0)
        nodes[i] = (min(i, j), max(i, j), g)
    return nodes


# ---------------------------------------------------------------------------------------------------------------------
# clouds
def comb_cloud(m):
    """One point per key bit (key 2^b for b = 1..29), key 0 once, key 2^30 - 1 once (it fixes the extent at 1023, so
    scale = 1 and q = p) and a run of 2^m identical points at key 1 right after key 0.  The tree peels one key bit per
    level (delta 2..31), then the run's index chain [1, 2^j - 1] for j = m..4: depth 28 + m = depth_bound(n)."""
    bits = np.zeros((29, 3), np.float32)
    bits[np.arange(29), np.arange(1, 30) % 3] = 2.0 ** (np.arange(1, 30) // 3)
    run = np.repeat(np.array([[1.0, 0.0, 0.0]], np.float32), 1 << m, axis=0)
    return np.concatenate([np.zeros((1, 3), np.float32), run, bits, np.full((1, 3), 1023.0, np.float32)])


def argsort_stable(keys):
    return np.argsort(np.asarray(keys), kind="stable")
