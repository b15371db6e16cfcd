"""Exact fp32 restatement of the feature matcher (k_feat_nn x2, k_first_hit, k_mutual; matcher.cc:378-455 and the TBB
branch of advancedMatching, matcher.cc:160-188), an fp64 certificate of it, and a numpy emulation of the records the kernels
order and filter (the k_fpfh tail, k_fcode).

Semantics (include/b200reg.h, b200reg_match_tap):
  d2(a, b)  = ((e0*e0 + e1*e1) + ...) + e32*e32 in fp32, e = a - b, no FMA
  nn(j)     = the usable row of fi with the least d2 to fj[j], the lowest row among equal d2; -1 when fj[j] is unusable,
              fi has no usable row, or (optimizedMatching) d2 > thr2 with thr2 = fp32(thr) * fp32(thr) (a square that
              overflows, or a NaN, drops nothing: `dis > thr2` is never true)
  first(i)  = the lowest j with nn(j) == i (advancedMatching: every such j qualifies)
  rnn(i)    = the usable row of fj nearest to fi[i], lowest row among ties, for every i that some j reached; -1 elsewhere
  mutual    = (i, j) in ascending j: nn(j) == i, rnn(i) == j and (optimizedMatching) j == first(i)
An all-zero row is unusable.  Two backends compute the same bits: numpy (crafted cases) and torch on the GPU (raw scans
of 100k points), both with separate sub / mul / add passes over the 33 bins so that nothing can fuse.
"""
import os
import re

import numpy as np

FLT_MAX = np.float32(3.4028234663852886e38)
U32 = np.float64(2.0 ** -24)  # unit roundoff of fp32
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gamma(n):
    return n * U32 / (1 - n * U32)


def thr2_of(thr, advanced=False):
    if advanced:
        return FLT_MAX
    with np.errstate(over="ignore", invalid="ignore"):
        return np.float32(thr) * np.float32(thr)


def usable(F):
    return (np.asarray(F) != 0).any(1)


# ---------------------------------------------------------------------------------------------------------------------
# nearest usable row, exact fp32
def _unique_rows(B, ok):
    """Bitwise distinct usable rows of B and the lowest row index of each: identical rows have identical d2, so the
    lowest-index rule only ever picks a run's first row."""
    rows = np.flatnonzero(ok)
    if len(rows) == 0:
        return np.zeros((0, 33), np.float32), np.zeros(0, np.int64)
    Bu = np.ascontiguousarray(B[rows])
    _, first = np.unique(Bu.view(np.dtype((np.void, 33 * 4))).ravel(), return_index=True)
    return Bu[first], rows[first]


def nearest_numpy(Q, B, okB, chunk=None):
    """-> (idx, d2): per row of Q the usable row of B with the least fp32 d2 (lowest index among ties), -1 / +inf if none."""
    Q = np.ascontiguousarray(Q, np.float32)
    Bu, rep = _unique_rows(np.ascontiguousarray(B, np.float32), okB)
    idx = np.full(len(Q), -1, np.int64)
    best = np.full(len(Q), np.inf, np.float32)
    if len(Bu) == 0:
        return idx, best
    chunk = chunk or max(1, (1 << 22) // len(Bu))
    for a in range(0, len(Q), chunk):
        q = Q[a:a + chunk]
        d = np.zeros((len(q), len(Bu)), np.float32)
        for k in range(33):
            e = np.subtract(q[:, k:k + 1], Bu[None, :, k], dtype=np.float32)
            d = np.add(d, np.multiply(e, e, dtype=np.float32), dtype=np.float32)
        m = d.min(1)
        idx[a:a + chunk] = np.where(d == m[:, None], rep[None, :], np.iinfo(np.int64).max).min(1)
        best[a:a + chunk] = m
    return idx, best


def nearest_torch(Q, B, okB, device="cuda", chunk=2048):
    """The same bits on the GPU (torch eager: every sub / mul / add is its own kernel, nothing fuses)."""
    import torch
    Bu, rep = _unique_rows(np.ascontiguousarray(B, np.float32), okB)
    idx = np.full(len(Q), -1, np.int64)
    best = np.full(len(Q), np.inf, np.float32)
    if len(Bu) == 0:
        return idx, best
    Bt = torch.from_numpy(np.ascontiguousarray(Bu.T)).to(device)  # (33, nb)
    rept = torch.from_numpy(rep).to(device)
    big = torch.tensor(np.iinfo(np.int64).max, device=device)
    Qt = torch.from_numpy(np.ascontiguousarray(Q, np.float32)).to(device)
    out_i, out_d = [], []
    for a in range(0, len(Q), chunk):
        q = Qt[a:a + chunk]
        d = torch.zeros((len(q), Bt.shape[1]), dtype=torch.float32, device=device)
        for k in range(33):
            e = torch.sub(q[:, k:k + 1], Bt[k:k + 1, :])
            d = torch.add(d, torch.mul(e, e))
        m = d.amin(1)
        out_i.append(torch.where(d == m[:, None], rept[None, :], big).amin(1))
        out_d.append(m)
    idx[:] = torch.cat(out_i).cpu().numpy()
    best[:] = torch.cat(out_d).cpu().numpy()
    return idx, best


def d2_fp32(a, b):
    """d2 of row pairs (a[k], b[k]) in the kernels' order."""
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    d = np.zeros(len(a), np.float32)
    for k in range(33):
        e = np.subtract(a[:, k], b[:, k], dtype=np.float32)
        d = np.add(d, np.multiply(e, e, dtype=np.float32), dtype=np.float32)
    return d


# ---------------------------------------------------------------------------------------------------------------------
def match_ref(fi, fj, thr=35.0, advanced=False, backend="numpy"):
    """-> dict(nn, dis, rnn, mutual, first) in the tap's layout (see the module docstring)."""
    fi = np.ascontiguousarray(fi, np.float32)
    fj = np.ascontiguousarray(fj, np.float32)
    near = nearest_torch if backend == "torch" else nearest_numpy
    oki, okj = usable(fi), usable(fj)
    t2 = thr2_of(thr, advanced)
    nn, dis = near(fj, fi, oki)
    with np.errstate(invalid="ignore"):
        gated = dis > t2  # False for thr2 = +inf or NaN
    nn = np.where(okj & (nn >= 0) & ~gated, nn, -1)
    first = np.full(len(fi), np.iinfo(np.int64).max, np.int64)
    js = np.flatnonzero(nn >= 0)
    np.minimum.at(first, nn[js], js)
    hit = np.flatnonzero(first != np.iinfo(np.int64).max)
    rnn = np.full(len(fi), -1, np.int64)
    if len(hit):
        rnn[hit] = near(fi[hit], fj, okj)[0]
    i = nn[js]
    keep = (rnn[i] == js) & (advanced | (first[i] == js))
    mutual = np.stack([i[keep], js[keep]], 1).astype(np.int32).reshape(-1, 2)
    return dict(nn=nn.astype(np.int32), dis=dis, rnn=rnn.astype(np.int32), mutual=mutual, first=first)


# ---------------------------------------------------------------------------------------------------------------------
# fp64 certificate of the fp32 winners
def certify_fp64(Q, B, okB, win, backend="numpy", device="cuda"):
    """For every query with a winner: the fp64 distance to the fp32 winner exceeds the fp64 minimum by at most what the
    fp32 sum can hide, d64(win) <= d64min * (1 + g) / (1 - g), g = gamma(35) (33 terms, each e = a - b and e*e rounded,
    32 additions).  Candidates for the fp64 minimum are the rows whose fp32 d2 lies within that factor of the winner's.
    -> dict(n, differ (winner is not the lowest-index fp64 argmin), max_gap, max_rel_gap, max_ratio (of the allowed))."""
    g = gamma(35)
    lim = (1 + g) / (1 - g)
    Q = np.ascontiguousarray(Q, np.float32)
    Bu, rep = _unique_rows(np.ascontiguousarray(B, np.float32), okB)
    sel = np.flatnonzero(win >= 0)
    pos = {int(r): k for k, r in enumerate(rep)}
    wu = np.array([pos[int(w)] for w in win[sel]], np.int64)
    differ, max_gap, max_rel, max_ratio = 0, 0.0, 0.0, 0.0
    if backend == "torch":
        import torch
        Bt = torch.from_numpy(np.ascontiguousarray(Bu.T)).to(device)
        B64 = torch.from_numpy(Bu.astype(np.float64)).to(device)
        Qt = torch.from_numpy(Q[sel]).to(device)
        wt = torch.from_numpy(wu).to(device)
        rept = torch.from_numpy(rep).to(device)
    chunk = 1024 if backend == "torch" else max(1, (1 << 23) // max(1, 33 * len(Bu)))
    for a in range(0, len(sel), chunk):
        if backend == "torch":
            q = Qt[a:a + chunk]
            d = torch.zeros((len(q), Bt.shape[1]), dtype=torch.float32, device=device)
            for k in range(33):
                e = torch.sub(q[:, k:k + 1], Bt[k:k + 1, :])
                d = torch.add(d, torch.mul(e, e))
            w = wt[a:a + chunk]
            dw = d.gather(1, w[:, None])[:, 0].double()
            rows, cols = torch.nonzero(d.double() <= dw[:, None] * lim * (1 + 4 * g), as_tuple=True)
            q64 = q.double()
            d64 = ((q64[rows] - B64[cols]) ** 2).sum(1)
            dmin = torch.full((len(q),), float("inf"), dtype=torch.float64, device=device).scatter_reduce(0, rows, d64, "amin")
            big = torch.tensor(np.iinfo(np.int64).max, device=device)
            amin = torch.full((len(q),), np.iinfo(np.int64).max, dtype=torch.int64, device=device).scatter_reduce(
                0, rows, torch.where(d64 == dmin[rows], rept[cols], big), "amin")
            dwin = ((q64 - B64[w]) ** 2).sum(1)
            dmin, amin, dwin, w_rep = dmin.cpu().numpy(), amin.cpu().numpy(), dwin.cpu().numpy(), rep[w.cpu().numpy()]
        else:
            q = Q[sel[a:a + chunk]]
            q64, B64 = q.astype(np.float64), Bu.astype(np.float64)
            d64 = ((q64[:, None, :] - B64[None, :, :]) ** 2).sum(2)
            dmin = d64.min(1)
            amin = np.where(d64 == dmin[:, None], rep[None, :], np.iinfo(np.int64).max).min(1)
            w = wu[a:a + chunk]
            dwin = d64[np.arange(len(q)), w]
            w_rep = rep[w]
        assert np.all(dwin <= dmin * lim + 1e-300), "an fp32 winner is farther in fp64 than the fp32 sum can explain"
        gap = dwin - dmin
        bad = amin != w_rep
        differ += int(bad.sum())
        if bad.any():
            max_gap = max(max_gap, float(gap[bad].max()))
            max_rel = max(max_rel, float((gap[bad] / np.maximum(dmin[bad], 1e-300)).max()))
        allowed = dmin * (lim - 1)
        pos_ = allowed > 0
        if pos_.any():
            max_ratio = max(max_ratio, float((gap[pos_] / allowed[pos_]).max()))
    return dict(n=len(sel), differ=differ, max_gap=max_gap, max_rel_gap=max_rel, max_ratio=max_ratio)


# ---------------------------------------------------------------------------------------------------------------------
# the records the kernels order and filter: fpfh_basis.cuh, the tail of k_fpfh (write_record) and k_fcode, in fp32
def _basis():
    txt = open(os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc", "fpfh_basis.cuh")).read()
    nums = lambda s: np.array([np.float32(x) for x in re.findall(r"([-+0-9.eE]+)f", s)], np.float32)
    mu = nums(re.search(r"FB_MU\[33\] = \{(.*?)\};", txt, re.S).group(1))
    U = nums(re.search(r"FB_U\[3\]\[33\] = \{(.*?)\};", txt, re.S).group(1)).reshape(3, 33)
    assert mu.shape == (33,) and U.shape == (3, 33)
    return mu, U


FB_MU, FB_U = _basis()


def filter_coords(F):
    """(n, 4) fp32 filter coordinates of write_record: x = v - mu; c_i = sum_k x_k * U_ik in k order; residual
    e_k = x_k - ((c0 U_0k + c1 U_1k) + c2 U_2k); r = sqrt(sum_k e_k^2) in k order.  No FMA (-fmad=false)."""
    F = np.ascontiguousarray(F, np.float32)
    f32 = np.float32
    x = np.subtract(F, FB_MU[None, :], dtype=f32)
    c = np.zeros((len(F), 3), f32)
    for k in range(33):
        c = np.add(c, np.multiply(x[:, k:k + 1], FB_U[None, :, k], dtype=f32), dtype=f32)
    rr = np.zeros(len(F), f32)
    for k in range(33):
        rec = np.add(np.add(np.multiply(c[:, 0], FB_U[0, k], dtype=f32), np.multiply(c[:, 1], FB_U[1, k], dtype=f32), dtype=f32),
                     np.multiply(c[:, 2], FB_U[2, k], dtype=f32), dtype=f32)
        e = np.subtract(x[:, k], rec, dtype=f32)
        rr = np.add(rr, np.multiply(e, e, dtype=f32), dtype=f32)
    return np.concatenate([c, np.sqrt(rr)[:, None]], 1).astype(f32)


def _fma32(a, b, c):
    """fp32 fma(a, b, c) through fp64: a*b of two floats is exact in fp64, one more rounding in the sum (the filter is
    not a parity value; this is for the margin measurement)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def filt_lb(q, b):
    """k_feat_nn's filt_lb: squared distance of the filter coordinates, fused as the kernel does."""
    e = np.subtract(np.asarray(q, np.float32), np.asarray(b, np.float32), dtype=np.float32)
    s = np.multiply(e[..., 0], e[..., 0], dtype=np.float32)
    for k in (1, 2, 3):
        s = _fma32(e[..., k], e[..., k], s)
    return s


def filt_margin(d2):
    """filt_bound's allowance in distance: sqrt(best) * 1e-5 + 4e-3."""
    return np.sqrt(np.asarray(d2, np.float64)) * 1e-5 + 4e-3


def max_centered_norm():
    """max |a - mu| over the descriptor domain (three 11-bin blocks, each >= 0 summing to 100): the squared norm is convex
    per block, so the maximum sits at a one-hot block, at the bin where mu is smallest."""
    mu = FB_MU.astype(np.float64).reshape(3, 11)
    return float(np.sqrt(sum(1e4 - 200 * m.min() + (m ** 2).sum() for m in mu)))


def derived_excess(xmax):
    """Worst-case amount by which the computed filter distance sqrt(filt_lb) can exceed the true projected distance (a
    lower bound of |a - b|) for |a - mu|, |b - mu| <= xmax, from the fp32 operation order of write_record and filt_lb:
      c_i:  33 products and 32 additions after x = v - mu      |dc| <= gamma(35) * sum_k |x_k U_ik| <= gamma(35) xmax
      r:    |x^ - x| + |sum_i dc_i U_i| + reconstruction (gamma(3) sqrt(3) |x|) + subtraction (u |x|) + the 33-term sum and
            the sqrt (gamma(18) |x|)
      each filter coordinate of a - b carries both records' errors and the rounding of the difference (u 2 xmax);
      filt_lb's fused sum rounds 4 times (gamma(4) relative, 2 xmax at most)."""
    u = U32
    dc = gamma(35) * xmax
    dr = u * xmax + np.sqrt(3.0) * dc + gamma(3) * np.sqrt(3.0) * xmax + u * xmax + gamma(18) * xmax
    ec, er = 2 * dc + u * 2 * xmax, 2 * dr + u * 2 * xmax
    return float(np.sqrt(3 * ec ** 2 + er ** 2) + gamma(4) * 2 * xmax)


def fnv_hash(F):
    """slot 35 of a record: FNV-style hash of the bins' bits."""
    bits = np.ascontiguousarray(F, np.float32).view(np.uint32).astype(np.uint64)
    h = np.full(len(F), 0x811C9DC5, np.uint64)
    for k in range(33):
        h = ((h ^ bits[:, k]) * 0x01000193) & 0xFFFFFFFF
        h ^= h >> 15
    return h.astype(np.uint32)


def fcode(P):
    """k_fcode's 28-bit Morton code of the filter coordinates."""
    P = np.asarray(P, np.float32)
    f32 = np.float32

    def q(v, off, scale):
        t = np.multiply(np.add(v, f32(off), dtype=f32), scale, dtype=f32)
        return np.clip(np.trunc(t.astype(np.float64)), 0, 127).astype(np.uint32)

    qs = [q(P[:, 0], 60, f32(128) / f32(120)), q(P[:, 1], 40, f32(128) / f32(80)), q(P[:, 2], 30, f32(128) / f32(60)),
          q(P[:, 3], 0, f32(128) / f32(60))]
    c = np.zeros(len(P), np.uint32)
    for b in range(7):
        for d in range(4):
            c |= ((qs[d] >> b) & 1) << (4 * b + d)
    return c


def sort_keys(F):
    """The matcher's sort key of every row: Morton code << 4 | 4 hash bits, 0xFFFFFFFF for unusable rows."""
    F = np.ascontiguousarray(F, np.float32)
    k = (fcode(filter_coords(F)).astype(np.uint64) << 4 | (fnv_hash(F) & 15)).astype(np.uint32)
    return np.where(usable(F), k, np.uint32(0xFFFFFFFF))


def sorted_order(F):
    """Rows in the order k_fgather stores them (stable sort by key, ties by row)."""
    return np.argsort(sort_keys(F), kind="stable")


def block_start_tiles(Fq, Fb, threads=128, tile=64):
    """s_t0 of every query block of k_feat_nn: the base tile where the code of the block's middle query would sit."""
    kq = np.sort(sort_keys(Fq), kind="stable")
    kb = np.sort(sort_keys(Fb), kind="stable")
    ntiles = (len(Fb) + tile - 1) // tile
    mids = np.minimum(len(Fq) - 1, np.arange(0, len(Fq), threads) + threads // 2)
    return np.minimum(ntiles - 1, np.searchsorted(kb, kq[mids], side="left") // tile)


def visit_rank(t, t0, ntiles):
    """Position of tile t in a block's sweep: t0, t0 + 1, ..., ntiles - 1, then t0 - 1, ..., 0."""
    t = np.asarray(t)
    return np.where(t >= t0, t - t0, (ntiles - t0) + (t0 - 1 - t))


# ---------------------------------------------------------------------------------------------------------------------
# crafted descriptors: in the domain (three blocks of 11 bins, each >= 0 summing to 100), integer or dyadic bins, so that
# every d2 below is exact in fp32 and equal d2 are real ties
def random_desc(rng, n, conc=1.0):
    p = rng.dirichlet(np.full(11, conc), size=(n, 3))
    return np.concatenate([np.stack([rng.multinomial(100, p[i, b]) for i in range(n)]) for b in range(3)], 1).astype(np.float32)


def unit_moves(c):
    """Every distinct +1 / -1 move inside one block of c (d2 = 2 from c), as (n, 33)."""
    out = []
    for b in range(3):
        for s in range(11):
            for t in range(11):
                if s != t and c[11 * b + t] >= 1:
                    d = c.copy()
                    d[11 * b + s] += 1
                    d[11 * b + t] -= 1
                    out.append(d)
    return np.array(out, np.float32)


def one_hot_extremes():
    """Every descriptor with one-hot blocks (|a - mu| up to 220.5), 11^3 of them."""
    g = np.stack(np.meshgrid(np.arange(11), np.arange(11), np.arange(11), indexing="ij"), -1).reshape(-1, 3)
    F = np.zeros((len(g), 33), np.float32)
    for b in range(3):
        F[np.arange(len(g)), 11 * b + g[:, b]] = 100
    return F


def tie_coverage(Q, B, searched=None, threads=128, tile=64):
    """Where the lowest-index member of an exact d2 tie lies in a tile that the query's block visits LATER than another
    tile holding a member: counts of such queries with the winner's tile above (>= s_t0) and below s_t0.  Q is the whole
    query cloud (its sorted order makes the blocks); `searched` masks the queries that search (the reverse search: the
    rows of fi that some j reached)."""
    ok = usable(B)
    okq = usable(Q) if searched is None else usable(Q) & searched
    order = sorted_order(B)
    tile_of = np.empty(len(B), np.int64)
    tile_of[order] = np.arange(len(B)) // tile
    ntiles = (len(B) + tile - 1) // tile
    qpos = np.empty(len(Q), np.int64)
    qpos[sorted_order(Q)] = np.arange(len(Q))
    t0 = block_start_tiles(Q, B, threads, tile)[qpos // threads]
    above = below = 0
    for q in np.flatnonzero(okq):
        d = d2_fp32(np.repeat(Q[q:q + 1], len(B), 0), B)
        d[~ok] = np.inf
        ties = np.flatnonzero(d == d.min())
        if len(ties) < 2 or not np.isfinite(d.min()):
            continue
        # identical records collapse to their run's head: only distinct records count as members in distinct tiles
        w = ties.min()
        rk = visit_rank(tile_of[ties], t0[q], ntiles)
        if visit_rank(tile_of[w], t0[q], ntiles) > rk.min():
            if tile_of[w] >= t0[q]:
                above += 1
            else:
                below += 1
    return above, below


def dyadic_mu(step=0.25):
    """FB_MU rounded to multiples of `step`, each block repaired (at its largest bin) to sum to exactly 100."""
    m = np.round(FB_MU.astype(np.float64) / step) * step
    for b in range(3):
        blk = m[11 * b:11 * b + 11]
        blk[np.argmax(blk)] += 100 - blk.sum()
    assert (m >= 0).all()
    return m


def projected_tight(rng, n_random=60, alphas=(0.75, 0.875, 0.9375)):
    """Pairs on which k_feat_nn's projected lower bound is tight.  The bound sum_i (u_i.(a - b))^2 + (|r_a| - |r_b|)^2 equals
    |a - b|^2 when the residuals r_a, r_b are parallel, which holds for b = alpha a + (1 - alpha) mu (then a - b =
    (1 - alpha)(a - mu)).  With mu rounded to quarters (m = dyadic_mu()) and dyadic alpha, b is in the domain (a convex
    combination of two in-domain descriptors), every bin is dyadic and every d2 below is exact in fp32; the rounding of mu
    leaves filt_lb within ~1e-4 of d2 in distance.  On top: an exact tie b' = alpha a + (1 - alpha) m' (m' = m with two
    bins swapped where a is 0: the same d2 to a, another record), and a duplicate of b.
    Anchors a: every one-hot descriptor at the bins of least mu (|a - mu| = 220.5) and near it, and random ones.
    fi = the b's (the base of the forward search) plus fillers, fj = the anchors."""
    m = dyadic_mu()
    mu = FB_MU.astype(np.float64).reshape(3, 11)
    lo = [np.argsort(mu[b])[:3] for b in range(3)]  # bins of least mu per block
    X = one_hot_extremes()
    hot = X.reshape(-1, 3, 11).argmax(2)
    ext = X[np.isin(hot[:, 0], lo[0]) & np.isin(hot[:, 1], lo[1]) & np.isin(hot[:, 2], lo[2])]
    A = np.concatenate([ext, random_desc(rng, n_random, conc=1.5)]).astype(np.float64)
    base = []
    for a in A:
        for al in alphas:
            b = al * a + (1 - al) * m
            base += [b, b]  # a duplicate: one run in the tile, or two heads when a tile border cuts it
            for blk in rng.permutation(3):
                z = 11 * blk + np.flatnonzero((a[11 * blk:11 * blk + 11] == 0) & (m[11 * blk:11 * blk + 11] > 0))
                pair = [(k, l) for k in z for l in z if k < l and m[k] != m[l]]
                if pair:
                    k, l = pair[rng.integers(len(pair))]
                    m2 = m.copy()
                    m2[k], m2[l] = m[l], m[k]
                    base.append(al * a + (1 - al) * m2)
                    break
    base = np.array(base)
    assert np.array_equal(base.astype(np.float32).astype(np.float64), base), "a bin is not exact in fp32"
    fi = np.concatenate([base.astype(np.float32), random_desc(rng, 200, conc=1.0)])
    return fi[rng.permutation(len(fi))], A.astype(np.float32)


def bound_approach(Q, B, okB=None):
    """sqrt(filt_lb) - sqrt(d2) of every query's winner and its exact-tie members with d2 > 0 (the pairs the filter must
    let through), from the emulated filter coordinates: -> array of one value per such pair.  A value above -4e-3 is a
    pair inside filt_bound's allowance, where a filter without its margin could drop the winner."""
    okB = usable(B) if okB is None else okB
    P, Pq = filter_coords(B), filter_coords(Q)
    out = []
    for q in np.flatnonzero(usable(Q)):
        d = d2_fp32(np.repeat(Q[q:q + 1], len(B), 0), B)
        d[~okB] = np.inf
        mn = d.min()
        if not np.isfinite(mn) or mn == 0:
            continue
        ties = np.flatnonzero(d == mn)
        lb = filt_lb(np.repeat(Pq[q:q + 1], len(ties), 0), P[ties]).astype(np.float64)
        out.append(np.sqrt(lb) - np.sqrt(d[ties].astype(np.float64)))
    return np.concatenate(out) if out else np.zeros(0)


class Case:
    def __init__(self, name, fi, fj, thrs=(35.0,)):
        self.name, self.fi, self.fj, self.thrs = name, np.asarray(fi, np.float32), np.asarray(fj, np.float32), tuple(thrs)


def _eps_moves(c, m, eps=2.0 ** -10):
    """m pairs of +eps / -eps in block 0 (bins 0..2m-1, each >= 1 in c): adds 2 m eps^2 to a d2, summed first."""
    d = c.copy()
    for p in range(m):
        d[2 * p] += eps
        d[2 * p + 1] -= eps
    return d


def tie_lattice(seed, n_centres=12, n_moves=3, shuffle=True):
    """Centres and every unit move around them (exact d2 = 2 ties between distinct records, spread over tiles by their
    filter coordinates), plus two-unit moves (d2 = 8) as fillers.  fi = moves in a random row order, fj = the centres and
    some moves."""
    rng = np.random.default_rng(seed)
    C = random_desc(rng, n_centres, conc=3.0)
    base, fillers = [], []
    for c in C:
        base.append(unit_moves(c))
        f = unit_moves(c)
        f = f + (f - c)  # +2 / -2: may leave the domain where c has a 1; keep those in the domain
        fillers.append(f[(f >= 0).all(1)])
    fi = np.concatenate(base + fillers)
    if shuffle:
        fi = fi[rng.permutation(len(fi))]
    fj = np.concatenate([C, fi[rng.choice(len(fi), n_moves * n_centres, replace=False)]])
    return fi, fj


def reverse_tie_lattice(seed, n_centres=20):
    """The tie lattice seen from the other side: fj = every unit move around the centres (the reverse search from a centre
    meets an exact d2 = 2 tie among them, spread over fj's tiles), fi = the centres among random fillers, so that the
    centres' query blocks in fi start at all kinds of tiles."""
    rng = np.random.default_rng(seed)
    C = random_desc(rng, n_centres, conc=3.0)
    fj = np.concatenate([unit_moves(c) for c in C])
    fj = fj[rng.permutation(len(fj))]
    fi = np.concatenate([C, random_desc(rng, len(fj), conc=0.7)])
    return fi[rng.permutation(len(fi))], fj


def crafted_cases():
    rng = np.random.default_rng(5)
    cases = []
    # exact ties between records in different tiles, lower index visited later (coverage asserted by the test)
    for s in range(3):
        fi, fj = tie_lattice(100 + s, n_moves=(3, 30, 60)[s])
        cases.append(Case("tie_lattice_%d" % s, fi, fj))
    fi, fj = reverse_tie_lattice(200)
    cases.append(Case("reverse_tie_lattice", fi, fj))
    # near-tight projected bounds (every pair within ~1e-3 of filt_lb = d2), exact ties on top, one-hot extremes
    fi, fj = projected_tight(rng)
    cases.append(Case("projected_tight_and_extremes", fi, fj))
    # the gate: d2 = 16 exactly, 16 + 2^-19 (next float), 16 + 2^-18, 16 + 3 * 2^-19, and 0; thresholds around them
    cen = random_desc(rng, 24, conc=4.0)
    cen[:, :6] = np.maximum(cen[:, :6], 1)
    for r in cen:  # block 0 may now sum above 100: take the surplus from its largest bin among 6..10
        blk = r[:11]
        k = 6 + np.argmax(blk[6:])
        blk[k] -= blk.sum() - 100
    cen = cen[(cen >= 0).all(1) & (cen[:, 11:22] >= 2).sum(1).astype(bool)]
    gi, gj = [], []
    for n, r in enumerate(cen):
        two = r.copy()
        bins = 11 + np.flatnonzero(r[11:22] >= 2)[:2]
        if len(bins) < 2:
            continue
        two[bins[0]] -= 2
        two[bins[1]] -= 2
        two[11 + np.setdiff1d(np.arange(11), bins - 11)[:2]] += 2  # d2 = 16: four bins moved by 2
        gj.append(r)
        gi.append(_eps_moves(two, n % 4) if n % 5 else r)  # n % 5 == 0: an identical record (d2 = 0)
    thr_up = float(np.nextafter(np.float32(4), np.float32(5)))
    cases.append(Case("gate", np.array(gi), np.array(gj), thrs=(4.0, float(np.nextafter(np.float32(4), np.float32(0))), thr_up,
                                                             0.0, 1e20, float("nan"))))
    # identical-descriptor runs longer than a tile, cut by tile borders, interleaved in row order with other records
    R = random_desc(rng, 3, conc=2.0)
    others = random_desc(rng, 400, conc=2.0)
    rows = np.concatenate([np.repeat(R, 150, 0), others])
    fi = rows[rng.permutation(len(rows))]
    fj = np.concatenate([R, unit_moves(R[0])[:60], others[:40]])
    cases.append(Case("long_identical_runs", fi, fj))
    # a run split by a record with the same 32-bit sort key (28-bit code + 4 hash bits) but other bins
    key = sort_keys(R[1:2])[0]
    mate = None
    for t in range(4000):
        cand = R[1].copy()
        a, b = rng.choice(11, 2, replace=False)
        if cand[a] < 1:
            continue
        e = 2.0 ** -int(rng.integers(6, 12))
        cand[a] -= e
        cand[b] += e
        if sort_keys(cand[None])[0] == key:
            mate = cand
            break
    assert mate is not None, "no sort-key collision found"
    fi = np.concatenate([np.repeat(R[1:2], 30, 0), mate[None], np.repeat(R[1:2], 30, 0), others[:100]])
    fj = np.concatenate([R[1:2], mate[None], others[:20]])
    cases.append(Case("run_split_by_key_collision", fi, fj))
    # first-hit / mutual structure: many j on one i; rnn(i) a j other than the first hit; rnn(i) tied with the first hit
    c0, c1 = random_desc(rng, 2, conc=3.0)
    mv = unit_moves(c0)
    fi = np.concatenate([c0[None], mv[40:41], c1[None], others[200:260]])  # mv[40] is an fi record too
    far = mv[:30] + (mv[:30] - c0)
    far = far[(far >= 0).all(1)]
    fj = np.concatenate([far,                 # j reaching c0 (d2 = 8), the lowest js: first hits, not rnn(c0)
                         mv[40:41],           # d2 = 0 to fi row 1, d2 = 2 to c0: rnn(c0) ties here at a lower j ...
                         mv[41:42],           # ... than this one, whose nn is c0 (d2 = 2)
                         c1[None], c1[None], others[200:210]])
    cases.append(Case("first_hit_and_mutual", fi, fj))
    # unusable rows: mixed; a whole 128-query block of them (sorted last); a base with no usable row; a base of one run
    U = random_desc(rng, 300, conc=1.5)
    fi = U.copy()
    fi[rng.choice(300, 70, replace=False)] = 0
    fj = np.concatenate([U[:128], np.zeros((128, 33), np.float32), U[128:150]])
    cases.append(Case("unusable_mixed_and_whole_block", fi, fj))
    cases.append(Case("base_without_usable_rows", np.zeros((90, 33), np.float32), U[:50]))
    cases.append(Case("base_one_run", np.repeat(U[:1], 200, 0), np.concatenate([U[:1], U[1:40]])))
    return cases


def size_cases():
    rng = np.random.default_rng(9)
    out = []
    sizes = [1, 2, 63, 64, 65, 127, 128, 129]
    for ni in sizes:
        for nj in sizes:
            if nj <= ni:
                fi = random_desc(rng, ni, conc=1.0)
                fj = np.concatenate([fi[rng.choice(ni, nj // 2, replace=True)], random_desc(rng, nj - nj // 2)])
                out.append(Case("n%d_%d" % (ni, nj), fi, fj))
    for t in (1, 2, 3, 8, 9, 40, 41, 73):
        ni = 64 * t - (t % 3) * 17  # partial last tiles
        fi = random_desc(rng, ni, conc=1.0)
        order = sorted_order(fi)
        ends = np.concatenate([order[:3], order[-3:]])  # copies of records in the first and last tiles
        nj = min(ni, 150)
        fj = np.concatenate([fi[ends], fi[rng.choice(ni, nj - len(ends) - nj // 3)], random_desc(rng, nj // 3)])[:nj]
        out.append(Case("tiles%d" % t, fi, fj))
    return out
