"""An fp64 restatement of the TEASER++ solve in QUATRO / PMC_HEU mode, numpy and the math module only, and the crafted
correspondence sets that drive the solve to its edges.

It states what k_teaser_solve, the k_big_* chain (fast-lio-sam-qn_b200/csrc/quatro.cu) and the CPU oracle compute, from
TEASER++'s published algorithm (Yang, Shi, Carlone, "TEASER: Fast and Certifiable Point Cloud Registration", T-RO 2020;
the QUATRO yaw-only rotation of Lim et al., ICRA 2022):

* the TIM graph: correspondences i < j are consistent when | ||D_j - D_i|| - ||S_j - S_i|| | <= 2 * noise_bound (cbar2 = 1);
* core numbers by peeling one minimum-degree vertex at a time (lowest index on ties);
* the clique order (core desc, degree desc, index asc), and the greedy clique grown from every start vertex; the largest
  clique wins, the lowest start rank on ties;
* the chain TIMs between consecutive clique members (ascending index) and the weighted 2-D Kabsch step, whose optimal
  rotation is the angle atan2(H01 - H10, H00 + H11) of H = sum w x y^T;
* GNC-TLS on the yaw: mu from the first residuals, the ``mu <= 0`` exit, the ``nb2 < 1e-16`` floor, weights and the
  cost-difference stop;
* per-axis TLS adaptive voting over the interval ends x_i -+ noise_bound, sorted by value with ties in slot order
  (+ end of i at slot 2i, - end at 2i + 1).

Every sum is a sequential Python loop in the order the oracle uses, and the transcendental functions are the C library's
(math.atan2 / cos / sin), so against the oracle the only differences left would be its own mistakes.  The device sums
in a fixed tree order and uses CUDA's atan2 / cos / sin, which is what its 1e-9 tolerance is for.

The switches (``strict``, ``prefer``, ``tie``, ``mu_exit``, ``nb2_floor``) state the wrong rule next to the right one:
each crafted case shows that flipping its switch changes the answer, so a kernel that got that rule wrong would fail.
"""
import math
from dataclasses import dataclass, field

import numpy as np

INF = float("inf")


def _div(a, b):
    """IEEE fp64 division (x / 0 is +-inf or NaN, as in C++), which Python floats do not give."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(a) / np.float64(b))


# ---- graph steps --------------------------------------------------------------------------------------------------
def tim_graph(S, D, noise_bound, strict=False):
    """Adjacency (n, n) bool of the TIM consistency graph; the squared lengths are summed x, y, z in that order."""
    S = np.asarray(S, np.float64)
    D = np.asarray(D, np.float64)
    a = np.zeros((len(S), len(S)))
    b = np.zeros((len(S), len(S)))
    for d in range(3):
        da = S[None, :, d] - S[:, None, d]
        db = D[None, :, d] - D[:, None, d]
        a = a + da * da
        b = b + db * db
    gap = np.abs(np.sqrt(a) - np.sqrt(b))
    beta = 2.0 * noise_bound
    adj = gap < beta if strict else gap <= beta
    np.fill_diagonal(adj, False)
    return adj


def core_numbers(adj):
    n = len(adj)
    d = adj.sum(1).astype(np.int64)
    alive = np.ones(n, bool)
    core = np.zeros(n, np.int64)
    k = 0
    big = np.iinfo(np.int64).max
    for _ in range(n):
        v = int(np.argmin(np.where(alive, d, big)))  # argmin: the lowest index among the minima
        k = max(k, int(d[v]))
        core[v], alive[v] = k, False
        d[adj[v] & alive] -= 1
    return core


def clique_order(adj, core, index_desc=False):
    """Vertices by (core desc, degree desc, index asc) -- index desc is the wrong rule, for the probes."""
    n = len(adj)
    idx = -np.arange(n) if index_desc else np.arange(n)
    return np.lexsort((idx, -adj.sum(1), -core))


def greedy_clique(adj, prefer="lowest", index_desc=False):
    """The greedy clique grown from every start rank; the largest wins, on ties the lowest start rank ("highest" is the
    wrong rule).  Returns the members, ascending."""
    n = len(adj)
    if n == 0:
        return np.zeros(0, np.int64)
    core = core_numbers(adj)
    order = clique_order(adj, core, index_desc)
    radj = adj[order][:, order]
    best = []
    for r in range(n):
        # a clique grown from r has at most core(r) + 1 members: skip starts that cannot win
        if core[order[r]] + 1 < len(best) or (prefer == "lowest" and core[order[r]] + 1 == len(best)):
            continue
        P, C = radj[r].copy(), [r]
        while True:
            u = int(P.argmax())  # the first candidate in the clique order
            if not P[u]:
                break
            C.append(u)
            P &= radj[u]
        if len(C) > len(best) or (prefer == "highest" and len(C) == len(best)):
            best = C
    return np.sort(order[best])


def _greedy_clique_numpy(S, D, noise_bound=0.3):
    return greedy_clique(tim_graph(S, D, noise_bound))


# ---- continuous steps ---------------------------------------------------------------------------------------------
def kabsch_yaw(X, Y, W):
    """Weighted 2-D Kabsch: the rotation R maximising sum w_k y_k . R x_k, as (cos, sin) of its angle."""
    h00 = h01 = h10 = h11 = 0.0
    for (x0, x1), (y0, y1), w in zip(X, Y, W):
        h00 += x0 * w * y0
        h01 += x0 * w * y1
        h10 += x1 * w * y0
        h11 += x1 * w * y1
    th = math.atan2(h01 - h10, h00 + h11)
    return math.cos(th), math.sin(th), (h00, h01, h10, h11)


def gnc_tls_yaw(A, B, noise_bound, gnc_factor, cost_thr, max_iter, mu_exit=True, nb2_floor=True):
    """GNC-TLS over the chain TIMs A -> B (3-D, the yaw fitted on x, y).  Returns (cos, sin, iterations)."""
    nt = len(A)
    X = [(float(a[0]), float(a[1])) for a in A]
    Y = [(float(b[0]), float(b[1])) for b in B]
    W = [1.0] * nt
    res = [0.0] * nt
    nb2 = noise_bound * noise_bound
    if nb2_floor and nb2 < 1e-16:
        nb2 = 1e-2
    mu, prev_cost = 1.0, INF
    cs, sn, iters = 1.0, 0.0, 0
    for it in range(max_iter):
        iters = it + 1
        cs, sn, _ = kabsch_yaw(X, Y, W)
        maxres = 0.0
        for k in range(nt):
            ax, ay, az = (float(v) for v in A[k])
            bx, by, bz = (float(v) for v in B[k])
            rx = bx - (cs * ax + -sn * ay)
            ry = by - (sn * ax + cs * ay)
            rz = bz - az
            res[k] = rx * rx + ry * ry + rz * rz
            maxres = max(maxres, res[k])
        if it == 0:
            mu = _div(1.0, _div(2.0 * maxres, nb2) - 1.0)
            if mu_exit and mu <= 0:
                break
        th1 = _div(mu + 1, mu) * nb2
        th2 = _div(mu, mu + 1) * nb2
        cost = 0.0
        for k in range(nt):
            cost += W[k] * res[k]
            if res[k] >= th1:
                W[k] = 0.0
            elif res[k] <= th2:
                W[k] = 1.0
            else:
                W[k] = float(np.sqrt(np.float64(_div(nb2 * mu * (mu + 1), res[k])))) - mu
        diff = abs(cost - prev_cost)
        mu *= gnc_factor
        prev_cost = cost
        if diff < cost_thr:
            break
    return cs, sn, iters


def tls_entries(x, rng, tie="stable"):
    """The 2m interval ends (value, eps, member), sorted by value; equal values in slot order ("reversed": the wrong rule)."""
    ends = []
    for i, v in enumerate(x):
        ends.append((v - rng, 2 * i, 1, i))
        ends.append((v + rng, 2 * i + 1, -1, i))
    sgn = 1 if tie == "stable" else -1
    ends.sort(key=lambda e: (e[0], sgn * e[1]))
    return [(e[0], e[2], e[3]) for e in ends]


def tls_estimate(x, rng, tie="stable"):
    """TEASER++'s scalar TLS estimator by adaptive voting: the consensus set of every elementary interval, the weighted
    mean of its members and its cost; the first strictly smallest cost wins (an empty set gives NaN and never wins)."""
    x = [float(v) for v in x]
    w = _div(1.0, rng * rng)
    ris, dxw, dwc, sxi, sxq, card = rng * len(x), 0.0, 0.0, 0.0, 0.0, 0
    best_cost, best = INF, 0.0
    for _, eps, i in tls_entries(x, rng, tie):
        card += eps
        dwc += eps * w
        dxw += eps * w * x[i]
        ris -= eps * rng
        sxi += eps * x[i]
        sxq += eps * x[i] * x[i]
        xh = _div(dxw, dwc)
        cost = (card * xh * xh + sxq - 2 * sxi * xh) + ris
        if cost < best_cost:
            best_cost, best = cost, xh
    return best


@dataclass
class Params:
    noise_bound: float = 0.3
    gnc_factor: float = 1.4
    cost_thr: float = 1e-4
    max_iter: int = 50


def solve(S, D, prm=Params(), **rules):
    """The whole solve on correspondences i = (S[i], D[i]) (fp32 values, fp64 arithmetic) -> (valid, clique, gnc_iters, T).
    rules: strict, prefer, index_desc, mu_exit, nb2_floor, tie -- the wrong variants, for the probes."""
    S = np.asarray(S, np.float32)[:, :3].astype(np.float64)
    D = np.asarray(D, np.float32)[:, :3].astype(np.float64)
    T = np.eye(4)
    if len(S) == 0:
        return False, np.zeros(0, np.int64), 0, T
    adj = tim_graph(S, D, prm.noise_bound, rules.get("strict", False))
    clique = greedy_clique(adj, rules.get("prefer", "lowest"), rules.get("index_desc", False))
    if len(clique) <= 1:
        return False, clique, 0, T
    A = S[clique[1:]] - S[clique[:-1]]
    B = D[clique[1:]] - D[clique[:-1]]
    cs, sn, iters = gnc_tls_yaw(A, B, prm.noise_bound, prm.gnc_factor, prm.cost_thr, prm.max_iter,
                                rules.get("mu_exit", True), rules.get("nb2_floor", True))
    T[0, 0], T[0, 1], T[1, 0], T[1, 1] = cs, -sn, sn, cs
    for d in range(3):
        x = []
        for c in clique:
            rs = (cs * S[c, 0] + -sn * S[c, 1]) if d == 0 else ((sn * S[c, 0] + cs * S[c, 1]) if d == 1 else S[c, 2])
            x.append(D[c, d] - rs)
        T[d, 3] = tls_estimate(x, prm.noise_bound, rules.get("tie", "stable"))
    return True, clique, iters, T


# ---- crafted sets -------------------------------------------------------------------------------------------------
@dataclass
class Case:
    """A correspondence set meant to reach one rule of the solve.  `probe(case)` returns True when the set really pins
    that rule: the restatement with the rule flipped gives another answer (or the reached state holds, where no wrong
    variant exists)."""
    name: str
    S: np.ndarray
    D: np.ndarray
    reaches: str
    probe: object
    prm: Params = field(default_factory=Params)

    @property
    def n(self):
        return len(self.S)

    def solve(self, **rules):
        key = tuple(sorted(rules.items()))
        cache = self.__dict__.setdefault("_cache", {})
        if key not in cache:
            cache[key] = solve(self.S, self.D, self.prm, **rules)
        return cache[key]


def _f32(a):
    a = np.asarray(a, np.float64)
    assert np.array_equal(a.astype(np.float32).astype(np.float64), a), "crafted coordinates must be exact in fp32"
    return a.astype(np.float32)


def _yaw(S, yaw, t):
    S = np.asarray(S, np.float64)
    c, s = math.cos(yaw), math.sin(yaw)
    D = np.c_[c * S[:, 0] - s * S[:, 1], s * S[:, 0] + c * S[:, 1], S[:, 2]] + np.asarray(t, np.float64)
    return D.astype(np.float32)


def _differs(a, b):
    return (a[0] != b[0] or not np.array_equal(a[1], b[1]) or a[2] != b[2]
            or not np.array_equal(a[3], b[3]))


def natural_set(n, seed, n_in=None, noise=0.02, yaw=0.3, t=(4.0, -2.5, 0.4)):
    """n correspondences: n_in inliers of a yaw + shift (plus uniform noise), the rest random pairs in a 120 x 120 x 12 m
    box.  Returns (S, D) as float32."""
    rng = np.random.default_rng(seed)
    n_in = n // 3 if n_in is None else n_in
    S = rng.uniform([-60, -60, -3], [60, 60, 9], (n, 3))
    D = rng.uniform([-60, -60, -3], [60, 60, 9], (n, 3))
    inl = rng.choice(n, n_in, replace=False)
    D[inl] = _yaw(S[inl], yaw, t) + rng.uniform(-noise, noise, (n_in, 3))
    return S.astype(np.float32), D.astype(np.float32)


def beta_margin(S, D, noise_bound):
    """Smallest distance of any TIM gap from 2 * noise_bound: sets meant to be rounding-proof keep it well above 1e-9."""
    S = np.asarray(S, np.float64)
    D = np.asarray(D, np.float64)
    dS = np.sqrt(((S[None] - S[:, None]) ** 2).sum(-1))
    dD = np.sqrt(((D[None] - D[:, None]) ** 2).sum(-1))
    gap = np.abs(dS - dD)
    np.fill_diagonal(gap, np.inf)
    return float(np.abs(gap - 2 * noise_bound).min()) if len(S) > 1 else np.inf


def crafted_cases():
    nb = Params(noise_bound=0.25)
    cases = []

    def add(name, S, D, reaches, probe, prm=nb):
        cases.append(Case(name, _f32(S), _f32(D), reaches, probe, prm))

    line3 = [[0, 0, 0], [4, 0, 0], [8, 0, 0]]
    add("n1", [[1, 2, 3]], [[5, 6, 7]], "one correspondence: no TIM, clique 1, invalid, identity",
        lambda c: not c.solve()[0] and list(c.solve()[1]) == [0] and c.solve()[2] == 0)
    add("n2_consistent", [[0, 0, 0], [3, 0, 0]], [[1, 1, 1], [4, 1, 1]],
        "clique of exactly 2: one chain TIM, valid",
        lambda c: c.solve()[0] and len(c.solve()[1]) == 2)
    add("n2_inconsistent", [[0, 0, 0], [3, 0, 0]], [[0, 0, 0], [5, 0, 0]], "two inconsistent: clique 1, invalid",
        lambda c: not c.solve()[0] and len(c.solve()[1]) == 1)
    add("n3_triangle", line3, [[2, 1, 0.5], [6, 1, 0.5], [10, 1, 0.5]], "three consistent: clique 3, noise-free",
        lambda c: c.solve()[0] and len(c.solve()[1]) == 3)
    # TIM length gap exactly 2 * noise_bound: 3.5 - 3 = 0.5 = 2 * 0.25, kept by "<=", dropped by "<"
    add("gap_equal_beta", [[0, 0, 0], [3, 0, 0]], [[0, 0, 0], [3.5, 0, 0]], "TIM gap == 2 noise_bound is an edge (<=)",
        lambda c: len(c.solve()[1]) == 2 and len(c.solve(strict=True)[1]) == 1)
    over = float(np.nextafter(np.float32(3.5), np.float32(4)))
    add("gap_one_ulp_over", [[0, 0, 0], [3, 0, 0]], [[0, 0, 0], [over, 0, 0]], "TIM gap 1 fp32 ulp above 2 noise_bound: no edge",
        lambda c: len(c.solve()[1]) == 1 and beta_margin(c.S, c.D, 0.25) < 1e-6)
    # all pairwise gaps large: every greedy clique has size 1; rank 0 = index 0 wins, index desc would pick n - 1
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 3, 0], [0, 0, 9], [5, 5, 0], [-7, 2, 1]], np.float64)
    add("all_inconsistent", pts, pts * 4, "no edge at all: clique 1 (lowest index), invalid, identity",
        lambda c: not c.solve()[0] and list(c.solve()[1]) == [0] and list(c.solve(index_desc=True)[1]) == [5]
        and list(c.solve(prefer="highest")[1]) == [5])
    # two disjoint triangles, interleaved: a 2-regular graph, every (core, degree) key equal.  A = {0, 2, 4} (identity),
    # B = {1, 3, 5} (shifted 50 m): rank 0 = index 0 wins; the highest rank (index 5) would give B
    tri = np.array([[0, 0, 0], [4, 0, 0], [0, 2, 0]], np.float64)
    S2 = np.zeros((6, 3))
    D2 = np.zeros((6, 3))
    S2[0::2], D2[0::2] = tri, tri + [1, 0.5, 0]
    S2[1::2], D2[1::2] = tri + [0, 50, 0], tri + [0, 100, 0]

    def equal_cliques(c):
        adj = tim_graph(c.S, c.D, 0.25)
        core, deg = core_numbers(adj), adj.sum(1)
        lo, hi = c.solve()[1], c.solve(prefer="highest")[1]
        return (len(set(core)) == 1 and len(set(deg)) == 1 and list(lo) == [0, 2, 4] and list(hi) == [1, 3, 5]
                and list(c.solve(index_desc=True)[1]) == [1, 3, 5])
    add("equal_cliques_regular", S2, D2, "two disjoint maximal cliques of equal size, regular graph: the lowest rank wins",
        equal_cliques)
    # three disjoint 4-cliques (3-regular), the winner holds index 0
    sq = np.array([[0, 0, 0], [4, 0, 0], [0, 4, 0], [4, 4, 1]], np.float64)
    S3 = np.concatenate([sq + [0, 40 * g, 0] for g in range(3)])[np.argsort(np.tile(np.arange(4), 3), kind="stable")]
    D3 = np.concatenate([sq + [2, 40 * g * (g + 1), 0] for g in range(3)])[np.argsort(np.tile(np.arange(4), 3), kind="stable")]
    add("three_cliques_regular", S3, D3, "3-regular graph of three equal cliques: every key equal, lowest rank wins",
        lambda c: len(set(core_numbers(tim_graph(c.S, c.D, 0.25)))) == 1
        and not np.array_equal(c.solve()[1], c.solve(prefer="highest")[1]))
    # duplicate source points: zero-length chain TIMs in the clique
    Sd = np.array([[0, 0, 0], [0, 0, 0], [6, 0, 0], [6, 0, 0], [6, 4, 2]], np.float64)
    add("duplicate_points", Sd, Sd + [0.5, -1, 0.25], "duplicate points: zero-length TIMs (A = B = 0) in the clique",
        lambda c: len(c.solve()[1]) == 5 and (np.abs(np.diff(c.S[c.solve()[1]], axis=0)).sum(1) == 0).sum() == 2)
    # noise-free yaw 0: residuals exactly 0, mu = -1: the first iteration exits (without the exit: a second one)
    Sn = np.array([[0, 0, 0], [8, 0, 1], [2, 6, 0], [-4, 3, 2], [5, -5, 0.5]], np.float64)
    add("noise_free_yaw0", Sn, Sn + [3, -2, 0.5], "noise-free (yaw 0): mu <= 0 exit, gnc_iters == 1",
        lambda c: c.solve()[2] == 1 and c.solve(mu_exit=False)[2] != 1 and c.solve()[3][0, 1] == 0)
    # every TIM vertical: H = 0, atan2(0, 0) = 0
    Sv = np.array([[1, 2, 0], [1, 2, 3], [1, 2, -2], [1, 2, 7]], np.float64)
    add("vertical_tims", Sv, Sv + [4, -1, 0.5], "every TIM vertical: H == 0, atan2(0, 0) = 0, R = I",
        lambda c: kabsch_yaw([(0.0, 0.0)] * 3, [(0.0, 0.0)] * 3, [1.0] * 3)[:2] == (1.0, 0.0)
        and np.array_equal(c.solve()[3][:3, :3], np.eye(3)) and len(c.solve()[1]) == 4)
    # yaw +pi exactly (D = (-x, -y, z)): H01 - H10 == +0, atan2(+0, < 0) = +pi
    Sp = np.array([[0, 0, 0], [8, 0, 1], [2, 6, 0], [-4, 3, 2], [5, -5, 0.5]], np.float64)
    add("yaw_pi", Sp, np.c_[-Sp[:, 0], -Sp[:, 1], Sp[:, 2]] + [1, 2, 0], "yaw pi: atan2(+0, H00 + H11 < 0) = +pi",
        lambda c: c.solve()[3][1, 0] > 0 and abs(c.solve()[3][0, 0] + 1) < 1e-15)
    for sign in (1, -1):  # either side of atan2's branch cut: sin(yaw) changes sign
        yaw = sign * (math.pi - 1e-9)
        Sc = np.array([[0, 0, 0], [10, 0, 0], [0, 0.5, 0], [10, 0.5, 1]], np.float64)
        Dc = np.c_[math.cos(yaw) * Sc[:, 0] - math.sin(yaw) * Sc[:, 1], math.sin(yaw) * Sc[:, 0] + math.cos(yaw) * Sc[:, 1],
                   Sc[:, 2]].astype(np.float32).astype(np.float64)
        add("yaw_%spi_minus_1e-9" % ("+" if sign > 0 else "-"), Sc, Dc,
            "yaw %s(pi - 1e-9): the %s side of atan2's branch cut" % ("+" if sign > 0 else "-", "upper" if sign > 0 else "lower"),
            lambda c, sign=sign: np.sign(c.solve()[3][1, 0]) == sign and abs(math.atan2(c.solve()[3][1, 0], c.solve()[3][0, 0])) > math.pi - 1e-7)
    # TLS: members 0, 1 along x with x-translations 1 and 1.5 (R = I exactly): the + end of 1 and the - end of 0 meet at 1.25.
    # Slot order closes 0 first; the reversed tie order would see {0, 1} and return 1.25.  y, z: coinciding intervals.
    add("tls_touching", line3[:2], [[1, 2, 0.5], [5.5, 2, 0.5]], "TLS: x_i + r == x_j - r, ties in slot order",
        lambda c: c.solve()[3][0, 3] == 1.0 and c.solve(tie="reversed")[3][0, 3] == 1.25
        and np.array_equal(c.solve()[3][:3, :3], np.eye(3)))
    # members with x-translations 1, 1.5, 1.5: two coinciding intervals that touch a third
    add("tls_coincide_touching", line3, [[1, 2, 0.5], [5.5, 2, 0.5], [9.5, 2, 0.5]],
        "TLS: coinciding intervals touching a third, ties in slot order",
        lambda c: c.solve()[3][0, 3] == 1.5 and c.solve(tie="reversed")[3][0, 3] != 1.5)
    # noise_bound 1e-9: nb2 = 1e-18 is floored to 1e-2.  D = S turned 90 deg about x: every TIM length exact, the yaw fit
    # leaves residuals < 5e-3, so with the floor mu < 0 (one iteration) and without it GNC keeps going
    Sf = np.array([[0, 0, 0], [8, 1 / 256, 1 / 128], [16, 1 / 128, 0], [24, 3 / 256, 1 / 256], [32, 0, 1 / 64]], np.float64)
    add("nb2_floor", Sf, np.c_[Sf[:, 0], -Sf[:, 2], Sf[:, 1]] + [2, 1, 0], "noise_bound 1e-9: the nb2 < 1e-16 floor",
        lambda c: c.solve()[2] == 1 and _differs(c.solve(), c.solve(nb2_floor=False)) and len(c.solve()[1]) == 5,
        Params(noise_bound=1e-9))
    # rot_max_iter 0 / 1 and cost_thr 0 on a noisy yawed set whose GNC takes several iterations
    Sg, Dg = natural_set(40, 11, n_in=30, noise=0.1)
    base = Params(noise_bound=0.3)
    add("max_iter_0", Sg, Dg, "rot_max_iter 0: no GNC iteration, R = I, valid",
        lambda c: c.solve()[0] and c.solve()[2] == 0 and np.array_equal(c.solve()[3][:3, :3], np.eye(3))
        and beta_margin(c.S, c.D, 0.3) > 1e-6, Params(noise_bound=0.3, max_iter=0))
    add("max_iter_1", Sg, Dg, "rot_max_iter 1: the cap stops GNC after one iteration",
        lambda c: c.solve()[2] == 1 and solve(c.S, c.D, base)[2] > 1, Params(noise_bound=0.3, max_iter=1))
    add("cost_thr_0", Sg, Dg, "cost_thr 0: GNC runs to rot_max_iter",
        lambda c: c.solve()[2] == 50 and solve(c.S, c.D, base)[2] < 50, Params(noise_bound=0.3, cost_thr=0.0))
    # the shared solver's 512 slots: bitonic sorts of 512 keys and 1024 interval ends, full bit rows
    for n in (509, 510, 511, 512):
        S, D = natural_set(n, n, n_in=n // 2)
        add("size_%d" % n, S, D, "%d correspondences: the shared solver near its 512 slots" % n,
            lambda c: c.solve()[0] and len(c.solve()[1]) >= c.n // 2 and beta_margin(c.S, c.D, 0.3) > 1e-6,
            Params(noise_bound=0.3))
    return cases
