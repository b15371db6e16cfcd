#!/usr/bin/env python
"""CPU emulation of knn_walk's traversal STACK (knn.cuh) on the bench's pairs: how deep does it get?

Same tree as profiles/emulate_knn_seeding.py (30-bit Morton order, Karras splits, <= 8-point leaves), walked per query as
knn_walk does (near child first, the far child pushed unless its bound is strictly greater than the current worst, strict
'>' pruning on pop).  Records the live stack depth at every push and the largest depth of every query, for three walks:

  cov15     the 15-NN self-queries of k_covariance<15>, seeded with the 15-point Morton window around the query
  unseeded  k_gicp_search's first correspondence pass: bound = +inf until the first leaf, so every far child on the way
            down is pushed
  seeded    k_gicp_search's later passes: the query moved by a small pose update, seeded with the previous pass's
            nearest neighbour

Prints, per walk, the distribution of the per-query maximum depth and the share of queries and of pushes that go deeper
than S for S in 2..16: the numbers behind the on-chip stack size chosen per kernel (DESIGN.md §3).

    python profiles/emulate_stack_depth.py [n_points] [n_queries] [seed]
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "fast-lio-sam-qn_b200"))
_spec = importlib.util.spec_from_file_location("emulate_knn_seeding", os.path.join(HERE, "emulate_knn_seeding.py"))
eks = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(eks)
K = 15


def walk(P, nodes, root, q, k, seeds, skip=()):
    """knn_walk with the result set seeded by `seeds`; returns (max depth, depth at every push)."""
    best = sorted((float(((P[s] - q) ** 2).sum()), s) for s in set(seeds))[:k]
    seen = set(seeds)

    def worst():
        return best[-1][0] if len(best) == k else np.inf

    def offer(pos):
        d2 = float(((P[pos] - q) ** 2).sum())
        if len(best) < k or (d2, pos) < best[-1]:
            if len(best) == k:
                best.pop()
            best.append((d2, pos))
            best.sort()

    stack, pushes, deepest = [], [], 0
    ref, dnode = root, 0.0
    while True:
        alive = not (dnode > worst())
        while alive and ref >= 0:
            lo0, hi0, r0, lo1, hi1, r1 = nodes[ref]
            d0, d1 = eks.box_d2(q, lo0, hi0), eks.box_d2(q, lo1, hi1)
            if d1 < d0:
                r0, r1, d0, d1 = r1, r0, d1, d0
            if not (d1 > worst()):
                stack.append((r1, d1))
                pushes.append(len(stack))
                deepest = max(deepest, len(stack))
            ref, dnode = r0, d0
            alive = not (d0 > worst())
        if alive:
            c = -1 - ref
            a, cnt = c >> 4, c & 15
            for pos in range(a, a + cnt):
                if pos not in seen and pos not in skip:
                    offer(pos)
        found = False
        while stack:
            ref, dnode = stack.pop()
            if not (dnode > worst()):
                found = True
                break
        if not found:
            break
    return deepest, pushes


def nearest(P, nodes, root, q):
    best = [np.inf, -1]
    stack = [(root, 0.0)]
    while stack:
        ref, d = stack.pop()
        if d > best[0]:
            continue
        if ref < 0:
            c = -1 - ref
            a, cnt = c >> 4, c & 15
            d2 = ((P[a:a + cnt] - q) ** 2).sum(1)
            j = int(np.argmin(d2))
            if d2[j] < best[0]:
                best = [float(d2[j]), a + j]
            continue
        lo0, hi0, r0, lo1, hi1, r1 = nodes[ref]
        stack.append((r1, eks.box_d2(q, lo1, hi1)))
        stack.append((r0, eks.box_d2(q, lo0, hi0)))
    return best[1]


def report(name, deepest, pushes):
    deepest, pushes = np.asarray(deepest), np.asarray(pushes)
    print("%-9s queries %d, pushes/query %.1f, max depth per query: p50 %d  p90 %d  p99 %d  max %d" %
          (name, len(deepest), len(pushes) / len(deepest), np.percentile(deepest, 50), np.percentile(deepest, 90),
           np.percentile(deepest, 99), deepest.max()))
    print("          S:                   " + " ".join("%6d" % s for s in range(2, 17, 2)))
    print("          queries deeper than S " + " ".join("%5.1f%%" % (100 * (deepest > s).mean()) for s in range(2, 17, 2)))
    print("          pushes deeper than S  " + " ".join("%5.1f%%" % (100 * (pushes > s).mean() if len(pushes) else 0) for s in range(2, 17, 2)))


def main():
    from b200reg import synth
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
    nq = int(sys.argv[2]) if len(sys.argv) > 2 else 2048
    seed = int(sys.argv[3]) if len(sys.argv) > 3 else 1000  # the bench's first pair
    src, dst, _ = synth.make_pair(seed, n, n)
    Ps, nodes_s, root_s = eks.build(src[:, :3].astype(np.float64))
    Pt, nodes_t, root_t = eks.build(dst[:, :3].astype(np.float64))
    rng = np.random.default_rng(0)
    starts = rng.integers(0, len(Ps) - 64, nq // 32)
    qs = np.concatenate([np.arange(s, s + 32) for s in starts])  # whole warps of Morton-consecutive queries
    print("pair seed %d: %d / %d points, tree depth <= %d records" % (seed, len(Ps), len(Pt), 64))

    def window(i):
        lo = max(0, i - K // 2)
        hi = min(len(Ps) - 1, lo + K - 1)
        lo = max(0, hi - (K - 1))
        return lo, hi

    deep, push = [], []
    for i in qs:
        lo, hi = window(i)
        d, p = walk(Ps, nodes_s, root_s, Ps[i], K, list(range(lo, hi + 1)), set(range(lo, hi + 1)))
        deep.append(d)
        push += p
    report("cov15", deep, push)

    # the LM's first pass queries the source at the identity guess; a later pass queries it after a small pose update
    # (1 cm, 0.05 deg about z) and starts from the previous pass's nearest neighbour
    a = np.deg2rad(0.05)
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    deep_u, push_u, deep_s, push_s = [], [], [], []
    for i in qs:
        q0 = Ps[i]
        d, p = walk(Pt, nodes_t, root_t, q0, 1, [])
        deep_u.append(d)
        push_u += p
        prev = nearest(Pt, nodes_t, root_t, q0)
        q1 = Rz @ q0 + np.array([0.01, 0.0, 0.0])
        d, p = walk(Pt, nodes_t, root_t, q1, 1, [prev])
        deep_s.append(d)
        push_s += p
    report("unseeded", deep_u, push_u)
    report("seeded", deep_s, push_s)


if __name__ == "__main__":
    main()
