"""The oracle's TEASER++ solve on a correspondence set larger than 8192, against a numpy restatement of its graph steps:
TIM graph, core numbers by one-at-a-time peeling, the (core desc, degree desc, index asc) order and the greedy clique
grown from every start (largest first, lowest rank on ties)."""
import numpy as np

from test_gpu_quatro_big import synthetic_set


def _greedy_clique_numpy(S, D, noise_bound=0.3):
    dS = np.sqrt(((S[None, :, :] - S[:, None, :]) ** 2).sum(-1))
    dD = np.sqrt(((D[None, :, :] - D[:, None, :]) ** 2).sum(-1))
    adj = np.abs(dS - dD) <= 2 * noise_bound
    np.fill_diagonal(adj, False)
    n = len(S)
    deg = adj.sum(1)
    d, alive, core, k = deg.copy(), np.ones(n, bool), np.zeros(n, np.int64), 0
    big = np.iinfo(np.int64).max
    for _ in range(n):
        v = int(np.argmin(np.where(alive, d, big)))
        k = max(k, int(d[v]))
        core[v], alive[v] = k, False
        d[adj[v] & alive] -= 1
    order = np.lexsort((np.arange(n), -deg, -core))
    radj = adj[order][:, order]
    best = []
    for r in range(n):
        if core[order[r]] + 1 <= len(best):  # cannot be strictly larger than a clique found at a lower rank
            continue
        P, C = radj[r].copy(), [r]
        while True:
            u = int(P.argmax())
            if not P[u]:
                break
            C.append(u)
            P &= radj[u]
        if len(C) > len(best):
            best = C
    return np.sort(order[best])


def test_oracle_solve_beyond_8192_matches_numpy(oracle, synth):
    n = 9000
    S, D, Texp = synthetic_set(n, seed=n)
    o = oracle.quatro_solve(S, D, np.repeat(np.arange(n, dtype=np.int32)[:, None], 2, 1))
    clique = _greedy_clique_numpy(S[:, :3].astype(np.float64), D[:, :3].astype(np.float64))
    assert np.array_equal(o["clique"], clique)
    assert o["valid"] and len(clique) >= 300
    rot, tr = synth.se3_error(o["T"], Texp)
    assert rot < 1e-2 and tr < 0.1
