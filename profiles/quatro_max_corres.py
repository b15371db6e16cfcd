#!/usr/bin/env python
"""optimizedMatching across max_corres: how many correspondences it keeps and what the selection and the solve cost.

Inputs: a 0.3 m-voxelised 100k x 100k pair (synth.make_pair(2003, ..., mode="quatro", voxel=0.3)) and the 11-keyframe
0.2 m sub-map pair of quatro_big_solve.py.  For max_corres in {200, 509, 1000, 2000, 4000, 8189}: n_mutual, n_corr,
clique size; the device time of k_tuple_select, of k_teaser_solve (sets of at most 512) and of the global-memory chain
k_big_* (larger sets), from torch.profiler CUDA activity of one call; the median wall time of the whole
b200reg_quatro_align call over --reps calls after one warm-up (descriptors already on the device); and, with --oracle,
the CPU oracle's matcher and solve on the device's descriptors on one host thread.
Prints one JSON line per case, with the card's name and power limit read in the same run.
    python profiles/quatro_max_corres.py [--reps 5] [--oracle]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import b200reg  # noqa: E402
from b200reg import native, synth  # noqa: E402
from quatro_big_solve import gpu_info, kernel_ms, timed  # noqa: E402
from test_gpu_quatro_big import make_submap_pair  # noqa: E402

CAPS = (200, 509, 1000, 2000, 4000, 8189)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle", action="store_true")
    a = ap.parse_args()
    gpu = gpu_info()
    ctx = b200reg.Context(0)
    if a.oracle:
        from oracle import oracle as orc
    inputs = [("voxel0.3_100k", synth.make_pair(2003, 100000, mode="quatro", voxel=0.3)[:2]),
              ("submap0.2", make_submap_pair(leaf=0.2)[:2])]
    for name, (src, dst) in inputs:
        cs, cd = ctx.create_clouds([src, dst])
        ctx.fpfh([cs, cd])
        fs, fd = ctx.get_fpfh(cs)[1], ctx.get_fpfh(cd)[1]
        for mc in CAPS:
            prm = native.default_quatro_params()
            prm.max_corres = mc
            info = {}
            fn = lambda: info.update(ctx.quatro_align([cs], [cd], params=prm, want_corr=True)[0])  # noqa: E731
            med, lo, hi = timed(fn, a.reps)
            km = kernel_ms(fn)
            big = sum(v for k, v in km.items() if k.startswith("k_big_"))
            rec = dict(case=name, n_src=len(src), n_dst=len(dst), max_corres=mc, n_mutual=info["n_mutual"], n_corr=info["n_corr"],
                       clique=info["clique_size"], valid=info["valid"], solver="k_teaser_solve" if info["n_corr"] <= 512 else "k_big",
                       tuple_select_ms=km.get("k_tuple_select", 0.0), teaser_solve_ms=km.get("k_teaser_solve", 0.0), big_chain_ms=big,
                       kernel_ms=sum(km.values()), wall_ms_median=med, wall_ms_min=lo, wall_ms_max=hi, gpu=gpu)
            if a.oracle:
                p = orc.QuatroParams.default()
                p.max_corres = mc
                t0 = time.perf_counter()
                corr, _ = orc.match(src, dst, fs, fd, p)
                t1 = time.perf_counter()
                orc.quatro_solve(src, dst, corr, p)
                t2 = time.perf_counter()
                rec.update(oracle_match_ms=1e3 * (t1 - t0), oracle_solve_ms=1e3 * (t2 - t1),
                           oracle_same_corr=bool(np.array_equal(corr, info["corr"])))
            print(json.dumps(rec), flush=True)
        cs.destroy(); cd.destroy()
    ctx.close()


if __name__ == "__main__":
    main()
