#!/usr/bin/env python
"""Time of the TEASER++ solve that follows advancedMatching, for correspondence sets beyond B200REG_ADV_CORR_CAPACITY.

Solve stage: b200reg_quatro_solve_tap on synthetic sets of n = 8192, 16384, 32768 and 65536 correspondences (300 of
them inliers of a known motion, the rest random pairs; tests/test_gpu_quatro_big.py's generator), on the path of large
sets (wide) and, at n = 8192, also on the batched path.  Per size: the device time of the call's kernels (CUDA activity
from torch.profiler), the median wall time of the whole call over --reps calls after one warm-up, and the clique size.
End to end: b200reg_quatro_align with advancedMatching on the 0.2 m sub-map pair of the tests (about 9000 surviving
correspondences), wall time per call, and the same split for the solve alone through the tap.
--oracle adds the CPU oracle's time for the same solves (single-threaded; skipped above --oracle-max).
Prints one JSON line per case, with the card's name and power limit.
    python profiles/quatro_big_solve.py [--reps 5] [--oracle] [--oracle-max 32768]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))

import b200reg  # noqa: E402
from b200reg import native  # noqa: E402
from test_gpu_quatro_big import make_submap_pair, synthetic_set  # noqa: E402


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts)), 1e3 * float(min(ts)), 1e3 * float(max(ts))


def kernel_ms(fn):
    """Device time of the kernels of one call, per kernel name."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fn()
    out = {}
    for e in p.key_averages():
        if e.device_type.name == "CUDA" and e.key.startswith("_ZN4b200") or e.key.startswith("b200::"):
            name = e.key.split("b200")[1].lstrip(":0123456789").split("E")[0].split("(")[0]
            out[name] = out.get(name, 0.0) + e.device_time_total / 1e3
    return out


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--oracle-max", type=int, default=32768)
    a = ap.parse_args()
    gpu = gpu_info()
    ctx = b200reg.Context(0)
    prm = native.default_quatro_params()
    prm.use_optimized_matching = 0
    if a.oracle:
        from oracle import oracle as orc
    for n in (8192, 16384, 32768, 65536):
        S, D, _ = synthetic_set(n, seed=n)
        for wide in ([False, True] if n <= 8192 else [True]):
            res = {}
            fn = lambda: res.update(ctx.quatro_solve_tap(S, D, prm, wide=wide))  # noqa: E731
            med, lo, hi = timed(fn, a.reps)
            km = kernel_ms(fn)
            rec = dict(case="solve_tap", n=n, path="wide" if wide else "batched", wall_ms_median=med, wall_ms_min=lo, wall_ms_max=hi,
                       kernel_ms=sum(km.values()), kernels=km, clique=res["clique_size"], gpu=gpu)
            if a.oracle and wide and n <= a.oracle_max:
                t0 = time.perf_counter()
                orc.quatro_solve(S, D, np.repeat(np.arange(n, dtype=np.int32)[:, None], 2, 1), _orc_params(orc))
                rec["oracle_cpu_ms"] = 1e3 * (time.perf_counter() - t0)
            print(json.dumps(rec), flush=True)
    src, dst, _ = make_submap_pair()
    cs, cd = ctx.create_clouds([src, dst])
    info = {}
    fn = lambda: info.update(ctx.quatro_align([cs], [cd], params=prm, want_corr=True)[0])  # noqa: E731
    med, lo, hi = timed(fn, a.reps)
    km = kernel_ms(fn)
    corr = info["corr"]
    solve = {}
    sfn = lambda: solve.update(ctx.quatro_solve_tap(src[corr[:, 0]], dst[corr[:, 1]], prm, wide=True))  # noqa: E731
    smed, _, _ = timed(sfn, a.reps)
    skm = kernel_ms(sfn)
    rec = dict(case="submap_0.2_end_to_end", n_src=len(src), n_dst=len(dst), n_corr=info["n_corr"], clique=info["clique_size"],
               wall_ms_median=med, wall_ms_min=lo, wall_ms_max=hi, kernel_ms=sum(km.values()), kernels=km,
               solve_wall_ms_median=smed, solve_kernel_ms=sum(skm.values()), gpu=gpu)
    if a.oracle:
        t0 = time.perf_counter()
        orc.quatro_solve(src, dst, corr, _orc_params(orc))
        rec["oracle_cpu_solve_ms"] = 1e3 * (time.perf_counter() - t0)
    print(json.dumps(rec), flush=True)
    cs.destroy(); cd.destroy()
    ctx.close()


def _orc_params(orc):
    return orc.QuatroParams.default()


if __name__ == "__main__":
    main()
