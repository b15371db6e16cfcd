#!/usr/bin/env python
"""Cost of b200reg_clouds_covariances_ex across k, next to the k-NN it contains: every point of a 100k cloud, on a raw
KITTI-shaped scan and on a 0.3 m-voxelised map, at k = 32 (k_covariance<32>, one thread per point) and 33, 48, 64, 128,
256, 257, 512 (k_covariance_large, one warp per point; 257 and 512 keep their lists in the scratch slab).

Per case: the device time of the covariance kernel alone and of the k-NN kernels of b200reg_knn with every point as a query
at the same k (CUDA activity from torch.profiler, per call), and the median wall time of the covariance call (method PLANE,
recomputed each call) over --reps calls after --warmup calls.  The difference between the two kernel times is what the
moments and the regularisation cost on top of the walk (the k-NN kernel also writes k results per query, which the
covariance kernel does not).  Prints one JSON line per case, with the card's name and power limit.
    python profiles/covariance_large_k.py [--reps 10] [--warmup 3]
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

import b200reg  # noqa: E402
from b200reg import synth  # noqa: E402

KS = (32, 33, 48, 64, 128, 256, 257, 512)


def clouds():
    raw = np.ascontiguousarray(synth.make_pair(31, 100000)[1][:, :3])
    poses = [synth.se3(t=(15.0 * k, 0.0, 1.73)) for k in range(10)]
    scans = np.concatenate([synth.to_map_frame(synth.scan(31, 100 + k, P, 100000), P) for k, P in enumerate(poses)])
    vox = synth.voxelize(scans, 0.3)[:, :3]
    return {"raw_100k": raw, "voxel_0.3_100k": np.ascontiguousarray(vox[:100000])}


def kernel_ms(fn, match, calls=3):
    """Device time per call of the CUDA kernels whose name contains one of `match`, recorded by torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    total, names = 0.0, set()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and any(m in e.name for m in match):
            total += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            names.add(e.name.split("(")[0])
    return (total / 1e3 / calls, sorted(names)) if names else (None, [])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    device = torch.cuda.get_device_name(0)
    try:  # the card's power limit is part of every number below
        device += ", " + subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                                 text=True).strip() + " limit"
    except (OSError, subprocess.CalledProcessError):
        pass
    ctx = b200reg.Context(0)
    for name, cloud in clouds().items():
        cl, = ctx.create_clouds([cloud])
        for k in KS:
            flip = [0]

            def cov():  # alternate NONE / PLANE so that the per-cloud cache never skips the pass
                flip[0] ^= 1
                ctx.covariances([cl], k, 3 if flip[0] else 0)
                torch.cuda.synchronize()
            knn = lambda: ctx.knn(cl, cloud, k)  # noqa: E731
            cov()
            knn()
            cms, cnames = kernel_ms(cov, ("k_covariance",))
            kms, knames = kernel_ms(knn, ("knn",))
            for _ in range(a.warmup):
                cov()
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                cov()
                ts.append(time.perf_counter() - t0)
            rec = dict(cloud=name, n=len(cloud), k=k, cov_kernels=cnames, cov_kernel_ms=cms, knn_kernels=knames, knn_kernel_ms=kms,
                       moments_over_knn_ms=(cms - kms) if cms is not None and kms is not None else None,
                       cov_call_ms_median=float(np.median(ts)) * 1e3, cov_call_ms_min=float(min(ts)) * 1e3,
                       cov_call_ms_max=float(max(ts)) * 1e3, reps=a.reps, warmup=a.warmup, device=device)
            print(json.dumps(rec), flush=True)
        cl.destroy()
    ctx.close()


if __name__ == "__main__":
    main()
