#!/usr/bin/env python
"""Throughput of b200reg_knn across k: every point of a 100k cloud as a query (self-queries), on a raw KITTI-shaped scan
and on a 0.3 m-voxelised map, at k = 32 (the one-thread-per-query kernels) and 33, 64, 128, 256, 1024 (knn_large.cu).

Per case: the device time of the search kernels alone (CUDA activity from torch.profiler, summed over the call's kernels),
the median wall time of the whole call (queries host -> device, search, results device -> host into pageable numpy arrays)
over --reps calls after --warmup calls, queries/s for both, and, as a baseline on the same inputs, the reference's own
kd-tree (oracle/_ref, nanoflann built from the reference sources) on all host threads.  Prints one JSON line per case,
with the card's name and power limit.
    python profiles/knn_large_k.py [--reps 5] [--warmup 2] [--no-ref]
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

KS = (32, 33, 64, 128, 256, 1024)


def clouds():
    raw = np.ascontiguousarray(synth.make_pair(31, 100000)[1][:, :3])
    poses = [synth.se3(t=(15.0 * k, 0.0, 1.73)) for k in range(10)]
    scans = np.concatenate([synth.to_map_frame(synth.scan(31, 100 + k, P, 100000), P) for k, P in enumerate(poses)])
    vox = synth.voxelize(scans, 0.3)[:, :3]
    return {"raw_100k": raw, "voxel_0.3_100k": np.ascontiguousarray(vox[:100000])}


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def kernel_ms(fn, calls=3):
    """Device time of the search kernels per call: CUDA kernel activity recorded by torch.profiler over `calls` calls."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    total, names = 0.0, set()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and ("knn" in e.name or "k_rs_" in e.name):
            total += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            names.add(e.name.split("(")[0])
    return (total / 1e3 / calls, sorted(names)) if names else (None, [])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-ref", action="store_true", help="skip the reference kd-tree baseline")
    a = ap.parse_args()
    import torch
    device = torch.cuda.get_device_name(0)
    try:  # the card's power limit is part of every number below
        device += ", " + subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                                 text=True).strip() + " limit"
    except (OSError, subprocess.CalledProcessError):
        pass
    ref = None
    if not a.no_ref:
        from oracle import oracle as orc
        if os.path.exists(orc.ref_so_path()):
            ref = orc
    ctx = b200reg.Context(0)
    for name, cloud in clouds().items():
        cl, = ctx.create_clouds([cloud])
        tree = ref.RefNanoflann(cloud) if ref else None
        for k in KS:
            call = lambda: ctx.knn(cl, cloud, k)  # noqa: E731
            call()
            kms, kernels = kernel_ms(call)
            med, lo, hi = timed(call, a.reps, a.warmup)
            rec = dict(cloud=name, n=len(cloud), queries=len(cloud), k=k, kernels=kernels, kernel_ms=kms,
                       kernel_queries_per_s=len(cloud) / (kms / 1e3) if kms else None,
                       call_ms_median=med * 1e3, call_ms_min=lo * 1e3, call_ms_max=hi * 1e3, call_queries_per_s=len(cloud) / med,
                       node_visits_per_query="not measured", points_tested_per_query="not measured",
                       merge_rounds_per_query="not measured", reps=a.reps, warmup=a.warmup, device=device)
            if tree is not None:
                tree.knn(cloud[:1000], k)
                rmed, _, _ = timed(lambda: tree.knn(cloud, k), max(1, a.reps // 2), 0)
                rec.update(ref_ms_median=rmed * 1e3, ref_queries_per_s=len(cloud) / rmed, ref_threads=ref.num_threads(),
                           ref_host_cpus=os.cpu_count())
            print(json.dumps(rec), flush=True)
        cl.destroy()
    ctx.close()


if __name__ == "__main__":
    main()
