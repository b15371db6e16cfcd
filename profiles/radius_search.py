#!/usr/bin/env python
"""Throughput of b200reg_radius_search (KdTreeFLANN::radiusSearch, batched, CSR output): every point of a 100k cloud as a
query, sq_radius 0.81 and 2.25, on a raw KITTI-shaped scan and on a voxelised (0.3 m) map of ten scans.

Per case: median wall time of the whole call (host -> device queries, order, count, scan, fill, segmented sort,
device -> host results into pageable numpy arrays) over --reps calls after --warmup calls, the same for the count-only
mode (no neighbour output), queries/s, neighbours/s and kernel launches per call.  Prints one JSON line per case.
    python profiles/radius_search.py [--reps 7] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))

import b200reg  # noqa: E402
from b200reg import native, synth  # noqa: E402


def clouds():
    raw = np.ascontiguousarray(synth.make_pair(31, 100000)[1][:, :3])
    poses = [synth.se3(t=(15.0 * k, 0.0, 1.73)) for k in range(10)]
    scans = np.concatenate([synth.to_map_frame(synth.scan(31, 100 + k, P, 100000), P) for k, P in enumerate(poses)])
    return {"raw_100k": raw, "voxel_0.3": np.ascontiguousarray(synth.voxelize(scans, 0.3)[:, :3])}


def count_only(ctx, cl, q, r2):
    off = np.empty(len(q) + 1, np.int64)
    rc = native.lib().b200reg_radius_search(ctx.h, cl.h, q.ctypes.data_as(C.c_void_p), C.c_size_t(len(q)), C.c_size_t(12),
                                            C.c_double(r2), 1, off.ctypes.data_as(C.c_void_p), C.c_size_t(0), None, None)
    assert rc == 0
    return off


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import subprocess
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
        for r2 in (0.81, 2.25):
            for sorted_ in (True, False):
                l0 = ctx.launch_count
                off, _, _ = ctx.radius_search(cl, cloud, r2, sorted=sorted_)
                launches = ctx.launch_count - l0
                total = int(off[-1])
                med, lo, hi = timed(lambda: ctx.radius_search(cl, cloud, r2, sorted=sorted_), a.reps, a.warmup)
                cmed, clo, chi = timed(lambda: count_only(ctx, cl, cloud, r2), a.reps, a.warmup)
                l1 = ctx.launch_count
                count_only(ctx, cl, cloud, r2)
                print(json.dumps(dict(cloud=name, n=len(cloud), queries=len(cloud), sq_radius=r2, sorted=sorted_, neighbours=total,
                                      ms_median=med * 1e3, ms_min=lo * 1e3, ms_max=hi * 1e3,
                                      queries_per_s=len(cloud) / med, neighbours_per_s=total / med,
                                      count_only_ms_median=cmed * 1e3, count_only_queries_per_s=len(cloud) / cmed,
                                      launches_per_call=launches, count_only_launches=ctx.launch_count - l1,
                                      reps=a.reps, warmup=a.warmup, device=device)), flush=True)
        cl.destroy()
    ctx.close()


if __name__ == "__main__":
    main()
