#!/usr/bin/env python
"""Where the time of the spatial index build goes: the 32 clouds of one 16-pair headline job (bench.py's primary_seeds()
1000..1015, 100k x 100k points, raw xyz records resident on the device) built in one b200reg_clouds_create call.

Prints, with the card's name and power limit:
  - the whole-call time from CUDA events, median and range over --calls calls after warm-up (clouds destroyed outside
    the timed region);
  - from torch.profiler CUDA activity, in a process of its own: device time per launch of every build kernel, averaged
    over --prof-calls calls, the gap between consecutive launches, and first start to last end;
  - the algorithmic bytes of each kernel, computed from the shapes, and the rate they imply.

Bytes per kernel (N points over all clouds, S = record stride in bytes, R = tree records written, i.e. internal nodes
that span more than LEAF points, counted on the built trees):
  k_bbox            S*N                      records read once
  k_morton_ghist    S*N + 8N                 records read, keys + indices written
  k_sort_pass       16N                      keys + values read and written
  k_sort_pass last  (32 + S)*N               keys + values read, keys written, records gathered, points + ranks written
  k_lbvh_topology   28N                      sorted keys read, (first, last, bits, split) + parents written
  k_lbvh_aabb       56N + 16N + 120R         work-item classification, leaf points, per record: 64 B written, the
                                             sibling's 32 B read back, the node's split, parent and flag
    python profiles/index_build_kernels.py [--pkg DIR] [--calls 50] [--prof-calls 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = range(1000, 1016)
POINTS = 100000
LEAF = 8
KERNELS = ["k_bbox", "k_morton_ghist", "k_sort_pass", "k_lbvh_topology", "k_lbvh_aabb"]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def job_records():
    from b200reg import synth
    import torch
    recs = []
    for s in SEEDS:
        src, dst, _ = synth.make_pair(s, POINTS, POINTS)
        recs += [torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()]
    torch.cuda.synchronize()
    return recs


def records_written(tnodes, root_ref):
    """Internal nodes reachable from the root: the records k_lbvh_aabb writes (unreached slots are never touched)."""
    if root_ref < 0:
        return 0
    refs = tnodes[:, [0, 2], 3].copy().view(np.int32)
    front, count = np.array([root_ref]), 0
    while len(front):
        count += len(front)
        ch = refs[front].ravel()
        front = ch[ch >= 0]
    return count


def kernel_bytes(n_total, stride, records):
    return {"k_bbox": stride * n_total, "k_morton_ghist": (stride + 8) * n_total, "k_sort_pass#0": 16 * n_total,
            "k_sort_pass#1": 16 * n_total, "k_sort_pass#2": (32 + stride) * n_total, "k_lbvh_topology": 28 * n_total,
            "k_lbvh_aabb": 72 * n_total + 120 * records}


def run_events(args):
    import torch
    import b200reg
    recs = job_records()
    ptrs, ns, stride = [r.data_ptr() for r in recs], [int(r.shape[0]) for r in recs], int(recs[0].shape[1]) * 4
    ctx = b200reg.Context(0)
    taps = ctx.index_tap(recs, device=True)
    records = sum(records_written(t["tnodes"], t["root_ref"]) for t in taps)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    for _ in range(5):
        for c in ctx.create_clouds_device(ptrs, ns, stride):
            c.destroy()
    l0 = ctx.launch_count
    for c in ctx.create_clouds_device(ptrs, ns, stride):
        c.destroy()
    launches = ctx.launch_count - l0
    ms = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.calls):
        stream.synchronize()
        e0.record(stream)
        cl = ctx.create_clouds_device(ptrs, ns, stride)
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
        for c in cl:
            c.destroy()
    ctx.close()
    return {"points": sum(ns), "clouds": len(ns), "stride": stride, "records_written": records, "launches": launches,
            "call_ms_median": statistics.median(ms), "call_ms_min": min(ms), "call_ms_max": max(ms)}


def run_profile(args):
    import torch
    from torch.profiler import ProfilerActivity, profile
    import b200reg
    recs = job_records()
    ptrs, ns, stride = [r.data_ptr() for r in recs], [int(r.shape[0]) for r in recs], int(recs[0].shape[1]) * 4
    ctx = b200reg.Context(0)
    for _ in range(5):
        for c in ctx.create_clouds_device(ptrs, ns, stride):
            c.destroy()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.prof_calls):
            for c in ctx.create_clouds_device(ptrs, ns, stride):
                c.destroy()
        torch.cuda.synchronize()
    ctx.close()
    evs = []
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        k = next((k for k in KERNELS if k in e.name), None)
        if k:
            evs.append((e.time_range.start, e.time_range.end, k))
    evs.sort()
    per_call = len(evs) // args.prof_calls
    assert per_call * args.prof_calls == len(evs), ("uneven launches per call", len(evs), args.prof_calls)
    names, dur, gap, span = [], {}, {}, []
    for c in range(args.prof_calls):
        call = evs[c * per_call:(c + 1) * per_call]
        seen = {}
        for j, (s, e, k) in enumerate(call):
            idx = seen.get(k, 0)
            seen[k] = idx + 1
            key = k if k != "k_sort_pass" else "%s#%d" % (k, idx)
            if c == 0:
                names.append(key)
            dur.setdefault(key, []).append((e - s) / 1000.0)
            if j:
                gap.setdefault(key, []).append((s - call[j - 1][1]) / 1000.0)
        span.append((call[-1][1] - call[0][0]) / 1000.0)
    return {"order": names, "kernel_ms": {k: statistics.mean(v) for k, v in dur.items()},
            "gap_ms_before": {k: statistics.mean(v) for k, v in gap.items()}, "span_ms": statistics.mean(span)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pkg", default=os.path.join(REPO, "fast-lio-sam-qn_b200"))
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--prof-calls", type=int, default=10)
    ap.add_argument("--what", choices=["all", "events", "profile"], default="all")
    ap.add_argument("--json", help="also write the results here")
    args = ap.parse_args()
    sys.path[:0] = [os.path.abspath(args.pkg)]
    if args.what != "all":
        print(json.dumps(run_events(args) if args.what == "events" else run_profile(args)))
        return
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    base = [sys.executable, os.path.abspath(__file__), "--pkg", args.pkg, "--calls", str(args.calls),
            "--prof-calls", str(args.prof_calls), "--what"]
    ev = json.loads(subprocess.run(base + ["events"], check=True, capture_output=True, text=True).stdout.splitlines()[-1])
    pr = json.loads(subprocess.run(base + ["profile"], check=True, capture_output=True, text=True).stdout.splitlines()[-1])
    name, power = card()
    byts = kernel_bytes(ev["points"], ev["stride"], ev["records_written"])
    print("%s, power limit %s; package %s" % (name, power, os.path.abspath(args.pkg)))
    print("%d clouds, %d points, record stride %d B, %d tree records written, %d launches per call"
          % (ev["clouds"], ev["points"], ev["stride"], ev["records_written"], ev["launches"]))
    print("| kernel | device ms | gap before, ms | MB (algorithmic) | GB/s |")
    print("|---|---|---|---|---|")
    tot = 0.0
    for k in pr["order"]:
        t = pr["kernel_ms"][k]
        tot += t
        b = byts.get(k)
        print("| %s | %.4f | %s | %s | %s |" % (k, t, "%.4f" % pr["gap_ms_before"][k] if k in pr["gap_ms_before"] else "-",
                                              "%.1f" % (b / 1e6) if b else "-", "%.0f" % (b / t / 1e6) if b else "-"))
    print("kernels %.4f ms, first start to last end %.4f ms; whole call (CUDA events, %d calls) median %.4f ms (%.4f-%.4f)"
          % (tot, pr["span_ms"], args.calls, ev["call_ms_median"], ev["call_ms_min"], ev["call_ms_max"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit": power, "events": ev, "profile": pr, "bytes": byts}, f, indent=1)


if __name__ == "__main__":
    main()
