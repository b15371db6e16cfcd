#!/usr/bin/env python
"""Cost of recording the fitness pass's residuals (b200reg_ctx_set_residuals) on icp_alignment jobs and on
b200reg_perform_loop_closure batches.
    python profiles/residuals_overhead.py [reps] [keyframes]
Workloads: (1) b200reg_icp_alignment over 16 pairs of 100k points (four distinct synthetic pairs, each four times), host
buffers; (2) bench.py's sequence arm at a shorter length -- a synthetic KITTI-05-shaped sequence of 30k-point keyframes
held on the device, batches of 16 queries that have a loop candidate, Quatro + Nano-GICP with the deployment's
configuration.  Each timed call is one call (host clock around it; it ends in a stream synchronise, and the recording
call also copies its rows to the host and the binding reads them out).  Recording off and on alternate over the same
inputs, `reps` rounds.  Prints one JSON line: medians and ranges in ms per call, the rows recorded per call, and the card's
name and power limit."""
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

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
nkf = int(sys.argv[2]) if len(sys.argv) > 2 else 700  # one lap is 514 keyframes: the last ~190 close loops
B = 16
ctx = b200reg.Context(0)


def timed(call, record):
    ctx.set_residuals(record)
    t0 = time.perf_counter()
    out = call()
    rows = sum(len(nn) for nn, _ in ctx.residuals()) if record else 0
    ms = (time.perf_counter() - t0) * 1e3
    ctx.set_residuals(False)
    return ms, out, rows


def measure(calls):
    """calls: list of () -> bytes.  Warm-up, then off / on alternating -> (times off, times on, rows per call)."""
    for c in calls:
        timed(c, False), timed(c, True)
    times = {False: [], True: []}
    rows = []
    for _ in range(reps):
        for c in calls:
            ms_off, out_off, _ = timed(c, False)
            ms_on, out_on, r = timed(c, True)
            assert out_on == out_off, "recording changed a result"
            times[False].append(ms_off)
            times[True].append(ms_on)
            rows.append(r)
    return times, rows


pairs = [synth.make_pair(3000 + k, 100000, 100000) for k in range(4)]
srcs = [pairs[k % 4][0] for k in range(B)]
dsts = [pairs[k % 4][1] for k in range(B)]
icp_times, icp_rows = measure([lambda: bytes(ctx.icp_alignment(srcs, dsts, raw=True))])

seq = synth.make_sequence(5, nkf, pts_per_keyframe=30000, threads=max(1, (os.cpu_count() or 8) // 8))
kf = ctx.keyframes()
kf.reserve(sum(len(c) for c in seq["clouds"]))
for c, T, t in zip(seq["clouds"], seq["poses"], seq["stamps"]):
    kf.add(c, T, t)
cfg = b200reg.default_loop_config()
allq = np.arange(nkf, dtype=np.int32)
closest = kf.fetch_closest(allq, cfg.loop_detection_radius, cfg.loop_detection_timediff_threshold)
cand = allq[closest >= 0]
batches = [(cand[i:i + B], closest[cand[i:i + B]]) for i in range(0, len(cand) - B + 1, B)]
assert batches, "sequence too short for loop candidates"


def attempt(q, cl):
    res, qi = kf.perform_loop_closure(q, cl, cfg, raw=True)
    return bytes(res) + bytes(qi)


lc_times, lc_rows = measure([lambda q=q, cl=cl: attempt(q, cl) for q, cl in batches])

try:  # the card's power limit is part of every number below
    device = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                                      "-i", "0"], text=True).strip()
except (OSError, subprocess.CalledProcessError):
    device = "unknown"
summary = lambda v: dict(median=round(float(np.median(v)), 3), min=round(min(v), 3), max=round(max(v), 3))


def report(times, rows):
    return dict(ms_off=summary(times[False]), ms_on=summary(times[True]),
                median_overhead_ms=round(float(np.median(np.array(times[True]) - np.array(times[False]))), 3),
                rows_per_call=dict(median=int(np.median(rows)), max=int(max(rows))))


print(json.dumps(dict(reps=reps, device=device,
                      icp_alignment=dict(workload="icp_alignment, %d pairs x 100k points, host buffers" % B, **report(icp_times, icp_rows)),
                      perform_loop_closure=dict(workload="perform_loop_closure, %d batches of %d candidate queries, %d keyframes x 30k points"
                                                % (len(batches), B, nkf), **report(lc_times, lc_rows)))))
kf.destroy()
ctx.close()
