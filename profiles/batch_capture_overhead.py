#!/usr/bin/env python
"""Cost of capturing the loop clouds (all four kinds) and the LM trace on batch-driver jobs (b200reg_batch_set_loop_clouds /
b200reg_batch_set_lm_trace) over the device keyframe store.
    python profiles/batch_capture_overhead.py [reps] [keyframes] [depth]
Workload: loop_clouds_overhead.py's -- a synthetic KITTI-05-shaped sequence of 30k-point keyframes held on the device,
batches of 16 queries that have a loop candidate, Quatro + Nano-GICP with the deployment's configuration -- as
b200reg_batch_submit_perform_loop_closure jobs (closest_idx NULL: the job runs the candidate search) on a driver of
`depth` contexts.  One pass submits every batch, then waits for each job in submit order; with capture on it also reads
every kind and the trace of each job by ticket (the host copies a node makes to publish them) and releases it.  Host clock
over the pass.  Capture off and on alternate over the same jobs, `reps` passes each, after one untimed pass of each.
Prints one JSON line: attempts/s and ms per job (pass time / jobs) per setting, median and range over the passes, each
job's submit-to-completion latency (median), the points and trials captured per job, and the card's name and power
limit."""
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
depth = int(sys.argv[3]) if len(sys.argv) > 3 else 3
B = 16
KINDS = (b200reg.CLOUD_SOURCE, b200reg.CLOUD_TARGET, b200reg.CLOUD_COARSE, b200reg.CLOUD_FINAL)
seq = synth.make_sequence(5, nkf, pts_per_keyframe=30000, threads=max(1, (os.cpu_count() or 8) // 8))
ctx = b200reg.Context(0)
kf = ctx.keyframes()
kf.reserve(sum(len(c) for c in seq["clouds"]))
for c, T, t in zip(seq["clouds"], seq["poses"], seq["stamps"]):
    kf.add(c, T, t)
ctx.synchronize()
cfg = b200reg.default_loop_config()
allq = np.arange(nkf, dtype=np.int32)
cand = allq[kf.fetch_closest(allq, cfg.loop_detection_radius, cfg.loop_detection_timediff_threshold) >= 0]
batches = [cand[i:i + B] for i in range(0, len(cand) - B + 1, B)]
assert batches, "sequence too short for loop candidates"
driver = b200reg.Batch(0, depth=depth)


def run(capture):
    driver.set_loop_clouds(15 if capture else 0)
    driver.set_lm_trace(capture)
    t0 = time.perf_counter()
    tickets = [driver.submit_perform_loop_closure(kf, q, None, cfg) for q in batches]
    out, lat, points, trials = [], [], [], []
    for t in tickets:
        (res, qi), ms = driver.wait(t, want_latency=True, want_quatro=True)
        out.append(bytes(res) + bytes(qi))
        lat.append(ms)
        if capture:
            points.append(sum(sum(len(r) for r in driver.loop_clouds(t, k)) for k in KINDS))
            trials.append(sum(len(r) for r in driver.lm_trace(t)))
            driver.release(t)
    return time.perf_counter() - t0, out, lat, points, trials


run(False), run(True)  # warm-up: arenas, graphs, pools, every batch's shapes on every context
passes = {False: [], True: []}
lat = {False: [], True: []}
points, trials = [], []
for _ in range(reps):
    s_off, out_off, l_off, _, _ = run(False)
    s_on, out_on, l_on, p, tr = run(True)
    assert out_on == out_off, "capture changed a result"
    passes[False].append(s_off)
    passes[True].append(s_on)
    lat[False] += l_off
    lat[True] += l_on
    points += p
    trials += tr

try:  # the card's power limit is part of every number below
    device = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                     text=True).strip()
except (OSError, subprocess.CalledProcessError):
    device = "unknown"
attempts = len(batches) * B


def arm(on):
    s = np.array(passes[on])
    return dict(attempts_per_s=dict(median=round(float(attempts / np.median(s)), 1), min=round(float(attempts / s.max()), 1),
                                    max=round(float(attempts / s.min()), 1)),
                ms_per_job=dict(median=round(float(np.median(s) * 1e3 / len(batches)), 3),
                                min=round(float(s.min() * 1e3 / len(batches)), 3), max=round(float(s.max() * 1e3 / len(batches)), 3)),
                latency_ms_median=round(float(np.median(lat[on])), 3))


print(json.dumps(dict(workload="batch driver depth %d, %d jobs of %d candidate queries, %d keyframes x 30k points" % (depth, len(batches), B, nkf),
                      reps=reps, device=device, capture_off=arm(False), capture_on=arm(True),
                      points_captured_per_job=dict(median=int(np.median(points)), max=int(max(points))),
                      lm_trials_per_job=dict(median=int(np.median(trials)), max=int(max(trials))))))
driver.close()
kf.destroy()
ctx.close()
