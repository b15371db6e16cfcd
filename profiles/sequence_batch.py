#!/usr/bin/env python
"""Loop attempts over the device keyframe store: the synchronous call against the batch driver.
    python profiles/sequence_batch.py [keyframes] [reps]
Workload: bench.py's sequence arm (configs[4]) -- a synthetic KITTI-05-shaped sequence of 30k-point keyframes held on the
device, every keyframe that has a loop candidate, 16 per call, Quatro + Nano-GICP with the deployment's configuration.  It
runs three ways over the same batches:
  sync      per batch b200reg_fetch_closest_keyframes + b200reg_perform_loop_closure on one context (bench.py's step);
  depth 3   every batch submitted as one b200reg_batch_submit_perform_loop_closure job (closest_idx NULL: the job runs
  depth 6   the candidate search itself) to a driver of 3 / 6 contexts, then every job waited for.
Each timed region is host clock from the first call to the last result on the host, after one untimed warm-up pass of
every batch per arm; `reps` timed passes per arm, alternating arms.  The three arms must return identical bytes.  Prints
one JSON line: attempts/s per arm (median and range over the passes), the speedups, and the card's name and power limit."""
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

nkf = int(sys.argv[1]) if len(sys.argv) > 1 else 2761  # KITTI 05, bench.py's default
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
B = 16
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
batches = [cand[i:i + B] for i in range(0, len(cand) - B + 1, B)]  # bench.py's batches
assert batches, "sequence too short for loop candidates"
drivers = {3: b200reg.Batch(0, depth=3), 6: b200reg.Batch(0, depth=6)}


def run_sync():
    out = []
    for q in batches:
        cl = kf.fetch_closest(q, cfg.loop_detection_radius, cfg.loop_detection_timediff_threshold)
        res, qi = kf.perform_loop_closure(q, cl, cfg, raw=True)
        out.append(bytes(res) + bytes(qi))
    return out


def run_driver(depth):
    d = drivers[depth]
    tickets = [d.submit_perform_loop_closure(kf, q, None, cfg) for q in batches]
    out = []
    for t in tickets:
        res, qi = d.wait(t, want_quatro=True)
        out.append(bytes(res) + bytes(qi))
    return out


arms = {"sync": run_sync, "depth3": lambda: run_driver(3), "depth6": lambda: run_driver(6)}
ref = {name: fn() for name, fn in arms.items()}  # warm-up: arenas, graphs, pools, every batch's shapes
identical = ref["depth3"] == ref["sync"] and ref["depth6"] == ref["sync"]
secs = {name: [] for name in arms}
for _ in range(reps):
    for name, fn in arms.items():
        t0 = time.perf_counter()
        got = fn()
        secs[name].append(time.perf_counter() - t0)
        identical &= got == ref["sync"]
attempts = B * len(batches)
rate = {name: dict(median=round(attempts / float(np.median(s)), 1), min=round(attempts / max(s), 1), max=round(attempts / min(s), 1))
        for name, s in secs.items()}
try:  # the card's power limit is part of every number below
    device = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                     text=True).strip()
except (OSError, subprocess.CalledProcessError):
    device = "unknown"
print(json.dumps(dict(workload="loop attempts over the device keyframe store: %d batches of %d candidate queries, %d keyframes x 30k points"
                               % (len(batches), B, nkf), reps=reps, device=device, identical_bytes=bool(identical),
                      attempts_per_s=rate,
                      speedup_depth3=round(rate["depth3"]["median"] / rate["sync"]["median"], 3),
                      speedup_depth6=round(rate["depth6"]["median"] / rate["sync"]["median"], 3))))
for d in drivers.values():
    d.close()
kf.destroy()
ctx.close()
sys.exit(0 if identical else 1)
