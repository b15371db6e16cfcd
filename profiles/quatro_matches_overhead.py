#!/usr/bin/env python
"""Cost of recording the Quatro matches (b200reg_ctx_set_quatro_matches) on b200reg_perform_loop_closure batches.
    python profiles/quatro_matches_overhead.py [reps] [keyframes]
Workload: the one of profiles/loop_clouds_overhead.py -- a synthetic KITTI-05-shaped sequence of 30k-point keyframes held on
the device, batches of 16 queries that have a loop candidate, Quatro + Nano-GICP with the deployment's configuration.  Each
timed call is one perform_loop_closure over one batch (host clock around the call, which ends in a stream synchronise; the
recording call also copies its matches to the host, and the getter's copy-out is timed with it).  Recording off and on
alternate over the same batches, `reps` rounds.  Prints one JSON line: medians and ranges in ms per batch, the matches
recorded per batch, and the card's name and power limit."""
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
seq = synth.make_sequence(5, nkf, pts_per_keyframe=30000, threads=max(1, (os.cpu_count() or 8) // 8))
ctx = b200reg.Context(0)
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


def run(b, record):
    ctx.set_quatro_matches(record)
    q, cl = batches[b]
    l0 = ctx.launch_count
    t0 = time.perf_counter()
    res, qi = kf.perform_loop_closure(q, cl, cfg, raw=True)
    rows = ctx.quatro_matches() if record else []
    ms = (time.perf_counter() - t0) * 1e3
    ctx.set_quatro_matches(False)
    return ms, bytes(res) + bytes(qi), sum(len(r["corr"]) for r in rows), ctx.launch_count - l0


for b in range(len(batches)):  # warm-up: arena, graph, pool, every batch's shapes
    run(b, False), run(b, True)
times = {False: [], True: []}
matches, extra = [], []
for _ in range(reps):
    for b in range(len(batches)):
        ms_off, out_off, _, l_off = run(b, False)
        ms_on, out_on, m, l_on = run(b, True)
        assert out_on == out_off, "recording changed a result"
        times[False].append(ms_off)
        times[True].append(ms_on)
        matches.append(m)
        extra.append(l_on - l_off)

try:  # the card's power limit is part of every number below
    device = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                     text=True).strip()
except (OSError, subprocess.CalledProcessError):
    device = "unknown"
summary = lambda v: dict(median=round(float(np.median(v)), 3), min=round(min(v), 3), max=round(max(v), 3))
print(json.dumps(dict(workload="perform_loop_closure, %d batches of %d candidate queries, %d keyframes x 30k points" % (len(batches), B, nkf),
                      reps=reps, device=device, batch_ms_recording_off=summary(times[False]), batch_ms_recording_on=summary(times[True]),
                      median_overhead_ms=round(float(np.median(np.array(times[True]) - np.array(times[False]))), 3),
                      matches_per_batch=dict(median=int(np.median(matches)), max=int(max(matches))),
                      extra_launches_per_batch=sorted(set(extra)))))
kf.destroy()
ctx.close()
