#!/usr/bin/env python
"""Cost of the LM trace (b200reg_ctx_set_lm_trace) on one 16-pair 100k x 100k job, profiles/one_job.py's unit.
    python profiles/lm_trace_overhead.py [reps]
The clouds and covariances are built once; each timed call is one b200reg_gicp_align over the 16 pairs (the LM loop as one
graph launch, host clock around the call, which ends in a stream synchronise).  Trace off and on alternate, `reps` each.
Then one host-polled pass of each (profiling mode) gives gicp_control's own CUDA-event time, the kernel that writes the
records.  Prints one JSON line: medians and ranges in ms, records written, and the card's name and power limit."""
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

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
pairs = [synth.make_pair(1000 + i, 100000, 100000) for i in range(16)]
ctx = b200reg.Context(0)
clouds = ctx.create_clouds([p[0] for p in pairs] + [p[1] for p in pairs])
src, tgt = clouds[:16], clouds[16:]
ctx.covariances(clouds, 15)


def solve(trace):
    ctx.set_lm_trace(trace)
    t0 = time.perf_counter()
    res = ctx.gicp_align(src, tgt)
    ms = (time.perf_counter() - t0) * 1e3
    records = sum(len(t) for t in ctx.lm_trace()) if trace else 0
    ctx.set_lm_trace(False)
    return ms, res, records


solve(False), solve(True)  # warm-up: arena, graph, pool
times = {False: [], True: []}
ref = None
records = 0
for _ in range(reps):
    for trace in (False, True):
        ms, res, rec = solve(trace)
        times[trace].append(ms)
        key = [(r["T"].tobytes(), r["fitness"], r["n_error"]) for r in res]
        assert ref is None or key == ref, "tracing changed a result"
        ref = key
        records = max(records, rec)

control = {}
ctx.set_profiling(True)
for trace in (False, True):
    ctx.reset_profile()
    solve(trace)
    control[trace] = ctx.get_profile()["gicp_control"]["ms"]
ctx.set_profiling(False)

try:  # the card's power limit is part of every number below
    device = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                     text=True).strip()
except (OSError, subprocess.CalledProcessError):
    device = "unknown"
summary = lambda v: dict(median=round(float(np.median(v)), 3), min=round(min(v), 3), max=round(max(v), 3))
print(json.dumps(dict(workload="16 pairs 100k x 100k, gicp_align on built clouds", reps=reps, device=device,
                      lm_call_ms_trace_off=summary(times[False]), lm_call_ms_trace_on=summary(times[True]),
                      records_written=records, record_bytes=200,
                      gicp_control_ms_host_polled=dict(off=round(control[False], 3), on=round(control[True], 3)))))
for c in clouds:
    c.destroy()
ctx.close()
