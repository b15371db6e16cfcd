#!/usr/bin/env python
"""Per-pair LM scheduling, measured: a 16-pair icpAlignment batch in which ONE pair runs all 32 outer iterations (synthetic
seed 1104: GICP itself diverges on it, identically on the CPU oracle) against the same batch with a clean pair in its place.
Round 1 kept launching the blocks of the 15 finished pairs until the last pair was done.
    python profiles/straggler.py > out/straggler.txt"""
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))
import torch  # noqa: E402
import b200reg  # noqa: E402
from b200reg import synth  # noqa: E402

clean = [synth.make_pair(1000 + i, 100000, 100000) for i in range(16)]
bad = synth.make_pair(1104, 100000, 100000)
ctx = b200reg.Context(0)


def run(pairs, reps=8):
    ds = [torch.from_numpy(p[0]).cuda() for p in pairs]
    dd = [torch.from_numpy(p[1]).cuda() for p in pairs]
    args = ([t.data_ptr() for t in ds], [t.shape[0] for t in ds], [t.data_ptr() for t in dd], [t.shape[0] for t in dd], 16, 1)
    res = ctx.icp_alignment_ptrs(*args)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        res = ctx.icp_alignment_ptrs(*args)
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), [r.n_linearize for r in res], [bool(r.converged) for r in res]


t_clean, nl, _ = run(clean)
t_bad, nl2, cv2 = run(clean[:15] + [bad])
print("clean 16-pair batch: %.2f ms (linearize passes %s)" % (t_clean, nl))
print("15 clean pairs + seed 1104: %.2f ms (linearize passes %s, converged %s)" % (t_bad, nl2, cv2))
print("latency ratio %.2f (the straggler's own chain of 32 x (linearize + trial) steps on 100k points is serial: ~50 us per step)" % (t_bad / t_clean))
ctx.close()

# throughput: the same two job types streamed through the batch driver (3 contexts, 6 jobs in flight): while one context
# spins through its straggler's steps (782 work items of a 4736-block grid), the other contexts' jobs fill the machine
batch = b200reg.Batch(0, depth=3)


def stream(pairs, jobs=24):
    ds = [torch.from_numpy(p[0]).cuda() for p in pairs]
    dd = [torch.from_numpy(p[1]).cuda() for p in pairs]
    args = ([t.data_ptr() for t in ds], [t.shape[0] for t in ds], [t.data_ptr() for t in dd], [t.shape[0] for t in dd], 16, 1)
    for _ in range(2):
        [batch.wait(t) for t in [batch.submit_icp(*args) for _ in range(6)]]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    inflight = []
    for j in range(jobs):
        inflight.append(batch.submit_icp(*args))
        if len(inflight) >= 6:
            batch.wait(inflight.pop(0))
    for t in inflight:
        batch.wait(t)
    return 16 * jobs / (time.perf_counter() - t0)


p_clean = stream(clean)
p_bad = stream(clean[:15] + [bad])
print("streamed through b200reg_batch: clean jobs %.0f pairs/s, jobs with one 32-iteration pair each %.0f pairs/s: cost ratio %.2f"
      % (p_clean, p_bad, p_clean / p_bad))
batch.close()
