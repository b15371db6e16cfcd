#!/usr/bin/env python
"""A few 16-pair icpAlignment jobs on ONE context (no pipelining): the unit the per-kernel profiles are taken on.
    python profiles/one_job.py [jobs] [pairs]          # prints the per-family CUDA-event times
    ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file out/launches.csv python profiles/one_job.py 3
"""
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))
import torch  # noqa: E402
import b200reg  # noqa: E402
from b200reg import synth  # noqa: E402

jobs = int(sys.argv[1]) if len(sys.argv) > 1 else 3
npairs = int(sys.argv[2]) if len(sys.argv) > 2 else 16
mode = sys.argv[3] if len(sys.argv) > 3 else "gicp"
pairs = [synth.make_pair((1000 if mode == "gicp" else 2000) + i, 100000, 100000, mode=mode, voxel=0.3 if mode == "quatro" else None)
         for i in range(npairs)]
ds = [torch.from_numpy(p[0]).cuda() for p in pairs]
dd = [torch.from_numpy(p[1]).cuda() for p in pairs]
torch.cuda.synchronize()
ctx = b200reg.Context(0)
args = ([t.data_ptr() for t in ds], [t.shape[0] for t in ds], [t.data_ptr() for t in dd], [t.shape[0] for t in dd], 16, 1)
fn = (lambda: ctx.icp_alignment_ptrs(*args)) if mode == "gicp" else (lambda: ctx.loop_closure_ptrs(*args))
fn()
ctx.set_profiling(True)
ctx.reset_profile()
for _ in range(jobs):
    res = fn()
prof = ctx.get_profile()
r0 = res[0] if mode == "gicp" else res[0][0]
print({k: round(v["ms"] / jobs, 3) for k, v in prof.items() if v["ms"] > 0}, "launches/job", {k: v["launches"] / jobs for k, v in prof.items() if v["ms"] > 0},
      "n_lin", [r.n_linearize for r in (res if mode == "gicp" else res[0])])
ctx.close()
