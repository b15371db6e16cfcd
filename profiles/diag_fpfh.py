#!/usr/bin/env python
"""Where the FPFH deviation between the CUDA path and the CPU oracle comes from (row a11; run on the GPU box):
    python profiles/diag_fpfh.py > out/diag_fpfh.txt
Compares (1) normals, (2) FPFH of the complete pipelines, (3) FPFH with the GPU's own normals fed to the oracle
(stage isolation: what remains is atan2f / summation order)."""
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))
import b200reg  # noqa: E402
from b200reg import synth  # noqa: E402
from oracle import oracle as orc  # noqa: E402

ctx = b200reg.Context(0)
for seed, n, voxel in ((2000, 8000, None), (2000, 100000, 0.3)):
    src, dst, _ = synth.make_pair(seed, n, n, mode="quatro", voxel=voxel)
    cl, = ctx.create_clouds([dst])
    ctx.fpfh([cl], 0.9, 1.5)
    gn, gf = ctx.get_fpfh(cl)
    on, osp, of = orc.fpfh(dst, 0.9, 1.5)
    ok = ~np.isnan(on[:, 0]) & ~np.isnan(gn[:, 0])
    dots = np.einsum("ij,ij->i", gn[ok], on[ok])
    err = np.abs(gf - of).max(1)
    _, of2 = orc.fpfh_from_normals(dst, np.where(np.isnan(gn), np.nan, gn), 1.5)
    err2 = np.abs(gf - of2).max(1)
    q = [0.5, 0.9, 0.98, 0.999, 1.0]
    print("seed %d  n=%d voxel=%s  points=%d" % (seed, n, voxel, len(dst)))
    print("  normals: 1-dot quantiles", np.quantile(1 - dots, q), " fraction with float-identical normals",
          float((gn[ok] == on[ok]).all(1).mean()))
    print("  FPFH |gpu - oracle| max/bin, own normals each  :", np.quantile(err, q))
    print("  FPFH |gpu - oracle| max/bin, SAME (gpu) normals:", np.quantile(err2, q), " frac > 1e-3:", float((err2 > 1e-3).mean()))
    cl.destroy()
ctx.close()
