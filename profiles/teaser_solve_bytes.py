#!/usr/bin/env python
"""Raw bytes of the TEASER++ solve on all three device paths, for comparing two builds of the package byte for byte.

Records T (raw fp64 bytes), the info counters, the clique and, end to end, the correspondences of:
  - b200reg_quatro_solve_tap on every tests/teaser_ref.py crafted case, on each path its size allows;
  - teaser_ref.natural_set at n = 2..512 (shared, global, wide), 513..8192 (global, wide) and 8193, 20000 (wide);
  - b200reg_quatro_align on a 0.3 m-voxelised 100k pair at max_corres 200, 509, 1000, 8189 and with advancedMatching;
  - the 0.2 m sub-map pair of tests/test_gpu_quatro_big.py at max_corres 1000 and 8189 (optimizedMatching sets beyond
    512, end to end) and with advancedMatching (the wide path, end to end).
The .npz is written with fixed member timestamps, so two runs that computed the same bytes give identical files.
    python profiles/teaser_solve_bytes.py --pkg DIR --out FILE.npz   (DIR holds the b200reg package to import)
"""
import argparse
import io
import os
import sys
import zipfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHARED_CAP, GLOBAL_CAP = 512, 8192


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pkg", default=os.path.join(REPO, "fast-lio-sam-qn_b200"))
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    sys.path[:0] = [os.path.abspath(a.pkg), os.path.join(REPO, "tests")]
    import b200reg
    from b200reg import native, synth
    import teaser_ref as tr
    from test_gpu_quatro_big import make_submap_pair
    rec = {}

    def put(name, info):
        rec[name + "/T"] = np.frombuffer(np.ascontiguousarray(info["T"], np.float64).tobytes(), np.uint8)
        rec[name + "/counters"] = np.array([info["valid"], info.get("n_mutual", -1), info.get("n_corr", -1), info["clique_size"],
                                            info["gnc_iterations"]], np.int64)
        for k in ("clique", "corr"):
            if k in info:
                rec[name + "/" + k] = np.asarray(info[k], np.int32)

    ctx = b200reg.Context(0)

    def tap(name, S, D, prm):
        p = native.default_quatro_params()
        p.noise_bound, p.rot_gnc_factor, p.rot_cost_thr, p.rot_max_iter = prm.noise_bound, prm.gnc_factor, prm.cost_thr, prm.max_iter
        n = len(S)
        paths = (["shared"] if n <= SHARED_CAP else []) + (["global"] if n <= GLOBAL_CAP else []) + ["wide"]
        for path in paths:
            put("%s/%s" % (name, path), ctx.quatro_solve_tap(S, D, p, path=path))

    for c in tr.crafted_cases():
        tap("crafted_" + c.name, c.S, c.D, c.prm)
    for n in (2, 37, 256, 500, 512, 513, 1000, 8192, 8193, 20000):
        S, D = tr.natural_set(n, 7000 + n, noise=0.1, yaw=-2.5)
        tap("natural_%d" % n, S, D, tr.Params(noise_bound=0.3))
    pairs = [("voxel0.3_100k", synth.make_pair(2003, 100000, mode="quatro", voxel=0.3)[:2], (200, 509, 1000, 8189, 0)),
             ("submap0.2", make_submap_pair(leaf=0.2)[:2], (1000, 8189, 0))]
    for name, (src, dst), caps in pairs:
        cs, cd = ctx.create_clouds([src, dst])
        for mc in caps:  # 0: advancedMatching
            prm = native.default_quatro_params()
            if mc:
                prm.max_corres = mc
            else:
                prm.use_optimized_matching = 0
            put("align_%s/%s" % (name, mc or "advanced"), ctx.quatro_align([cs], [cd], params=prm, want_corr=True)[0])
        cs.destroy(); cd.destroy()
    ctx.close()
    with zipfile.ZipFile(a.out, "w") as z:
        for k in sorted(rec):
            buf = io.BytesIO()
            np.save(buf, rec[k])
            z.writestr(zipfile.ZipInfo(k + ".npy"), buf.getvalue())
    print("%d records -> %s" % (len(rec), a.out))


if __name__ == "__main__":
    main()
