#!/usr/bin/env python
"""Raw output bytes of every user of the shared radix sort, for comparing two builds of the package byte for byte.

Records, on seeded inputs:
  - b200reg_index_tap on clouds of 1, 8, 9, 2047, 2048, 2049 and 100k points (keys, points, rank, tree records, root);
  - b200reg_sort_tap with 30- and 32-bit keys (duplicates, sizes around the 2048-key tile);
  - b200reg_radius_search, sorted and unsorted, including one call with more than 2^23 neighbours (several chunks);
  - keyframe assembly with the voxel grid (b200reg_assemble_clouds), the index-overflow case included;
  - b200reg_clouds_fpfh + b200reg_get_fpfh;
  - b200reg_match_tap, optimized and advanced;
  - b200reg_quatro_align with the correspondences;
  - b200reg_perform_loop_closure: its results, Quatro infos and the four loop clouds.
The .npz is written with fixed member timestamps, so two runs that computed the same bytes give identical files.
    python profiles/sort_users_bytes.py --pkg DIR --out FILE.npz   (DIR holds the b200reg package to import)
"""
import argparse
import io
import os
import sys
import zipfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pkg", default=os.path.join(REPO, "fast-lio-sam-qn_b200"))
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    sys.path[:0] = [os.path.abspath(a.pkg), os.path.join(REPO, "tests")]
    import b200reg
    from b200reg import native, synth
    import voxel_cases as vc
    rec = {}

    def put(name, x):
        if isinstance(x, dict):
            for k in sorted(x):
                put("%s/%s" % (name, k), x[k])
        elif isinstance(x, (list, tuple)):
            for i, v in enumerate(x):
                put("%s/%d" % (name, i), v)
        else:
            rec[name] = np.frombuffer(np.ascontiguousarray(np.asarray(x)).tobytes(), np.uint8)

    ctx = b200reg.Context(0)
    rng = np.random.default_rng(2024)

    # index build
    sizes = (1, 8, 9, 2047, 2048, 2049, 100000)
    clouds = [rng.normal(0, 10, (n, 3)).astype(np.float32) for n in sizes]
    for n, o in zip(sizes, ctx.index_tap(clouds)):
        put("index_tap/%d" % n, o)

    # shared sort
    for bits in (30, 32):
        hi = 1 << bits
        keys = [rng.integers(0, hi, n, dtype=np.uint64).astype(np.uint32) for n in (1, 2047, 2049, 100000)]
        keys.append(rng.integers(0, 64, 70000, dtype=np.uint64).astype(np.uint32))  # long runs of equal keys
        vals = [rng.integers(0, 1 << 32, len(k), dtype=np.uint64).astype(np.uint32) for k in keys]
        put("sort_tap/%d" % bits, ctx.sort_tap(keys, vals, key_bits=bits))

    # radius search
    cloud = np.ascontiguousarray(synth.make_pair(31, 30000)[1][:, :3])
    cl, = ctx.create_clouds([cloud])
    q = np.concatenate([cloud[::7] + rng.normal(0, 0.3, (len(cloud[::7]), 3)).astype(np.float32),
                        rng.normal(0, 30, (500, 3)).astype(np.float32)])
    for sorted_ in (True, False):
        put("radius/%d" % sorted_, ctx.radius_search(cl, q, 4.0, sorted=sorted_))
    cl.destroy()
    cloud = np.ascontiguousarray(synth.make_pair(32, 20000)[1][:, :3])
    cl, = ctx.create_clouds([cloud])
    for sorted_ in (True, False):
        off, idx, d2 = ctx.radius_search(cl, cloud[::20], 1e12, sorted=sorted_)
        assert off[-1] > (1 << 23)
        put("radius_chunked/%d" % sorted_, (off, idx, d2))
    cl.destroy()

    # keyframe assembly + voxel grid (one job overflows the index guard)
    seq = vc.sweep_sequence(synth)
    kclouds = [vc.run_total(1, 101), vc.guard_above(16), vc.own_voxels(14), vc.index_wrap(17), seq["clouds"][3] + np.float32(0),
               vc.run_total(2049, 102), vc.guard_below(15), vc.one_voxel(13)]
    kf = ctx.keyframes()
    for k, c in enumerate(kclouds):
        kf.add(c, np.eye(4), float(k))
    idx = np.arange(len(kclouds), dtype=np.int32)
    for leaf in (1.0, 0.3):
        cfg = b200reg.default_loop_config()
        cfg.enable_quatro, cfg.enable_submap_matching, cfg.voxel_res = 1, 0, leaf
        sc, dc = kf.assemble(idx, idx, cfg)
        for i, c in enumerate(sc + dc):
            put("assemble/%g/%d" % (leaf, i), ctx.cloud_points(c))
            c.destroy()
    kf.destroy()

    # descriptors, matcher, Quatro
    src, dst = synth.make_pair(2003, 100000, mode="quatro", voxel=0.3)[:2]
    cs, cd = ctx.create_clouds([src, dst])
    ctx.fpfh([cs, cd])
    put("fpfh", [ctx.get_fpfh(cs), ctx.get_fpfh(cd)])
    fs, fd = ctx.get_fpfh(cs)[1], ctx.get_fpfh(cd)[1]
    fi, fj = (fs, fd) if len(fs) >= len(fd) else (fd, fs)
    for adv in (False, True):
        put("match_tap/%d" % adv, ctx.match_tap([(fi, fj), (fi[:3000], fi[:2047])], advanced=adv))
    for mc in (200, 0):  # 0: advancedMatching
        prm = native.default_quatro_params()
        if mc:
            prm.max_corres = mc
        else:
            prm.use_optimized_matching = 0
        info = ctx.quatro_align([cs], [cd], params=prm, want_corr=True)[0]
        put("quatro_align/%s" % (mc or "advanced"), {k: v for k, v in info.items() if k in ("T", "corr", "valid", "n_mutual",
                                                                                            "n_corr", "clique_size")})
    cs.destroy(); cd.destroy()

    # loop closure over a keyframe store, with its loop clouds
    s = synth.make_sequence(7, 140, pts_per_keyframe=6000, spacing=3.0, speed=8.0)
    kf = ctx.keyframes()
    for c, T, t in zip(s["clouds"], s["poses"], s["stamps"]):
        kf.add(c, T, t)
    queries = np.array([137, 139, 118], np.int32)
    closest = kf.fetch_closest(queries)
    ctx.set_loop_clouds(15)
    res, qi = kf.perform_loop_closure(queries, closest)
    put("loop/closest", closest)
    put("loop/results", [{k: np.asarray(v) for k, v in r.items()} for r in res])
    put("loop/quatro", [{k: np.asarray(v) for k, v in r.items()} for r in qi])
    for kind in (1, 2, 4, 8):
        put("loop/clouds/%d" % kind, ctx.loop_clouds(kind))
    ctx.set_loop_clouds(0)
    kf.destroy()
    ctx.close()

    with zipfile.ZipFile(a.out, "w") as z:
        for k in sorted(rec):
            buf = io.BytesIO()
            np.save(buf, rec[k])
            z.writestr(zipfile.ZipInfo(k + ".npy"), buf.getvalue())
    print("%d records -> %s" % (len(rec), a.out))


if __name__ == "__main__":
    main()
