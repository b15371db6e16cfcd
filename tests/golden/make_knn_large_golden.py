#!/usr/bin/env python
"""Generates tests/golden/ref_nanoflann_knn_large.npz: KdTreeFLANN::nearestKSearch answers of the REFERENCE kd-tree for k > 32.

    python tests/golden/make_knn_large_golden.py

Uses oracle.RefNanoflann, the reference's own nanoflann built into oracle/_ref by oracle/Makefile (target `ref`), and records
k x (index, d2) rows for
  * a seeded KITTI-shaped 20k scan, raw and 0.3 m-voxelised, with the CRC32 of each generated cloud;
  * k in 33, 64, 100, 256 and 1000;
  * sampled self, shifted and far (400 m away) queries;
  * a 12 x 12 x 12 lattice of pitch 0.5, where many points share one squared distance (ties across rank k).
The reference keeps the first-visited point among equal distances, so where a tie straddles rank k its indices are one valid
choice among several; the tests check them against a brute force with that in mind.  Only this fixture is written.  The
tests read the .npz; they never need the reference tree.
"""
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))

from b200reg import synth  # noqa: E402

KS = (33, 64, 100, 256, 1000)


def knn_large_clouds():
    """The fixture's inputs: a seeded KITTI-shaped 20k scan, raw and 0.3 m-voxelised (x, y, z only), and a 12 x 12 x 12
    lattice of pitch 0.5 (every squared distance between its points is an exact multiple of 0.25)."""
    scan = synth.make_pair(5152, 20000)[1]
    raw = np.ascontiguousarray(scan[:, :3])
    vox = np.ascontiguousarray(synth.voxelize(scan, 0.3)[:, :3])
    g = np.arange(12, dtype=np.float32) * np.float32(0.5)
    lattice = np.ascontiguousarray(np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + np.float32(10.0))
    return {"raw": raw, "vox": vox, "lattice": lattice}


def query_sets(tag, cloud, rng):
    if tag == "lattice":
        return {"self": cloud[::72], "shift": cloud[5::72] + np.float32(0.25)}
    rows = np.sort(rng.choice(len(cloud), 12, replace=False))
    return {"self": cloud[rows],
            "shift": (cloud[rows] + rng.normal(0, 0.5, (12, 3))).astype(np.float32),
            "far": (cloud[rows[:4]] + np.float32(400.0)).astype(np.float32)}


def main():
    from oracle import oracle as orc
    assert os.path.exists(orc.ref_so_path()), "build oracle/_ref first (make -C oracle ref)"
    rng = np.random.default_rng(78)
    out = {}
    for tag, cloud in knn_large_clouds().items():
        out[tag + "_crc"] = np.array(zlib.crc32(cloud.tobytes()), np.uint32)
        tree = orc.RefNanoflann(cloud)
        for qn, q in query_sets(tag, cloud, rng).items():
            q = np.ascontiguousarray(q, np.float32)
            out["%s_q_%s" % (tag, qn)] = q
            for k in KS:
                assert k < len(cloud)  # the reference's KNNResultSet assumes k <= n
                idx, d2 = tree.knn(q, k)
                out["%s_%s_%d_idx" % (tag, qn, k)] = idx
                out["%s_%s_%d_d2" % (tag, qn, k)] = d2
        del tree
    np.savez_compressed(os.path.join(HERE, "ref_nanoflann_knn_large.npz"), **out)
    print("knn large golden:", sum(v.size for k, v in out.items() if k.endswith("_idx")), "neighbours")


if __name__ == "__main__":
    main()
