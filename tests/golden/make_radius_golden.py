#!/usr/bin/env python
"""Generates tests/golden/ref_nanoflann_radius.npz: KdTreeFLANN::radiusSearch answers of the REFERENCE kd-tree.

    python tests/golden/make_radius_golden.py <reference source tree>

Compiles ref_radius_shim.cpp (this directory) against the reference's own nanoflann_impl.hpp into a temporary directory
with the CPU oracle's flags (-O3, -ffp-contract=off: the FMA-free fp32 distance), then records, as CSR arrays in the
SORTED mode (RadiusResultSet through findNeighbors, std::sort with IndexDist_Sorter):
  * a seeded KITTI-shaped 20k scan, raw and 0.3 m-voxelised, with the CRC32 of each generated cloud;
  * sampled self, shifted and far (400 m away: empty) queries at squared radii 0.09, 0.81, 2.25 and 25;
  * a 6 x 6 x 6 lattice of pitch 0.5 whose squared distances land exactly on the bounds 0.25, 0.5, 1.0 and 1.25.
The unsorted mode returns the same sets in the tree's visit order (checked here), which nothing but that tree reproduces,
so only the sets are kept.  Only this fixture is written.  The tests read the .npz; they never need the reference tree.
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))

from b200reg import synth  # noqa: E402

RADIUS_SQ = (0.09, 0.81, 2.25, 25.0)  # squared radii, passed to radiusSearch unchanged (0.3, 0.9, 1.5, 5 m balls)
LATTICE_SQ = (0.25, 0.5, 1.0, 1.25)   # squared lattice distances: every one of them lands exactly on some bound


def radius_clouds():
    """The fixture's inputs: a seeded KITTI-shaped 20k scan, raw and 0.3 m-voxelised (x, y, z only), and a 6 x 6 x 6 lattice
    of pitch 0.5 (every squared distance between its points is an exact multiple of 0.25)."""
    scan = synth.make_pair(5150, 20000)[1]
    raw = np.ascontiguousarray(scan[:, :3])
    vox = np.ascontiguousarray(synth.voxelize(scan, 0.3)[:, :3])
    g = np.arange(6, dtype=np.float32) * np.float32(0.5)
    lattice = np.ascontiguousarray(np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + np.float32(10.0))
    return {"raw": raw, "vox": vox, "lattice": lattice}


def build_shim(ref_tree, out_dir):
    inc = os.path.join(ref_tree, "third_party", "nano_gicp", "include")
    assert os.path.exists(os.path.join(inc, "nano_gicp", "impl", "nanoflann_impl.hpp")), "not a reference source tree: " + ref_tree
    so = os.path.join(out_dir, "libref_radius.so")
    subprocess.check_call(["g++", "-O3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-w", "-I" + inc, "-shared", "-o", so,
                           os.path.join(HERE, "ref_radius_shim.cpp")])
    lib = C.CDLL(so)
    lib.ref_radius_build.restype = C.c_void_p
    return lib


def radius_golden(lib):
    rng = np.random.default_rng(77)
    out = {}
    for tag, cloud in radius_clouds().items():
        out[tag + "_crc"] = np.array(zlib.crc32(cloud.tobytes()), np.uint32)
        h = C.c_void_p(lib.ref_radius_build(cloud.ctypes.data_as(C.c_void_p), len(cloud)))
        if tag == "lattice":
            qsets = {"self": cloud.copy(), "shift": cloud[::7] + np.float32(0.25)}
            radii = LATTICE_SQ
        else:
            rows = np.sort(rng.choice(len(cloud), 32, replace=False))
            qsets = {"self": cloud[rows],
                     "shift": (cloud[rows] + rng.normal(0, 0.5, (32, 3))).astype(np.float32),
                     "far": (cloud[rows[:8]] + np.float32(400.0)).astype(np.float32)}
            radii = RADIUS_SQ
        for qn, q in qsets.items():
            q = np.ascontiguousarray(q, np.float32)
            out["%s_q_%s" % (tag, qn)] = q
            for r2 in radii:
                offs, idxs, d2s = [0], [], []
                for i in range(len(q) if r2 < 10 else min(len(q), 6)):  # the 5 m balls hold thousands: the first rows only
                    sets = []
                    for sorted_ in (1, 0):
                        cap = len(cloud)
                        ii = np.empty(cap, np.int32)
                        dd = np.empty(cap, np.float32)
                        m = lib.ref_radius_search(h, q[i].ctypes.data_as(C.c_void_p), C.c_double(r2), sorted_, cap,
                                                  ii.ctypes.data_as(C.c_void_p), dd.ctypes.data_as(C.c_void_p))
                        sets.append((ii[:m].copy(), dd[:m].copy()))
                    (si, sd), (ui, ud) = sets
                    o = np.argsort(ui, kind="stable")
                    assert np.array_equal(np.sort(si), ui[o]) and np.array_equal(sd[np.argsort(si, kind="stable")], ud[o])
                    idxs.append(si)
                    d2s.append(sd)
                    offs.append(offs[-1] + len(si))
                key = "%s_%s_%g" % (tag, qn, r2)
                out[key + "_off"] = np.array(offs, np.int64)
                out[key + "_idx"] = np.concatenate(idxs).astype(np.int32)
                out[key + "_d2"] = np.concatenate(d2s).astype(np.float32)
        lib.ref_radius_free(h)
    np.savez_compressed(os.path.join(HERE, "ref_nanoflann_radius.npz"), **out)
    print("radius golden:", sum(v.size for k, v in out.items() if k.endswith("_idx")), "neighbours")


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    with tempfile.TemporaryDirectory() as tmp:
        radius_golden(build_shim(sys.argv[1], tmp))


if __name__ == "__main__":
    main()
