"""Fixed-radius search, CPU side: the reference kd-tree's radiusSearch answers (tests/golden/ref_nanoflann_radius.npz) are
re-derived by a numpy fp32 brute force that evaluates the reference's distance expression, and the KdTreeFLANN facade
compiles as C++14 in both facade configurations."""
import importlib.util
import os
import subprocess
import zlib

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden", "ref_nanoflann_radius.npz")
HOST = os.path.join(REPO, "fast-lio-sam-qn_b200", "host")
CSRC = os.path.join(REPO, "fast-lio-sam-qn_b200", "csrc")
MOCK_PCL = os.path.join(REPO, "tests", "cpp", "mock_pcl")
CLIENT_SRC = os.path.join(REPO, "tests", "cpp", "kdtree_client.cpp")


def golden_module():
    spec = importlib.util.spec_from_file_location("make_radius_golden", os.path.join(REPO, "tests", "golden", "make_radius_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def golden_cases():
    """-> {cloud tag: cloud}, [(cloud tag, query set, r2, queries, offsets, idx, d2)] with the clouds' CRCs checked."""
    g = np.load(GOLDEN)
    clouds = golden_module().radius_clouds()
    for tag, c in clouds.items():
        assert zlib.crc32(c.tobytes()) == int(g[tag + "_crc"]), "the generated %s cloud drifted from the fixture" % tag
    cases = []
    for k in sorted(g.files):
        if not k.endswith("_off"):
            continue
        tag, qn, r2 = k[:-4].split("_")
        off = g[k]
        q = g["%s_q_%s" % (tag, qn)][:len(off) - 1]
        cases.append((tag, qn, float(r2), q, off, g[k[:-4] + "_idx"], g[k[:-4] + "_d2"]))
    return clouds, cases


def brute_force(cloud, q, r2):
    """The reference's fp32 squared distance (diff = query - point, ((dx*dx) + dy*dy) + dz*dz) and RadiusResultSet's strict
    test; -> (indices ascending, their d2)."""
    diff = q[None, :].astype(np.float32) - cloud
    d2 = (diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2]
    idx = np.flatnonzero(d2 < np.float32(r2))
    return idx.astype(np.int32), d2[idx]


def test_golden_radius_sets_equal_numpy_brute_force():
    clouds, cases = golden_cases()
    assert len(cases) == 2 * 4 + 2 * 3 * 4  # lattice: 2 query sets x 4 radii; raw / vox: 3 query sets x 4 radii
    bound_hits = 0
    for tag, qn, r2, q, off, idx, d2 in cases:
        cloud = clouds[tag]
        for i in range(len(q)):
            gi, gd = idx[off[i]:off[i + 1]], d2[off[i]:off[i + 1]]
            bi, bd = brute_force(cloud, q[i], r2)
            o = np.argsort(gi, kind="stable")
            assert np.array_equal(gi[o], bi), (tag, qn, r2, i)
            assert np.array_equal(gd[o].view(np.uint32), bd.view(np.uint32)), (tag, qn, r2, i)
            # IndexDist_Sorter: ascending d2 (ties in unspecified order)
            assert np.all(np.diff(gd) >= 0), (tag, qn, r2, i)
            if tag == "lattice":
                diff = q[i][None, :] - cloud
                full = (diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2]
                bound_hits += int(np.sum(full == np.float32(r2)))
    assert bound_hits > 0  # the lattice puts points exactly on the bound, and they are excluded


def test_golden_covers_what_it_claims():
    _, cases = golden_cases()
    totals = {(t, qn, r2): int(off[-1]) for t, qn, r2, _, off, _, _ in cases}
    assert all(totals[("raw", "far", r2)] == 0 and totals[("vox", "far", r2)] == 0 for r2 in (0.09, 0.81, 2.25, 25.0))
    assert totals[("raw", "self", 25.0)] > 10000 and totals[("vox", "self", 0.09)] > 0


def _build(tmp, pcl_config=False):
    from b200reg.build import build_native
    build_native()
    exe = os.path.join(tmp, "kd_client_pcl" if pcl_config else "kd_client")
    extra = ["-I" + MOCK_PCL, "-DB200REG_EXPECT_PCL"] if pcl_config else []
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-I" + HOST] + extra + ["-o", exe, CLIENT_SRC,
                           "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    return exe


@pytest.mark.parametrize("pcl_config", [False, True])
def test_kdtree_client_compiles_as_cxx14(tmp_path, pcl_config):
    """<nano_gicp/nanoflann.hpp>, KdTreeFLANN's surface and NanoGICP::source_kdtree_ / target_kdtree_ compile and link."""
    assert os.path.exists(_build(str(tmp_path), pcl_config))
