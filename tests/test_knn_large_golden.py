"""Exact k-NN for k > 32, CPU side: the reference kd-tree's nearestKSearch answers (tests/golden/ref_nanoflann_knn_large.npz)
are re-derived by a numpy fp32 brute force that evaluates the reference's distance expression.  The reference keeps the
first-visited point among equal distances; the engine keeps the lower index.  So d2 columns must agree bit for bit,
indices wherever a distance is not tied, and index SETS within every group of equal distances that lies wholly inside
the first k.  For a group straddling rank k, the reference's indices must be members of the group."""
import importlib.util
import os
import subprocess
import zlib

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden", "ref_nanoflann_knn_large.npz")


def golden_module():
    spec = importlib.util.spec_from_file_location("make_knn_large_golden", os.path.join(REPO, "tests", "golden", "make_knn_large_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def golden_cases():
    """-> {cloud tag: cloud}, [(cloud tag, query set, k, queries, idx (nq, k), d2 (nq, k))] with the clouds' CRCs checked."""
    g = np.load(GOLDEN)
    clouds = golden_module().knn_large_clouds()
    for tag, c in clouds.items():
        assert zlib.crc32(c.tobytes()) == int(g[tag + "_crc"]), "the generated %s cloud drifted from the fixture" % tag
    cases = []
    for key in sorted(g.files):
        if not key.endswith("_idx"):
            continue
        tag, qn, k = key[:-4].split("_")
        cases.append((tag, qn, int(k), g["%s_q_%s" % (tag, qn)], g[key], g[key[:-4] + "_d2"]))
    return clouds, cases


def all_d2(cloud, q):
    """The reference's fp32 squared distance of q to every point: diff = query - point, ((dx*dx) + dy*dy) + dz*dz."""
    diff = np.asarray(q, np.float32)[None, :3] - cloud[:, :3]
    return (diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2]


def brute_knn(cloud, q, k):
    """The engine's contract for one query: the k smallest (d2, index) pairs ascending, among points with d2 below +inf
    (a NaN query has none); the rest of the row is (-1, FLT_MAX)."""
    d2 = all_d2(cloud, q)
    ok = np.flatnonzero(d2 < np.float32(np.inf))
    o = ok[np.lexsort((ok, d2[ok]))][:k]
    idx = np.full(k, -1, np.int32)
    dd = np.full(k, np.finfo(np.float32).max, np.float32)
    idx[:len(o)] = o
    dd[:len(o)] = d2[o]
    return idx, dd


def check_reference_row(cloud, q, k, idx, d2):
    """A reference row against the brute force, tie-aware (module docstring).  Returns the number of tied groups seen."""
    bi, bd = brute_knn(cloud, q, k)
    assert np.array_equal(d2.view(np.uint32), bd.view(np.uint32))
    full = all_d2(cloud, q)
    ties = 0
    for v in np.unique(bd):
        mine = np.sort(idx[d2 == v])
        group = np.sort(np.flatnonzero(full == v))
        if len(group) > 1:
            ties += 1
        if v == bd[-1] and len(group) > len(mine):  # straddles rank k: any members of the group
            assert np.all(np.isin(mine, group))
        else:
            assert np.array_equal(mine, group)
    return ties


def test_golden_knn_large_equals_numpy_brute_force():
    clouds, cases = golden_cases()
    assert len(cases) == 5 * (3 + 3 + 2)  # k x (raw / vox: self, shift, far; lattice: self, shift)
    ties = {"lattice": 0, "raw": 0, "vox": 0}
    for tag, qn, k, q, idx, d2 in cases:
        assert idx.shape == (len(q), k) and d2.shape == (len(q), k)
        for i in range(len(q)):
            ties[tag] += check_reference_row(clouds[tag], q[i], k, idx[i], d2[i])
    assert ties["lattice"] > 100  # the lattice exercises equal distances inside and across rank k


def test_golden_covers_what_it_claims():
    clouds, cases = golden_cases()
    ks = sorted({k for _, _, k, _, _, _ in cases})
    assert ks == [33, 64, 100, 256, 1000]
    for tag, qn, k, q, idx, d2 in cases:
        assert np.all(idx >= 0) and np.all(idx < len(clouds[tag]))  # k < n everywhere: no padding in the reference rows
        if qn == "far":
            assert np.all(d2[:, 0] > 400.0 ** 2)
        if qn == "self":
            assert np.all(d2[:, 0] == 0)
    # the lattice: at some k, the k-th distance is shared with points beyond rank k
    straddle = 0
    for tag, qn, k, q, idx, d2 in cases:
        if tag == "lattice":
            for i in range(len(q)):
                straddle += int(np.sum(all_d2(clouds[tag], q[i]) == d2[i, -1]) > np.sum(d2[i] == d2[i, -1]))
    assert straddle > 0


CLIENT_SRC = os.path.join(REPO, "tests", "cpp", "kdtree_knn_client.cpp")


def build_knn_client(tmp, pcl_config=False):
    from b200reg.build import build_native
    from test_radius_golden import CSRC, HOST, MOCK_PCL
    build_native()
    exe = os.path.join(tmp, "kd_knn_client_pcl" if pcl_config else "kd_knn_client")
    extra = ["-I" + MOCK_PCL, "-DB200REG_EXPECT_PCL"] if pcl_config else []
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-I" + HOST] + extra + ["-o", exe, CLIENT_SRC,
                           "-L" + CSRC, "-lb200reg", "-Wl,-rpath," + CSRC])
    return exe


@pytest.mark.parametrize("pcl_config", [False, True])
def test_kdtree_knn_client_compiles_as_cxx14(tmp_path, pcl_config):
    """nearestKSearch with k > 32 through NanoGICP::target_kdtree_ and a standalone KdTreeFLANN compiles and links."""
    assert os.path.exists(build_knn_client(str(tmp_path), pcl_config))
