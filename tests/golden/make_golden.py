#!/usr/bin/env python
"""Generates the committed golden fixtures.  Run where the reference source tree is available (needs
oracle/_ref = the reference's own nanoflann kd-tree); the tests only read the .npz files.

  knn_ref_nanoflann.npz  exact k-NN answers of the REFERENCE kd-tree
                         (third_party/nano_gicp/include/nano_gicp/impl/nanoflann_impl.hpp, configured as in
                         nano_gicp/nanoflann.hpp:100-114) on a 3000-point KITTI-shaped cloud
  gicp_oracle_3k.npz     the CPU oracle's Nano-GICP outputs on a 3000 x 3500 pair (covariances, one
                         linearization, the full align) -- pins the oracle against silent drift
  quatro_oracle_2k.npz   the CPU oracle's Quatro outputs on a 2000 x 2300 pair (normals / FPFH samples, both matchers'
                         correspondence lists, both solves) -- same purpose (`python make_golden.py quatro` writes
                         only this one)
  ref_nanoflann_samples.npz  the REFERENCE kd-tree's k-NN answers on sampled rows of the query sets the oracle and the
                         CUDA k-NN are checked against, and the oracle's align with that kd-tree behind it
                         (`python make_golden.py ref` writes only this one)
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
from oracle import oracle  # noqa: E402


def quatro_golden():
    src, dst, Texp = synth.make_pair(4343, 2000, 2300, mode="quatro")
    src3, dst3 = np.ascontiguousarray(src[:, :3]), np.ascontiguousarray(dst[:, :3])
    ns, _, fs = oracle.fpfh(src3)
    nd, _, fd = oracle.fpfh(dst3)
    opt, mutual = oracle.match(src3, dst3, fs, fd)
    adv = oracle.match_advanced(src3, dst3, fs, fd)
    so, sa = oracle.quatro_solve(src3, dst3, opt), oracle.quatro_solve(src3, dst3, adv)
    np.savez_compressed(os.path.join(HERE, "quatro_oracle_2k.npz"), src=src3, dst=dst3, T_expected=Texp,
                        normals_src_sample=ns[::25], fpfh_src_sample=fs[::25], fpfh_dst_sample=fd[::25],
                        corr_opt=opt, n_mutual=len(mutual), corr_adv=adv,
                        T_opt=so["T"], clique_opt=so["clique"], gnc_opt=so["gnc_iters"],
                        T_adv=sa["T"], clique_adv=sa["clique"], gnc_adv=sa["gnc_iters"])
    print("quatro golden:", len(opt), "optimized /", len(adv), "advanced correspondences; cliques", len(so["clique"]), len(sa["clique"]))


def ref_samples_golden():
    """The reference kd-tree's answers on the query sets of tests/test_oracle.py and tests/test_gpu_gicp.py, on a fixed
    seeded sample of rows; the CRC32 of each generated cloud pins the synthetic input."""
    rng = np.random.default_rng(2024)
    out = {}

    def sets(tag, src, dst, specs):
        out[tag + "_crc"] = np.array([zlib.crc32(src.tobytes()), zlib.crc32(dst.tobytes())], np.uint32)
        ref = oracle.RefNanoflann(dst)
        for name, (q, k) in specs.items():
            rows = np.sort(rng.choice(len(q), min(len(q), 1024 if k == 1 else 128), replace=False)).astype(np.int32)
            out["%s_rows_%s" % (tag, name)] = rows
            out["%s_idx_%s" % (tag, name)], out["%s_d2_%s" % (tag, name)] = ref.knn(q[rows], k)

    src, dst, _ = synth.make_pair(77, 6000, 7000)
    sets("cpu", src, dst, {"a": (dst[:2000], 15), "b": (src, 1), "c": (src[:500] + np.float32(2.5), 15)})
    assert oracle.use_ref_nanoflann(True) == 0
    r = oracle.gicp_align(src, dst)
    oracle.use_ref_nanoflann(False)
    out["cpu_T_ref"], out["cpu_fitness_ref"] = r["T"], r["fitness"]
    src, dst, _ = synth.make_pair(1000, 20000)
    sets("gpu", src, dst, {"a": (src, 1), "b": (dst[:8000], 15), "c": (src + np.float32(3.0), 1), "d": (src[:4000], 20)})
    np.savez_compressed(os.path.join(HERE, "ref_nanoflann_samples.npz"), **out)


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "quatro":
        return quatro_golden()
    assert os.path.exists(oracle.ref_so_path()), "build oracle/_ref first (make -C oracle ref)"
    if len(sys.argv) > 1 and sys.argv[1] == "ref":
        return ref_samples_golden()
    src, dst, Texp = synth.make_pair(4242, 3000, 3500)
    src3, dst3 = np.ascontiguousarray(src[:, :3]), np.ascontiguousarray(dst[:, :3])
    # ---- k-NN from the reference kd-tree
    ref = oracle.RefNanoflann(dst3)
    rng = np.random.default_rng(1)
    q_self = dst3[:600]
    q_shift = (src3[:400] + rng.normal(0, 1.5, (400, 3))).astype(np.float32)
    i15, d15 = ref.knn(q_self, 15)
    i1, d1 = ref.knn(q_shift, 1)
    i20, d20 = ref.knn(q_shift[:100], 20)
    np.savez_compressed(os.path.join(HERE, "knn_ref_nanoflann.npz"), cloud=dst3, q_self=q_self, q_shift=q_shift,
                        idx15=i15, d15=d15, idx1=i1, d1=d1, idx20=i20, d20=d20)
    # ---- oracle GICP
    oracle.use_ref_nanoflann(False)
    cov_s = oracle.covariances(src3, 15)
    cov_t = oracle.covariances(dst3, 15)
    lin = oracle.linearize(src3, dst3, cov_s, cov_t, np.eye(4))
    res = oracle.gicp_align(src3, dst3, want_trace=True)
    np.savez_compressed(os.path.join(HERE, "gicp_oracle_3k.npz"), src=src3, dst=dst3, T_expected=Texp,
                        cov_src_sample=cov_s[::60], cov_tgt_sample=cov_t[::70], H=lin["H"], b=lin["b"], err=lin["err"],
                        corr=lin["corr"], sqd=lin["sqd"], T=res["T"], Tf=res["Tf"], fitness=res["fitness"],
                        converged=res["converged"], iterations=res["iterations"], n_linearize=res["n_linearize"],
                        n_error=res["n_error"], trace=res["trace"])
    quatro_golden()
    ref_samples_golden()
    print("wrote", os.listdir(HERE))


if __name__ == "__main__":
    main()
