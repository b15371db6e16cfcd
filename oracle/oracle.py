"""ctypes binding of the CPU oracle (oracle/liboracle.so) -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
leg may import this module.  The product (fast-lio-sam-qn_b200/) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class GicpParams(C.Structure):
    # effective defaults of the reference deployment (SURVEY.md App. A.1)
    _fields_ = [("k_correspondences", C.c_int), ("max_iterations", C.c_int), ("max_corr_dist", C.c_double),
                ("transformation_eps", C.c_double), ("rotation_eps", C.c_double), ("lm_max_iterations", C.c_int),
                ("lm_init_lambda_factor", C.c_double), ("regularization", C.c_int)]

    @staticmethod
    def default():
        return GicpParams(15, 32, 52.5, 0.01, 2e-3, 10, 1e-9, 3)


class GicpResult(C.Structure):
    _fields_ = [("T", C.c_double * 16), ("Tf", C.c_float * 16), ("fitness", C.c_double), ("converged", C.c_int),
                ("iterations", C.c_int), ("n_linearize", C.c_int), ("n_error", C.c_int), ("lm_failed", C.c_int),
                ("pad", C.c_int), ("ms_build", C.c_double), ("ms_cov", C.c_double), ("ms_align", C.c_double),
                ("ms_fitness", C.c_double)]


def build(force=False):
    """Compile liboracle.so (+ oracle/_ref when /root/reference is present)."""
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("oracle_gicp.cpp", "oracle_quatro.cpp", "linalg.hpp", "Makefile")]
    stale = force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if stale:
        subprocess.check_call(["make", "-C", _HERE, "-s", "all"], stdout=subprocess.DEVNULL)
    elif not os.path.exists(ref_so_path()) and os.path.exists("/root/reference"):
        subprocess.check_call(["make", "-C", _HERE, "-s", "ref"], stdout=subprocess.DEVNULL)
    return so


def ref_so_path():
    return os.path.join(_HERE, "_ref", "libref_nanoflann.so")


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.orc_linearize.restype = C.c_double
        _LIB.orc_compute_error.restype = C.c_double
        _LIB.orc_num_threads.restype = C.c_int
    return _LIB


def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] >= 3
    return a


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def num_threads():
    return lib().orc_num_threads()


def use_ref_nanoflann(enable=True):
    """Route the oracle's kNN through the reference's own nanoflann (oracle/_ref)."""
    if not enable:
        return lib().orc_use_ref_nanoflann(None)
    p = ref_so_path()
    if not os.path.exists(p):
        return -1
    return lib().orc_use_ref_nanoflann(p.encode())


def knn(pts, queries, k, brute=False):
    pts, queries = _f32(pts), _f32(queries)
    idx = np.empty((len(queries), k), np.int32)
    d2 = np.empty((len(queries), k), np.float32)
    fn = lib().orc_knn_bruteforce if brute else lib().orc_knn
    fn(_p(pts, C.c_float), len(pts), pts.shape[1], _p(queries, C.c_float), len(queries), queries.shape[1], k,
       _p(idx, C.c_int), _p(d2, C.c_float))
    return idx, d2


class RefNanoflann:
    """The reference's kd-tree (third_party/nano_gicp/.../nanoflann_impl.hpp) via oracle/_ref."""

    def __init__(self, pts):
        self.l = C.CDLL(ref_so_path())
        self.l.ref_nf_build.restype = C.c_void_p
        self.pts = _f32(pts)
        self.h = C.c_void_p(self.l.ref_nf_build(_p(self.pts, C.c_float), len(self.pts), self.pts.shape[1]))

    def knn(self, queries, k):
        q = _f32(queries)
        idx = np.empty((len(q), k), np.int32)
        d2 = np.empty((len(q), k), np.float32)
        self.l.ref_nf_knn(self.h, _p(q, C.c_float), len(q), q.shape[1], k, _p(idx, C.c_int), _p(d2, C.c_float))
        return idx, d2

    def __del__(self):
        try:
            self.l.ref_nf_free(self.h)
        except Exception:
            pass


def covariances_ex(pts, k=15, method=3):
    """RegularizationMethod: 0 NONE, 1 MIN_EIG, 2 NORMALIZED_MIN_EIG, 3 PLANE, 4 FROBENIUS (nano_gicp_impl.hpp:323-353)."""
    pts = _f32(pts)
    cov = np.empty((len(pts), 3, 3), np.float64)
    lib().orc_covariances_ex(_p(pts, C.c_float), len(pts), pts.shape[1], k, int(method), _p(cov, C.c_double))
    return cov


def covariances(pts, k=15, return_knn=False):
    pts = _f32(pts)
    cov = np.empty((len(pts), 3, 3), np.float64)
    kidx = np.empty((len(pts), k), np.int32)
    lib().orc_covariances(_p(pts, C.c_float), len(pts), pts.shape[1], k, _p(cov, C.c_double), _p(kidx, C.c_int))
    return (cov, kidx) if return_knn else cov


def transform_queries(T, pts):
    pts = _f32(pts)
    T = np.ascontiguousarray(T, np.float64)
    out = np.empty((len(pts), 3), np.float32)
    lib().orc_transform_queries(_p(T, C.c_double), _p(pts, C.c_float), len(pts), pts.shape[1], _p(out, C.c_float))
    return out


def transform_output(Tf, pts):
    pts = _f32(pts)
    Tf = np.ascontiguousarray(Tf, np.float32)
    out = np.empty((len(pts), 3), np.float32)
    lib().orc_transform_output(_p(Tf, C.c_float), _p(pts, C.c_float), len(pts), pts.shape[1], _p(out, C.c_float))
    return out


def linearize(src, tgt, cov_src, cov_tgt, T, max_corr_dist=52.5):
    src, tgt = _f32(src), _f32(tgt)
    cov_src = np.ascontiguousarray(cov_src, np.float64)
    cov_tgt = np.ascontiguousarray(cov_tgt, np.float64)
    T = np.ascontiguousarray(T, np.float64)
    H = np.empty((6, 6), np.float64)
    b = np.empty(6, np.float64)
    corr = np.empty(len(src), np.int32)
    sqd = np.empty(len(src), np.float32)
    mah = np.empty((len(src), 3, 3), np.float64)
    y = lib().orc_linearize(_p(src, C.c_float), len(src), src.shape[1], _p(tgt, C.c_float), len(tgt), tgt.shape[1],
                            _p(cov_src, C.c_double), _p(cov_tgt, C.c_double), _p(T, C.c_double),
                            C.c_double(max_corr_dist), _p(H, C.c_double), _p(b, C.c_double), _p(corr, C.c_int),
                            _p(sqd, C.c_float), _p(mah, C.c_double))
    return dict(H=H, b=b, err=y, corr=corr, sqd=sqd, mahal=mah)


def compute_error(src, tgt, cov_src, cov_tgt, T_lin, T_trial, max_corr_dist=52.5):
    """NanoGICP::compute_error at T_trial with the correspondences / Mahalanobis matrices of a linearize at T_lin."""
    src, tgt = _f32(src), _f32(tgt)
    cov_src = np.ascontiguousarray(cov_src, np.float64)
    cov_tgt = np.ascontiguousarray(cov_tgt, np.float64)
    Tl, Tt = np.ascontiguousarray(T_lin, np.float64), np.ascontiguousarray(T_trial, np.float64)
    return lib().orc_compute_error(_p(src, C.c_float), len(src), src.shape[1], _p(tgt, C.c_float), len(tgt), tgt.shape[1],
                                   _p(cov_src, C.c_double), _p(cov_tgt, C.c_double), _p(Tl, C.c_double), _p(Tt, C.c_double),
                                   C.c_double(max_corr_dist))


def gicp_align(src, tgt, params=None, guess=None, want_aligned=False, want_trace=False):
    """LoopClosure::icpAlignment restated (fast_lio_sam_qn/src/loop_closure.cpp:110-136)."""
    src, tgt = _f32(src), _f32(tgt)
    prm = params or GicpParams.default()
    res = GicpResult()
    aligned = np.empty((len(src), 3), np.float32) if want_aligned else None
    trace = np.zeros((prm.max_iterations, 64), np.float64) if want_trace else None
    g = None if guess is None else np.ascontiguousarray(guess, np.float64)
    rc = lib().orc_gicp_align(_p(src, C.c_float), len(src), src.shape[1], _p(tgt, C.c_float), len(tgt), tgt.shape[1],
                              C.byref(prm), None if g is None else _p(g, C.c_double), C.byref(res),
                              None if aligned is None else _p(aligned, C.c_float),
                              None if trace is None else _p(trace, C.c_double), prm.max_iterations)
    if rc != 0:
        raise RuntimeError("orc_gicp_align failed: %d" % rc)
    out = dict(T=np.array(res.T).reshape(4, 4), Tf=np.array(res.Tf, np.float32).reshape(4, 4), fitness=res.fitness,
               converged=bool(res.converged), iterations=res.iterations, n_linearize=res.n_linearize,
               n_error=res.n_error, lm_failed=bool(res.lm_failed), ms_build=res.ms_build, ms_cov=res.ms_cov,
               ms_align=res.ms_align, ms_fitness=res.ms_fitness)
    if want_aligned:
        out["aligned"] = aligned
    if want_trace:
        out["trace"] = trace[:res.n_linearize]
    return out


# ---------------------------------------------------------------------------------------------
# Quatro half (oracle/oracle_quatro.cpp)
class QuatroParams(C.Structure):
    _fields_ = [("fpfh_normal_radius", C.c_double), ("fpfh_radius", C.c_double), ("noise_bound", C.c_double),
                ("rot_gnc_factor", C.c_double), ("rot_cost_thr", C.c_double), ("rot_max_iter", C.c_int),
                ("max_corres", C.c_int), ("distance_threshold", C.c_double), ("tuple_scale", C.c_double),
                ("seed", C.c_uint64), ("use_optimized_matching", C.c_int), ("pad_", C.c_int)]

    @staticmethod
    def default():
        p = QuatroParams()
        lib().orc_quatro_default_params(C.byref(p))
        return p


def fpfh(pts, normal_radius=0.9, fpfh_radius=1.5):
    """-> (normals (n,3), spfh (n,33), fpfh (n,33)) float32; PCL NormalEstimation + FPFHEstimationOMP restated."""
    pts = _f32(pts)
    n = len(pts)
    nrm = np.empty((n, 3), np.float32)
    sp = np.empty((n, 33), np.float32)
    fp = np.empty((n, 33), np.float32)
    lib().orc_fpfh(_p(pts, C.c_float), n, pts.shape[1], C.c_double(normal_radius), C.c_double(fpfh_radius),
                   _p(nrm, C.c_float), _p(sp, C.c_float), _p(fp, C.c_float))
    return nrm, sp, fp


def fpfh_from_normals(pts, normals, fpfh_radius=1.5):
    pts = _f32(pts)
    nrm = np.ascontiguousarray(normals, np.float32)
    n = len(pts)
    sp = np.empty((n, 33), np.float32)
    fp = np.empty((n, 33), np.float32)
    lib().orc_fpfh_from_normals(_p(pts, C.c_float), n, pts.shape[1], _p(nrm, C.c_float), C.c_double(fpfh_radius),
                                _p(sp, C.c_float), _p(fp, C.c_float))
    return sp, fp


def match(src, dst, fsrc, fdst, params=None):
    """Matcher::optimizedMatching -> (corr (k,2) (src,dst), mutual (m,2) (i,j) in fi/fj numbering)."""
    src, dst = _f32(src), _f32(dst)
    fs = np.ascontiguousarray(fsrc, np.float32)
    fd = np.ascontiguousarray(fdst, np.float32)
    p = params or QuatroParams.default()
    corr = np.empty((p.max_corres + 8, 2), np.int32)
    mut = np.empty((min(len(src), len(dst)), 2), np.int32)
    nm = C.c_int()
    k = lib().orc_match(_p(src, C.c_float), len(src), src.shape[1], _p(dst, C.c_float), len(dst), dst.shape[1],
                        _p(fs, C.c_float), _p(fd, C.c_float), C.byref(p), _p(corr, C.c_int), C.byref(nm), _p(mut, C.c_int))
    return corr[:k].copy(), mut[:nm.value].copy()


def match_advanced(src, dst, fsrc, fdst, params=None, crosscheck=True, tuple_test=True):
    """Matcher::advancedMatching (matcher.cc:118-356) -> (k, 2) sorted unique (src, dst) pairs."""
    src, dst = _f32(src), _f32(dst)
    fs = np.ascontiguousarray(fsrc, np.float32)
    fd = np.ascontiguousarray(fdst, np.float32)
    p = params or QuatroParams.default()
    cap = 2 * (len(src) + len(dst))
    corr = np.empty((cap, 2), np.int32)
    k = lib().orc_match_advanced(_p(src, C.c_float), len(src), src.shape[1], _p(dst, C.c_float), len(dst), dst.shape[1],
                                 _p(fs, C.c_float), _p(fd, C.c_float), C.byref(p), int(crosscheck), int(tuple_test),
                                 _p(corr, C.c_int), cap)
    return corr[:min(k, cap)].copy()


def quatro_solve(src, dst, corr, params=None):
    src, dst = _f32(src), _f32(dst)
    corr = np.ascontiguousarray(corr, np.int32)
    p = params or QuatroParams.default()
    T = np.empty(16, np.float64)
    clique = np.empty(max(len(corr), 1), np.int32)
    cs, it = C.c_int(), C.c_int()
    valid = lib().orc_quatro_solve(_p(src, C.c_float), src.shape[1], _p(dst, C.c_float), dst.shape[1], _p(corr, C.c_int),
                                   len(corr), C.byref(p), _p(T, C.c_double), _p(clique, C.c_int), C.byref(cs), C.byref(it))
    return dict(T=T.reshape(4, 4), valid=bool(valid), clique=clique[:cs.value].copy(), gnc_iters=it.value)


def quatro_align(src, dst, params=None):
    """quatro<T>::align restated (third_party/Quatro/src/quatro_module.cc:48-79)."""
    src, dst = _f32(src), _f32(dst)
    p = params or QuatroParams.default()
    T = np.empty(16, np.float64)
    nc = C.c_int()
    t1, t2, t3 = C.c_double(), C.c_double(), C.c_double()
    valid = lib().orc_quatro_align(_p(src, C.c_float), len(src), src.shape[1], _p(dst, C.c_float), len(dst), dst.shape[1],
                                   C.byref(p), _p(T, C.c_double), C.byref(nc), C.byref(t1), C.byref(t2), C.byref(t3))
    return dict(T=T.reshape(4, 4), valid=bool(valid), n_corr=nc.value, ms_fpfh=t1.value, ms_match=t2.value, ms_solve=t3.value)


def coarse_to_fine(src, dst, qparams=None, gparams=None, quatro_T=None):
    """LoopClosure::coarseToFineAlignment (fast_lio_sam_qn/src/loop_closure.cpp:138-159).

    quatro_T: use this coarse transform instead of running the oracle's own Quatro stage (stage isolation)."""
    q = quatro_align(src, dst, qparams) if quatro_T is None else dict(T=np.asarray(quatro_T, np.float64), valid=True)
    out = dict(quatro=q, valid=False, T=q["T"].copy())
    if not q["valid"]:
        return out
    src = _f32(src)
    coarse = src.copy()
    # transformPcd: Matrix4d, double math, cast to float (utilities.hpp:164-175, SURVEY App. B.2)
    coarse[:, :3] = (src[:, :3].astype(np.float64) @ q["T"][:3, :3].T + q["T"][:3, 3]).astype(np.float32)
    g = gicp_align(coarse, dst, gparams)
    out.update(gicp=g, T=g["Tf"].astype(np.float64) @ q["T"], fitness=g["fitness"], converged=g["converged"],
               valid=bool(g["converged"] and g["fitness"] < 1.5))
    return out


# ---------------------------------------------------------------------------------------------
# "next" rows (SURVEY §8f): cloud assembly and candidate search
def transform_pcd(pts, T):
    pts = np.ascontiguousarray(pts, np.float32)
    T = np.ascontiguousarray(T, np.float64)
    out = np.empty_like(pts)
    lib().orc_transform_pcd(_p(pts, C.c_float), len(pts), pts.shape[1], _p(T, C.c_double), _p(out, C.c_float))
    return out


def pose_pcd_ingest(world_pts, position, quat_xyzw):
    """PosePcd::PosePcd (pose_pcd.hpp:21-43): -> (cloud in the LiDAR frame (n,4) float32, pose_eig_ (4,4))."""
    pts = np.ascontiguousarray(world_pts, np.float32)
    pos = np.ascontiguousarray(position, np.float64)
    q = np.ascontiguousarray(quat_xyzw, np.float64)
    out = np.empty_like(pts)
    pose = np.empty(16, np.float64)
    lib().orc_pose_pcd_ingest(_p(pts, C.c_float), len(pts), pts.shape[1], _p(pos, C.c_double), _p(q, C.c_double), _p(out, C.c_float),
                              _p(pose, C.c_double))
    return out, pose.reshape(4, 4)


def voxelize(pts, leaf):
    """pcl::VoxelGrid restated; pts (n,4) x,y,z,intensity -> (m,4) centroids in voxel-index order."""
    pts = np.ascontiguousarray(pts, np.float32)
    assert pts.shape[1] == 4
    out = np.empty_like(pts)
    m = lib().orc_voxelize(_p(pts, C.c_float), len(pts), C.c_float(leaf), _p(out, C.c_float))
    return pts.copy() if m < 0 else out[:m].copy()


def fetch_closest(pos, stamps, q, radius=35.0, tdiff=30.0):
    pos = np.ascontiguousarray(pos, np.float64)
    st = np.ascontiguousarray(stamps, np.float64)
    return lib().orc_fetch_closest(_p(pos, C.c_double), _p(st, C.c_double), int(q), C.c_double(radius), C.c_double(tdiff))


def set_src_and_dst_cloud(kf_clouds, kf_poses, src_idx, dst_idx, submap_range=5, voxel_res=0.3, enable_quatro=True,
                          enable_submap_matching=False, n_keyframes=None):
    """LoopClosure::setSrcAndDstCloud (fast_lio_sam_qn/src/loop_closure.cpp:58-108)."""
    nk = n_keyframes if n_keyframes is not None else len(kf_clouds)

    def merged(center):
        parts = [transform_pcd(kf_clouds[i], kf_poses[i]) for i in range(center - submap_range, center + submap_range + 1)
                 if 0 <= i < nk - 1]
        return np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)
    if enable_submap_matching:
        src, dst = merged(src_idx), merged(dst_idx)
    else:
        src = transform_pcd(kf_clouds[src_idx], kf_poses[src_idx])
        dst = transform_pcd(kf_clouds[dst_idx], kf_poses[dst_idx]) if enable_quatro else merged(dst_idx)
    return voxelize(src, voxel_res), voxelize(dst, voxel_res)


# ---------------------------------------------------------------------------------------------
# result consumption (SURVEY §8f rank 3)
def _pose_rpy_roundtrip(P):
    """poseEigToGtsamPose (fast_lio_sam_qn/include/utilities.hpp:67-75): tf getRPY, then gtsam Rot3::RzRyRx."""
    P = np.asarray(P, np.float64)
    m20 = P[2, 0]
    if abs(m20) >= 1.0:  # gimbal lock branch of tf's getEulerYPR
        yaw, roll = 0.0, np.arctan2(P[2, 1], P[2, 2])
        pitch = np.pi / 2 if m20 < 0 else -np.pi / 2
    else:
        pitch = -np.arcsin(m20)
        cp = np.cos(pitch)
        roll = np.arctan2(P[2, 1] / cp, P[2, 2] / cp)
        yaw = np.arctan2(P[1, 0] / cp, P[0, 0] / cp)
    cx, sx, cy, sy, cz, sz = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    return Rz @ Ry @ Rx, P[:3, 3].copy()


def loop_factor(T_between, pose_latest, pose_closest, score):
    """BetweenFactor measurement + variances of an accepted loop (fast_lio_sam_qn/src/fast_lio_sam_qn.cpp:220-231)."""
    R1, t1 = _pose_rpy_roundtrip(np.asarray(T_between, np.float64) @ np.asarray(pose_latest, np.float64))
    R2, t2 = _pose_rpy_roundtrip(pose_closest)
    M = np.eye(4)
    M[:3, :3] = R1.T @ R2
    M[:3, 3] = R1.T @ (t2 - t1)
    return M, np.full(6, float(score))
