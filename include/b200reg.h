/* b200reg.h -- C ABI of the H100-native loop-closure registration engine.
 *
 * This is the drop-in boundary for the ONE hot path of engcang/FAST-LIO-SAM-QN that
 * this repository replaces: the registration that FastLioSamQn::loopTimerFunc
 * (fast_lio_sam_qn/src/fast_lio_sam_qn.cpp:203-252) reaches through
 * LoopClosure::performLoopClosure (fast_lio_sam_qn/src/loop_closure.cpp:168-205), i.e.
 * everything behind nano_gicp::NanoGICP<PointType,PointType>
 * (third_party/nano_gicp/include/nano_gicp/nano_gicp.hpp:58-137) and quatro<PointType>
 * (third_party/Quatro/include/quatro/quatro_module.h:19-37).
 *
 * The reference has no FFI: both libraries are linked C++ templates.  The host-side
 * facade classes in fast-lio-sam-qn_b200/host/ keep those class surfaces and call the
 * functions below; INTEGRATION.md shows the binding.
 *
 * Conventions
 *   - every function returns 0 on success, a negative B200REG_E* code otherwise; nothing
 *     throws across this boundary;
 *   - all 4x4 matrices are ROW-MAJOR (Eigen is column-major: the facade transposes);
 *   - a context is bound to one CUDA device and one stream; use one context per host
 *     thread / per GPU rank (LoopClosure itself is single-instance and not re-entrant,
 *     fast_lio_sam_qn/src/fast_lio_sam_qn.cpp:81);
 *   - point buffers are (x, y, z [, ...]) fp32 records `stride_bytes` apart, so
 *     pcl::PointXYZI (32 B: x,y,z,1,intensity,pad) uploads without repacking;
 *   - host buffers passed to a call (pinned or pageable) have been consumed when the call returns; device buffers passed
 *     with on_device != 0 must stay valid until the context's stream has been synchronised or the call has returned a result;
 *   - b200reg_ctx_set_stream may only be called while the context is idle (everything it owns is ordered on ONE stream);
 *   - there is NO CPU fallback: if no CUDA device is present b200reg_ctx_create fails.
 */
#ifndef B200REG_H
#define B200REG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200REG_OK 0
#define B200REG_EINVAL (-1)   /* bad argument */
#define B200REG_ECUDA (-2)    /* CUDA runtime error (see b200reg_last_error) */
#define B200REG_ENODEV (-3)   /* no usable GPU */
#define B200REG_ESTATE (-4)   /* call order violated (e.g. align before covariances) */
#define B200REG_ENCCL (-5)    /* collective layer error */

typedef struct b200reg_ctx b200reg_ctx;
typedef struct b200reg_cloud b200reg_cloud;

/* Mirrors NanoGICPConfig (fast_lio_sam_qn/include/loop_closure.h:25-36) + the LsqRegistration
 * constructor defaults (third_party/nano_gicp/include/nano_gicp/impl/lsq_registration_impl.hpp:49-63). */
typedef struct b200reg_gicp_params {
  int32_t k_correspondences;     /* setCorrespondenceRandomness, loop_closure.cpp:10 (15); any k >= 1 */
  int32_t max_iterations;        /* setMaximumIterations, loop_closure.cpp:11 (32)          */
  double max_corr_dist;          /* setMaxCorrespondenceDistance, loop_closure.cpp:13 (52.5)*/
  double transformation_eps;     /* setTransformationEpsilon, loop_closure.cpp:14 (0.01)    */
  double rotation_eps;           /* lsq_registration_impl.hpp:53 (2e-3)                     */
  int32_t lm_max_iterations;     /* lsq_registration_impl.hpp:58 (10)                       */
  int32_t regularization;        /* RegularizationMethod (gicp/gicp_settings.hpp:47): 0 NONE, 1 MIN_EIG,
                                    2 NORMALIZED_MIN_EIG, 3 PLANE (default, nano_gicp_impl.hpp:61), 4 FROBENIUS */
  double lm_init_lambda_factor;  /* lsq_registration_impl.hpp:59 (1e-9)                     */
  double icp_score_thr;          /* validity gate, loop_closure.cpp:129 (config.yaml:21: 1.5) */
} b200reg_gicp_params;

/* RegistrationOutput (fast_lio_sam_qn/include/loop_closure.h:64-70) plus solver telemetry. */
typedef struct b200reg_result {
  double T[16];        /* final SE(3), fp64, row-major: maps src onto dst                      */
  float Tf[16];        /* x0.cast<float>() -- what getFinalTransformation() returns            */
  double pose_between[16]; /* RegistrationOutput::pose_between_eig_ exactly as the reference leaves it
                          (loop_closure.cpp:129-134, 156): icpAlignment: Tf.cast<double>() when valid, Identity otherwise;
                          coarseToFineAlignment: (valid fine stage ? Tf_fine : Identity) * T_quatro, or the coarse
                          stage's own output when Quatro itself is invalid; Identity for the dummy output        */
  double final_hessian[36]; /* LsqRegistration::getFinalHessian() (lsq_registration.hpp:88): H of the last linearize,
                          6x6 row-major (symmetric); Identity before any (lsq_registration_impl.hpp:62)            */
  double fitness;      /* getFitnessScore(): mean 1-NN d^2 over ALL source points              */
  int32_t converged;   /* hasConverged()                                                       */
  int32_t valid;       /* converged && fitness < icp_score_thr (loop_closure.cpp:129)          */
  int32_t iterations;  /* nr_iterations_ (index of the last outer iteration)                   */
  int32_t n_linearize; /* number of linearize() passes (= 1-NN passes)                         */
  int32_t n_error;     /* number of compute_error() passes                                     */
  int32_t lm_failed;   /* "lm not converged!!" (lsq_registration_impl.hpp:105-108)             */
  int32_t status;      /* 0 ok; <0 error for this pair                                         */
  int32_t tag;         /* caller-defined, set to 0 by the engine and carried through b200reg_allgather_results
                          (e.g. the global pair index of a sharded batch)                                      */
} b200reg_result;

/* Mirrors QuatroConfig (fast_lio_sam_qn/include/loop_closure.h:38-50) and the quatro<T> constructor arguments
 * (third_party/Quatro/include/quatro/quatro_module.h:30-32), with the EFFECTIVE deployment values as defaults
 * (SURVEY.md App. A.1: normal radius 0.9, FPFH radius 1.5, max correspondences 200 because of the rosparam typo). */
typedef struct b200reg_quatro_params {
  double fpfh_normal_radius;   /* fpfh_normal_radi (0.9)                                              */
  double fpfh_radius;          /* fpfh_radi (1.5)                                                     */
  double noise_bound;          /* 0.3                                                                 */
  double rot_gnc_factor;       /* 1.4                                                                 */
  double rot_cost_thr;         /* 1e-4                                                                */
  int32_t rot_max_iter;        /* 50                                                                  */
  int32_t max_corres;          /* num_max_corres (200); optimizedMatching: 1..8189 (B200REG_ADV_CORR_CAPACITY - 3) */
  double distance_threshold;   /* FEATURE-space gate of optimizedMatching (matcher.cc:422/444) (35)   */
  double tuple_scale;          /* 0.95 (quatro_module.cc:61)                                          */
  uint64_t seed;               /* replaces srand(time(NULL)) (matcher.cc:465) by a counter-based RNG  */
  int32_t estimate_scale;      /* must be 0 (QN/config: estimating_scale false)                       */
  int32_t use_optimized_matching; /* 1 (config.yaml:32): optimizedMatching; 0: advancedMatching       */
} b200reg_quatro_params;

/* Telemetry of one quatro<T>::align call. */
typedef struct b200reg_quatro_info {
  double T[16];          /* out_tf_ (row-major); Identity when !valid                                  */
  int32_t valid;         /* if_valid (quatro_module.cc:63-72)                                          */
  int32_t n_mutual;      /* correspondences after the mutual check                                     */
  int32_t n_corr;        /* after the tuple test (<= max_corres + 3)                                   */
  int32_t clique_size;   /* max-clique inliers                                                         */
  int32_t gnc_iterations;
  int32_t reserved;
} b200reg_quatro_info;

void b200reg_default_gicp_params(b200reg_gicp_params* p);
void b200reg_default_quatro_params(b200reg_quatro_params* p);
const char* b200reg_last_error(void);                /* message of the calling thread's last failure               */
void b200reg_set_last_error(const char* message);  /* used by the batch driver to hand a worker's message over     */
const char* b200reg_version(void);
/* One Levenberg-Marquardt trial of the Nano-GICP solve: one pass through the body of step_lm's
 * `for (i < lm_max_iterations_)` loop (lsq_registration_impl.hpp:170-205), recorded when tracing is enabled
 * (b200reg_ctx_set_lm_trace).  LsqRegistration::setDebugPrint prints one table row per such trial (:183-189). */
typedef struct b200reg_lm_trial {
  int32_t outer;       /* outer iteration: nr_iterations_ during the trial                                          */
  int32_t trial;       /* step_lm's i: the first column of the reference's table                                    */
  int32_t decision;    /* 1 accepted (x0 <- xi); 0 rejected (lambda <- nu lambda); 2 rejected but is_converged(delta)
                          held, so the solve returns without moving x0 (:191-194); 3 rejected on the last allowed trial,
                          "lm not converged!!" (:105-108)                                                              */
  int32_t reserved;    /* 0                                                                                          */
  double y0;           /* error of the linearization this trial belongs to                                           */
  double yi;           /* compute_error at the trial pose                                                            */
  double rho;          /* (y0 - yi) / d.(lambda d - b)                                                               */
  double lambda;       /* the lambda the trial was solved with (the value the reference prints)                      */
  double nu;           /* the nu in force during the trial                                                           */
  double d[6];         /* the step (rotation, translation): |delta| = ||d||                                          */
  double T[12];        /* x0 after the decision, row-major 3 x 4                                                     */
} b200reg_lm_trial;

/* One input of b200reg_lm_step_tap: the LM controller's state at one point of step_lm. */
typedef struct b200reg_lm_case {
  double R[9], t[3];   /* x0, row-major                                                                           */
  double H[36];        /* symmetric 6 x 6, row-major (mode 0 reads the upper triangle, as linearize hands it over)  */
  double b[6];
  double y0;           /* error at x0                                                                              */
  double yi;           /* mode 1: compute_error at the trial pose                                                  */
  double lambda;       /* lm_lambda_ in force; < 0 = not yet set (mode 0 then applies the init rule)                */
  double nu;           /* mode 1: the nu in force (mode 0 resets it to 2)                                           */
  b200reg_gicp_params params;  /* the controller reads max_iterations, lm_max_iterations, transformation_eps,
                                  rotation_eps and lm_init_lambda_factor                                            */
  int32_t outer_it;    /* nr_iterations_                                                                           */
  int32_t inner_it;    /* mode 1: step_lm's i of this trial                                                        */
  int32_t mode;        /* 0: the start of step_lm after linearize (H, b, y0) and its first trial's step;
                          1: one trial: the step from (H, b, lambda), then the decision on yi                        */
  int32_t reserved;
} b200reg_lm_case;

/* One output of b200reg_lm_step_tap. */
typedef struct b200reg_lm_step {
  double d[6];         /* the trial's step (rotation, translation), from the device's solve of (H + lambda I) d = -b  */
  double dR[9];        /* so3_exp(d[0..2]), row-major                                                              */
  double dt[3];
  double Rt[9], tt[3]; /* the trial pose delta * x0                                                                */
  double R[9], t[3];   /* x0 after the decision                                                                    */
  double lambda, nu;   /* after the decision                                                                       */
  b200reg_lm_trial record;  /* mode 1: the trial's trace record (rho, decision, ...)                              */
  int32_t phase;       /* 0 linearize next, 1 a trial is prepared, 2 the solve is finished                         */
  int32_t converged;
  int32_t lm_failed;
  int32_t has_trial;   /* a trial was prepared (d .. tt hold it)                                                    */
  int32_t outer_it, inner_it;  /* after the decision                                                               */
} b200reg_lm_step;

/* sizeof() of the ABI structs as compiled into the library, so that a binding (ctypes, cgo, JNI ...) can check its own
 * layout at load time: 0 gicp_params, 1 result, 2 quatro_params, 3 quatro_info, 4 loop_config, 5 loop_factor,
 * 6 lm_trial, 7 lm_case, 8 lm_step.  0 = unknown. */
size_t b200reg_struct_size(int which);

/* ---- context ---------------------------------------------------------------------- */
int b200reg_ctx_create(int device, b200reg_ctx** out);
int b200reg_ctx_destroy(b200reg_ctx* ctx);
/* Use an externally owned CUDA stream (cudaStream_t passed as void*); NULL = the context's own. */
int b200reg_ctx_set_stream(b200reg_ctx* ctx, void* cuda_stream);
int b200reg_ctx_synchronize(b200reg_ctx* ctx);
/* Number of kernels this context has launched so far (bench.py reports it as gpu_launches). */
int64_t b200reg_ctx_launch_count(const b200reg_ctx* ctx);

/* Per-kernel-family timing with CUDA events recorded on the launching stream (bench.py roofline).
 * Families: 0 index_build, 1 knn_covariance, 2 gicp_step (the LM loop as ONE graph launch), 3 misc, 4 fpfh,
 * 5 quatro_match_solve, 6 gicp_search, 7 gicp_accum, 8 gicp_control.  While profiling is enabled the LM loop is not run as
 * a graph: its three kernels are launched one by one (host-polled) so that each gets its own events -- families 6-8 fill,
 * family 2 stays empty.  algo_bytes follows SURVEY.md §8(d).                                                         */
int b200reg_ctx_set_profiling(b200reg_ctx* ctx, int enable);
int b200reg_ctx_reset_profile(b200reg_ctx* ctx);
int b200reg_ctx_get_profile(b200reg_ctx* ctx, int family, const char** name, double* ms, double* algo_bytes,
                            int64_t* launches);

/* LM trace (LsqRegistration::setDebugPrint, lsq_registration_impl.hpp:95-99, 183-189).  Off by default.  While enabled,
 * every call that runs the LM solve (b200reg_gicp_align, b200reg_icp_alignment, b200reg_loop_closure,
 * b200reg_perform_loop_closure) records each trial of each pair.  The device buffer holds count x max_iterations x
 * max(lm_max_iterations, 1) records (no pair can have more, nothing is truncated) and lives for the call only; if it cannot
 * be allocated the call returns B200REG_ECUDA with the bytes in the message.  Tracing changes no result and no launch.
 * Each such call discards the stored trace on entry and stores its own only if it succeeds with tracing on; a refused or
 * failed call, or one with tracing off, leaves none.  With tracing off nothing is recorded or allocated.               */
int b200reg_ctx_set_lm_trace(b200reg_ctx* ctx, int enable);
/* The trace of the context's most recent call that ran the LM solve, as CSR over that call's pairs (the CALLER's pair
 * indices; a pair whose fine stage did not run -- invalid Quatro, no loop candidate -- has no records): the trials of pair
 * i are trials_out[offsets_out[i] .. offsets_out[i + 1]), in execution order; offsets_out has count + 1 entries.  If the
 * records exceed `capacity` the call fills offsets_out, writes nothing else and returns B200REG_ESTATE.  offsets_out ==
 * NULL: returns that call's pair count (>= 0) and writes nothing.  Before any traced solve, and after a call that ran
 * untraced, was refused or failed: B200REG_ESTATE.                                                                      */
int b200reg_lm_trace(b200reg_ctx* ctx, int64_t* offsets_out, size_t capacity, b200reg_lm_trial* trials_out);

/* Loop clouds: the four clouds loopTimerFunc publishes after each loop attempt (fast_lio_sam_qn.cpp:245-248), as the batched
 * calls b200reg_icp_alignment, b200reg_loop_closure and b200reg_perform_loop_closure produce them.  Every point is four
 * floats (x, y, z, intensity), pcl::PointXYZI without its padding; intensity is carried through every step.
 *   SOURCE  LoopClosure::getSourceCloud (loop_closure.cpp:185): the assembled, voxelised source -- b200reg_cloud_points of it,
 *           in voxel-index order, intensity the voxel mean (fp32 running sums in ascending point order; the unfiltered
 *           merged cloud when the voxel grid's int32 guard trips, as PCL returns it).  b200reg_perform_loop_closure only.
 *   TARGET  getTargetCloud (:186): the same for the target.  b200reg_perform_loop_closure only.
 *   COARSE  getCoarseAlignedCloud (:152): transformPcd(source, quatro_out[i].T) -- double math cast to float, the source's
 *           order -- for pairs whose Quatro stage is valid; empty otherwise, as the reference clears it (:142).
 *   FINAL   getFinalAlignedCloud (:124; lsq_registration_impl.hpp:114): NanoGICP::align's output cloud, the fine source
 *           (COARSE in Quatro mode, else the source) through the fine stage's fp32 transform, byte-equal to
 *           b200reg_transform_cloud; present whenever the fine stage ran, converged or not.  Where it did not run the row is
 *           empty (the reference would keep the previous tick's cloud; a batch has no previous tick).
 * The raw-buffer calls take the intensity from their records as b200reg_keyframes_add does: float 3 for strides of 16 to
 * 31 bytes, float 4 from 32 bytes (pcl::PointXYZI), 0 for 12-byte records.                                             */
#define B200REG_CLOUD_SOURCE 1
#define B200REG_CLOUD_TARGET 2
#define B200REG_CLOUD_COARSE 4
#define B200REG_CLOUD_FINAL 8
/* Capture the kinds in `mask` (an OR of B200REG_CLOUD_*; 0, the default, turns capture off) in the following calls of the
 * three entry points above; no other entry point touches the stored clouds.  Each such call discards the stored clouds
 * on entry and stores its own only if it succeeds with capture on; a refused or failed call, or one with capture off,
 * leaves none.  Capture changes no result, trace or solve.  Its device slab (16 bytes per point per kind: 512 pairs x
 * 100k points x 4 kinds is about 3.3 GB) lives for the call only and is sized before Quatro for every row that can be
 * present; if it cannot be allocated the call returns B200REG_ECUDA with the bytes in the message.  With capture off
 * nothing is allocated or launched.                                                                                   */
int b200reg_ctx_set_loop_clouds(b200reg_ctx* ctx, int mask);
/* The clouds of one kind from the context's most recent capturing call, as CSR over that call's pairs (the CALLER's pair
 * order): pair i's points are xyzi_out[4 * offsets_out[i] .. 4 * offsets_out[i + 1]), in the order above; offsets_out has
 * count + 1 entries; pairs without such a cloud (no loop candidate, invalid Quatro ...) have empty rows.  If the points
 * exceed `capacity` the call fills offsets_out, writes nothing else and returns B200REG_ESTATE.  offsets_out == NULL:
 * returns that call's pair count (>= 0) and writes nothing.  A kind that call did not capture, and after a call that
 * ran uncaptured, was refused or failed: B200REG_ESTATE.  A kind that is not one B200REG_CLOUD_* bit: B200REG_EINVAL. */
int b200reg_loop_clouds(b200reg_ctx* ctx, int kind, int64_t* offsets_out, size_t capacity, float* xyzi_out);

/* ---- clouds: replaces KdTreeFLANN::setInputCloud / buildIndex
 *      (third_party/nano_gicp/include/nano_gicp/nanoflann.hpp:131-138) ----------------- */
/* Upload `count` clouds (host or device pointers) and build their spatial indices in one
 * batched pass.  on_device != 0: the xyz pointers are device pointers (no H2D copy).      */
int b200reg_clouds_create(b200reg_ctx* ctx, int count, const float* const* xyz, const size_t* n,
                          size_t stride_bytes, int on_device, b200reg_cloud** out);
int b200reg_cloud_destroy(b200reg_ctx* ctx, b200reg_cloud* cloud);
size_t b200reg_cloud_size(const b200reg_cloud* cloud);

/* NanoGICP::calculateSourceCovariances / calculateTargetCovariances
 * (third_party/nano_gicp/include/nano_gicp/impl/nano_gicp_impl.hpp:151-159, 298-357), batched.  k in 1..32 here;
 * b200reg_clouds_covariances_ex takes any k >= 1. */
int b200reg_clouds_covariances(b200reg_ctx* ctx, int count, b200reg_cloud* const* clouds, int k);
/* NanoGICP::setSourceCovariances / setTargetCovariances (nano_gicp.hpp:91-93, nano_gicp_impl.hpp:142-150): the caller's
 * per-point covariances (n x 9 doubles: the row-major 3x3 block of each Matrix4d, ORIGINAL point order) replace the
 * computed ones; align() then does not recompute them (nano_gicp_impl.hpp:162-167) until the input cloud changes.   */
int b200reg_set_covariances(b200reg_ctx* ctx, b200reg_cloud* cloud, const double* cov9, size_t n);
/* Same with an explicit RegularizationMethod (setRegularizationMethod, nano_gicp.hpp:84); the plain call uses PLANE.
 * Any k >= 1 (setCorrespondenceRandomness): each point's k nearest points of its own cloud, itself included; all of the
 * cloud when k >= n, the mean and covariance still divided by k.  k <= 32 runs one thread per point; k > 32 one warp per
 * point, O(k) per point, with the moments summed in neighbour order ((d2, original index), fp64, no FMA).  Its neighbour
 * lists live in shared memory up to 256 entries and beyond that in device scratch of one list per resident warp, at most
 * max(128 MiB, 32 * min(k, largest cloud) bytes) per call whatever the cloud sizes.                                  */
int b200reg_clouds_covariances_ex(b200reg_ctx* ctx, int count, b200reg_cloud* const* clouds, int k, int method);

/* ---- registration ----------------------------------------------------------------- */
/* pcl::Registration::align + getFitnessScore + hasConverged + getFinalTransformation for
 * `count` (src, tgt) pairs at once (call sites fast_lio_sam_qn/src/loop_closure.cpp:124-133).
 * guess16: count x 16 doubles row-major, or NULL for identity (the reference always uses identity).
 * Covariances are computed on demand if a cloud has none (nano_gicp_impl.hpp:162-167).       */
int b200reg_gicp_align(b200reg_ctx* ctx, int count, b200reg_cloud* const* src, b200reg_cloud* const* tgt,
                       const double* guess16, const b200reg_gicp_params* params, b200reg_result* out);

/* LoopClosure::icpAlignment (loop_closure.cpp:110-136) in one call, raw buffers in, results out:
 * index build x2, covariances x2, align, fitness, validity gate -- for `count` pairs.          */
int b200reg_icp_alignment(b200reg_ctx* ctx, int count, const float* const* src_xyz, const size_t* src_n,
                          const float* const* tgt_xyz, const size_t* tgt_n, size_t stride_bytes, int on_device,
                          const b200reg_gicp_params* params, b200reg_result* out);

/* ---- Quatro (global registration) --------------------------------------------------------- */
/* teaser::FPFHEstimation::computeFPFHFeatures (third_party/Quatro/src/fpfh.cc:14-42) for `count` clouds:
 * normals (radius search, viewpoint (0,0,0)) -> SPFH -> FPFH, kept on the device with the cloud.     */
int b200reg_clouds_fpfh(b200reg_ctx* ctx, int count, b200reg_cloud* const* clouds, double normal_radius,
                        double fpfh_radius);
/* quatro<PointType>::align (third_party/Quatro/src/quatro_module.cc:48-79) for `count` pairs: FPFH on demand,
 * optimizedMatching (matcher.cc:358-561) or, with use_optimized_matching = 0, advancedMatching (matcher.cc:118-356:
 * ungated forward / reverse 1-NN, cross check, three-edge tuple test, sort + unique), then the TEASER++ QUATRO solve.
 * corr_out (optional): count x 2*CAP ints, the (src, dst) ORIGINAL indices of the final correspondences of each
 * pair, CAP = B200REG_CORR_CAPACITY (optimized) or B200REG_ADV_CORR_CAPACITY (advanced).  advancedMatching sets of any
 * size (below 2^20) are solved; a set larger than B200REG_ADV_CORR_CAPACITY does not fit corr_out, so with a non-NULL
 * corr_out such a set fails the call with B200REG_ESTATE (nothing is truncated silently), and with corr_out NULL the
 * call solves it.  optimizedMatching keeps at most max_corres + 3 correspondences (up to 8192); the same rule holds at
 * its CAP: with max_corres > 509 a set of more than B200REG_CORR_CAPACITY fails a call with a non-NULL corr_out with
 * B200REG_ESTATE, naming the pair and the count.  b200reg_quatro_align_ex returns the correspondences of any size.
 * Pairs with at most B200REG_ADV_CORR_CAPACITY correspondences are solved together; larger sets are solved one pair at
 * a time in one device workspace sized for the largest (about n^2 / 4 bytes for n correspondences: 1 GB at n = 65536).
 * If that workspace cannot be allocated the call returns B200REG_ECUDA with the bytes needed in the message.     */
#define B200REG_CORR_CAPACITY 512
#define B200REG_ADV_CORR_CAPACITY 8192
int b200reg_quatro_align(b200reg_ctx* ctx, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst,
                         const b200reg_quatro_params* params, b200reg_quatro_info* out, int32_t* corr_out);
/* Same solve; the final correspondences come back as CSR, as b200reg_radius_search returns neighbours: those of pair i
 * are the (src, dst) pairs corr_out[2 * offsets_out[i] ..  2 * offsets_out[i + 1]), offsets_out has count + 1 entries
 * and must not be NULL.  If the total exceeds `capacity` (in pairs) the call fills offsets_out, writes nothing else and
 * returns B200REG_ESTATE.  corr_out == NULL: offsets and `out` only.                                              */
int b200reg_quatro_align_ex(b200reg_ctx* ctx, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst,
                            const b200reg_quatro_params* params, b200reg_quatro_info* out, int64_t* offsets_out,
                            size_t capacity, int32_t* corr_out);
/* LoopClosure::coarseToFineAlignment (fast_lio_sam_qn/src/loop_closure.cpp:138-159) for `count` pairs from raw
 * buffers: Quatro -> transformPcd(src, T_quatro) -> icpAlignment -> T = T_gicp * T_quatro.
 * out[i].T is the composed transform; quatro_out (optional) receives the coarse stage.                   */
int b200reg_loop_closure(b200reg_ctx* ctx, int count, const float* const* src_xyz, const size_t* src_n,
                         const float* const* tgt_xyz, const size_t* tgt_n, size_t stride_bytes, int on_device,
                         const b200reg_quatro_params* qparams, const b200reg_gicp_params* gparams,
                         b200reg_result* out, b200reg_quatro_info* quatro_out);

/* Quatro matches: the correspondences the coarse stage solved (Matcher::calculateCorrespondences, quatro_module.cc:60-61)
 * and which of them are in the solve's max clique (RobustRegistrationSolver::getInlierMaxClique, :69-76), per pair.
 *   Which calls record.  Recording is off by default.  While it is on, every call that reaches the Quatro stage records:
 *     b200reg_quatro_align, b200reg_quatro_align_ex, b200reg_loop_closure, b200reg_perform_loop_closure, and the batch
 *     jobs of b200reg_batch_submit_loop_closure and b200reg_batch_submit_perform_loop_closure (b200reg_batch_set_quatro_matches).
 *     Each such call replaces the stored matches.  Such a call with recording off discards them.  b200reg_quatro_solve_tap
 *     and the calls without a Quatro stage leave them untouched.
 *   Rows.  Rows follow the caller's pair or query order.  Pair i's matches are the solver's input set, in the order
 *     b200reg_quatro_align_ex returns it.  A query with no candidate, b200reg_perform_loop_closure with enable_quatro = 0,
 *     and a pair whose matcher kept nothing have empty rows.
 *   Inliers.  inlier_out is 1 for the members of the pair's max clique and 0 otherwise.  The number of 1s of a pair equals
 *     its b200reg_quatro_info::clique_size, also for an invalid solve with a clique of 0 or 1.
 *   Indices and points.  The indices are rows of the clouds Quatro matched, in their original order.  For the raw-buffer
 *     calls those are the caller's buffers.  For b200reg_perform_loop_closure they are the assembled, voxelised clouds, whose
 *     rows are the rows of its SOURCE and TARGET loop clouds.  The xyz values are those rows' floats, bit for bit.
 *   Cost.  With recording off nothing is allocated or launched.  With it on, a call allocates 36 bytes per match and one
 *     clique row per pair for its own duration, and adds one kernel launch.  Results, Quatro records, LM traces and loop
 *     clouds stay byte-identical.  If the slab cannot be allocated the call returns B200REG_ECUDA with the bytes needed.  */
int b200reg_ctx_set_quatro_matches(b200reg_ctx* ctx, int enable);
/* The matches of the context's most recent recording call, as CSR over that call's pairs: pair i's matches are rows
 * offsets_out[i] .. offsets_out[i + 1]), offsets_out has count + 1 entries.  Row r is corr_out[2r] (src) and
 * corr_out[2r + 1] (dst), inlier_out[r], src_xyz_out[3r .. 3r + 3) and dst_xyz_out[3r .. 3r + 3).  Any of the four output
 * pointers may be NULL.  If the matches exceed `capacity` (in rows) the call fills offsets_out, writes nothing else and
 * returns B200REG_ESTATE.  offsets_out == NULL: returns that call's pair count (>= 0) and writes nothing.  Before any
 * recording call, after a call that did not record, and after a call that failed: B200REG_ESTATE.                      */
int b200reg_quatro_matches(b200reg_ctx* ctx, int64_t* offsets_out, size_t capacity, int32_t* corr_out, int32_t* inlier_out,
                           float* src_xyz_out, float* dst_xyz_out);

/* Residuals: what the fitness pass of the fine stage (getFitnessScore, b200reg_result::fitness) found per source point
 * at the final pose, per pair: the nearest target point and its squared distance.
 *   Which calls record.  Recording is off by default.  While it is on, every call that runs the fine stage records:
 *     b200reg_gicp_align, b200reg_icp_alignment, b200reg_loop_closure, b200reg_perform_loop_closure, and the batch jobs of
 *     all three kinds (b200reg_batch_set_residuals).  Each such call replaces the stored rows.  Such a call with recording
 *     off discards them.  b200reg_quatro_align, b200reg_quatro_align_ex and the taps leave them untouched.
 *   Rows.  Pairs follow the caller's pair or query order; pair i has one row per point of its source cloud, in the cloud's
 *     ORIGINAL point order.  Row r is nn_out[r], the original index of the nearest target point after the final fp32
 *     transformation (x*c0 + (y*c1 + (z*c2 + c3)), ties to the lower index; -1 only if no target point is a candidate), and
 *     d2_out[r], its fp32 squared distance: bit for bit the value the fitness pass sums, so the mean of a pair's d2 is its
 *     fitness up to that pass's fixed summation order.  A pair whose fine stage did not run has an empty row: a query with
 *     no candidate, and a pair whose Quatro solve is invalid.
 *   Indices.  For the raw-buffer calls the rows and nn are rows of the caller's buffers.  For b200reg_perform_loop_closure
 *     the rows are rows of its SOURCE loop cloud (the same rows as COARSE in Quatro mode) and nn indexes its TARGET loop
 *     cloud.  For b200reg_gicp_align they are rows of the cloud handles.
 *   Cost.  With recording off nothing is allocated or launched.  With it on, a call allocates 8 bytes per source point of
 *     every pair that can run the fine stage, before its first stage, for its own duration, and adds one kernel launch per
 *     fine stage.  Results, LM traces, loop clouds and Quatro matches stay byte-identical.  If the rows cannot be allocated
 *     the call returns B200REG_ECUDA with the bytes needed.  */
int b200reg_ctx_set_residuals(b200reg_ctx* ctx, int enable);
/* The residuals of the context's most recent recording call, as CSR over that call's pairs: pair i's rows are
 * offsets_out[i] .. offsets_out[i + 1]), offsets_out has count + 1 entries.  Either output pointer may be NULL.  If the
 * rows exceed `capacity` the call fills offsets_out, writes nothing else and returns B200REG_ESTATE.  offsets_out == NULL:
 * returns that call's pair count (>= 0) and writes nothing.  Before any recording call, after a call that did not record,
 * and after a call that failed: B200REG_ESTATE.                                                                          */
int b200reg_residuals(b200reg_ctx* ctx, int64_t* offsets_out, size_t capacity, int32_t* nn_out, float* d2_out);

/* ---- "next" rows (SURVEY.md §8f): device-resident keyframes, candidate search, cloud assembly ---------- */
typedef struct b200reg_keyframes b200reg_keyframes;

/* Mirrors LoopClosureConfig (fast_lio_sam_qn/include/loop_closure.h:52-62) with the EFFECTIVE deployment values
 * (SURVEY.md §5: num_submap_keyframes 5 because of the rosparam typo). */
typedef struct b200reg_loop_config {
  int32_t enable_quatro;            /* config.yaml:29 (1)                                   */
  int32_t enable_submap_matching;   /* config.yaml:9 (0)                                    */
  int32_t num_submap_keyframes;     /* submap_range (5)                                     */
  int32_t reserved;
  double voxel_res;                 /* config.yaml:16 (0.3)                                 */
  double loop_detection_radius;     /* config.yaml:13 (35.0)                                */
  double loop_detection_timediff_threshold; /* config.yaml:14 (30.0)                        */
  b200reg_gicp_params gicp;
  b200reg_quatro_params quatro;
} b200reg_loop_config;
void b200reg_default_loop_config(b200reg_loop_config* cfg);

int b200reg_keyframes_create(b200reg_ctx* ctx, b200reg_keyframes** out);
int b200reg_keyframes_destroy(b200reg_ctx* ctx, b200reg_keyframes* kf);
/* Keyframe clouds are kept in device slabs of their own (128 MB unless reserved), apart from the context's scratch pool.
 * A node that knows roughly how many points its map will hold reserves them once at start (std::vector::reserve for
 * keyframes_, fast_lio_sam_qn.h:63): no keyframe added afterwards allocates until the reservation is used up.        */
int b200reg_keyframes_reserve(b200reg_ctx* ctx, b200reg_keyframes* kf, size_t n_points);
/* PosePcd (fast_lio_sam_qn/include/pose_pcd.hpp:7-43): cloud in the LiDAR frame as fp32 records `stride_bytes` apart (host
 * memory): packed (x, y, z, intensity) for strides below 32 bytes, the pcl::PointXYZI layout (x, y, z, 1, intensity, pad...)
 * from 32 bytes on; its corrected pose (row-major 4x4) and timestamp.  Returns the index.                          */
int b200reg_keyframes_add(b200reg_ctx* ctx, b200reg_keyframes* kf, const float* xyzi, size_t n, size_t stride_bytes,
                          const double* pose16, double timestamp);
/* The PosePcd constructor itself (pose_pcd.hpp:21-43) as a device step: the scan arrives in the WORLD frame with the odometry
 * pose as position + quaternion (x, y, z, w; nav_msgs::Odometry); pose_eig_ = [tf::Matrix3x3(q) | p], pose_corrected_eig_ =
 * pose_eig_, and the stored cloud is transformPcd(scan, pose_eig_.inverse()) (LiDAR frame).  Returns the index.        */
int b200reg_keyframes_add_world(b200reg_ctx* ctx, b200reg_keyframes* kf, const float* xyzi_world, size_t n, size_t stride_bytes,
                                const double* position3, const double* quat_xyzw, double timestamp);
/* Read a keyframe back: its LiDAR-frame cloud (n x 4 floats: x, y, z, intensity; NULL to skip), corrected pose (16 doubles,
 * row-major; NULL to skip) and timestamp (NULL to skip) -- what the reference saves per keyframe (fast_lio_sam_qn.cpp:344-376). */
int b200reg_keyframes_get(b200reg_ctx* ctx, const b200reg_keyframes* kf, int idx, float* xyzi_out, double* pose16_out,
                          double* timestamp_out);
size_t b200reg_keyframes_cloud_size(const b200reg_keyframes* kf, int idx);
/* pose_corrected_eig_ rewrite after an accepted loop (fast_lio_sam_qn/src/fast_lio_sam_qn.cpp:180-188).     */
int b200reg_keyframes_set_pose(b200reg_ctx* ctx, b200reg_keyframes* kf, int idx, const double* pose16);
int b200reg_keyframes_size(const b200reg_keyframes* kf);
/* LoopClosure::fetchClosestKeyframeIdx (loop_closure.cpp:34-56) for `count` query keyframes at once; each query
 * is treated as the latest keyframe at its time, so its candidates are the indices below it. -1 = none.       */
int b200reg_fetch_closest_keyframes(b200reg_ctx* ctx, b200reg_keyframes* kf, int count, const int32_t* query_idx,
                                    double radius, double timediff_threshold, int32_t* closest_out);
/* LoopClosure::setSrcAndDstCloud (loop_closure.cpp:58-108) for `count` (src, dst) keyframe index pairs:
 * transformPcd by the corrected poses, +-submap merge, pcl::VoxelGrid at voxel_res; the resulting clouds are
 * indexed and stay on the device.  n_keyframes = size of the keyframe vector at the time (0 = current size).  */
int b200reg_assemble_clouds(b200reg_ctx* ctx, b200reg_keyframes* kf, int count, const int32_t* src_idx,
                            const int32_t* dst_idx, const b200reg_loop_config* cfg, int n_keyframes,
                            b200reg_cloud** src_out, b200reg_cloud** dst_out);
/* Points of a cloud in their ORIGINAL order as (x, y, z) (debug tap for the assembled / voxelised clouds).    */
/* Same with the size of the keyframe vector given PER PAIR (n_keyframes[i] = latest keyframe index + 1 at the tick the
 * pair was formed): a batch that replays several loopTimerFunc ticks sees, for each query, exactly the sub-map bounds
 * `i < keyframes.size() - 1` the reference evaluated at that tick (loop_closure.cpp:72,79,100).                      */
int b200reg_assemble_clouds_at(b200reg_ctx* ctx, b200reg_keyframes* kf, int count, const int32_t* src_idx,
                               const int32_t* dst_idx, const b200reg_loop_config* cfg, const int32_t* n_keyframes,
                               b200reg_cloud** src_out, b200reg_cloud** dst_out);
int b200reg_cloud_points(b200reg_ctx* ctx, const b200reg_cloud* cloud, float* xyz_out);
/* LoopClosure::performLoopClosure (loop_closure.cpp:168-205) for `count` query keyframes with given closest
 * indices (-1 = no candidate -> invalid dummy output): assemble, then coarse-to-fine (enable_quatro) or GICP only. */
int b200reg_perform_loop_closure(b200reg_ctx* ctx, b200reg_keyframes* kf, int count, const int32_t* query_idx,
                                 const int32_t* closest_idx, const b200reg_loop_config* cfg, b200reg_result* out,
                                 b200reg_quatro_info* quatro_out);

/* Result consumption (SURVEY.md §8f rank 3; fast_lio_sam_qn/src/fast_lio_sam_qn.cpp:220-237): the loop constraint the
 * reference hands to GTSAM for an accepted registration,
 *   BetweenFactor<Pose3>(latest.idx_, closest_idx, pose_from.between(pose_to), Diagonal::Variances(score x 6)),
 *   pose_from = poseEigToGtsamPose(pose_between_eig_ * latest.pose_corrected_eig_)   ("take care of the order", :224)
 *   pose_to   = poseEigToGtsamPose(closest.pose_corrected_eig_)
 * with poseEigToGtsamPose's roll/pitch/yaw round trip (utilities.hpp:67-75: tf getRPY, then Rot3::RzRyRx).  The pose
 * graph itself (GTSAM iSAM2) stays with the caller; corrected poses come back through b200reg_keyframes_set_pose.   */
typedef struct b200reg_loop_factor {
  int32_t from_idx;        /* key of the latest keyframe                                        */
  int32_t to_idx;          /* key of the matched keyframe                                       */
  int32_t valid;           /* RegistrationOutput::is_valid_; 0: the reference adds no factor    */
  int32_t reserved;
  double measurement[16];  /* pose_from.between(pose_to), row-major 4x4                         */
  double variances[6];     /* score in every slot                                               */
} b200reg_loop_factor;
/* Pure host arithmetic (no context, no GPU): one factor from explicit poses.                                        */
int b200reg_loop_factor_from_poses(const double* T_between16, const double* pose_latest16, const double* pose_closest16,
                                   double score, int valid, int from_idx, int to_idx, b200reg_loop_factor* out);
/* The factors of a batch of b200reg_perform_loop_closure results, poses taken from the keyframe store.              */
int b200reg_loop_factors(b200reg_ctx* ctx, const b200reg_keyframes* kf, int count, const int32_t* query_idx,
                         const int32_t* closest_idx, const b200reg_result* results, b200reg_loop_factor* out);

/* ---- batch driver (SURVEY.md §8(b)(2) "b200reg_batch"): `depth` engine contexts, each on its own host thread with its own
 *      streams and memory pool, take alternate jobs, so the PCIe upload and the host-side polling of one job hide behind
 *      the kernels of the others.  The reference registers ONE pair per timer tick (fast_lio_sam_qn.cpp:203-219); a
 *      batch of independent candidate pairs is this engine's unit of work.
 *      Jobs are submitted from ONE host thread; the pointer arrays are copied at submit time, the point buffers and the
 *      output arrays must stay valid until the job has been waited for. ------------------------------------------------ */
typedef struct b200reg_batch b200reg_batch;
int b200reg_batch_create(int device, int depth, b200reg_batch** out);
int b200reg_batch_destroy(b200reg_batch* b);
/* LoopClosure::icpAlignment (loop_closure.cpp:110-136) for `count` pairs; returns a ticket >= 0 or a B200REG_E* code. */
int64_t b200reg_batch_submit_icp(b200reg_batch* b, int count, const float* const* src_xyz, const size_t* src_n,
                                 const float* const* tgt_xyz, const size_t* tgt_n, size_t stride_bytes, int on_device,
                                 const b200reg_gicp_params* params, b200reg_result* out);
/* LoopClosure::coarseToFineAlignment (loop_closure.cpp:138-159) for `count` pairs. */
int64_t b200reg_batch_submit_loop_closure(b200reg_batch* b, int count, const float* const* src_xyz, const size_t* src_n,
                                          const float* const* tgt_xyz, const size_t* tgt_n, size_t stride_bytes,
                                          int on_device, const b200reg_quatro_params* qparams,
                                          const b200reg_gicp_params* gparams, b200reg_result* out,
                                          b200reg_quatro_info* quatro_out);
/* LoopClosure::performLoopClosure for `count` query keyframes of the device keyframe store, as a job of the batch driver:
 * loopTimerFunc off the caller's thread, its stages overlapping those of other jobs.  closest_idx NULL: the job runs
 * fetchClosestKeyframeIdx itself first, with cfg's loop_detection_radius and loop_detection_timediff_threshold.
 *   Same bytes: a job writes the same b200reg_result and b200reg_quatro_info records, byte for byte, as
 *     b200reg_perform_loop_closure on the same store state, queries and config, at every driver depth; a NULL closest_idx
 *     answers as b200reg_fetch_closest_keyframes followed by that call.
 *   Snapshot at submit: the job sees the store as it is when it is submitted -- the keyframe count, the corrected poses,
 *     the clouds.  Keyframes added and poses rewritten (b200reg_keyframes_set_pose) after the submit do not change its
 *     answer.  The uploads of earlier adds are ordered before the job's reads on the device (an event per add, waited
 *     for by the job's stream); the submitting thread does not block on them.
 *   Lifetime: b200reg_keyframes_destroy on a store that jobs still read returns B200REG_ESTATE and frees nothing; after
 *     their b200reg_batch_wait (or _wait_all) it behaves as before.
 *   Errors: refused at submit with B200REG_EINVAL, as b200reg_perform_loop_closure refuses them: count <= 0 (count = 0
 *     too), NULL query_idx / cfg / out, a query outside the store (every query when closest_idx is NULL, else every one
 *     with a candidate), a candidate above its query, num_submap_keyframes or voxel_res out of range, and a store on
 *     another device than the driver.  Everything else (Quatro and GICP parameter refusals, device failures) comes back
 *     from b200reg_batch_wait with its message.
 *   Threads: submits, keyframe adds and pose rewrites of a store that jobs read come from ONE host thread.
 *   Loop clouds and LM trace: as for the other two job kinds, b200reg_batch_set_loop_clouds / _set_lm_trace (below).  */
int64_t b200reg_batch_submit_perform_loop_closure(b200reg_batch* b, b200reg_keyframes* kf, int count,
                                                  const int32_t* query_idx, const int32_t* closest_idx,
                                                  const b200reg_loop_config* cfg, b200reg_result* out,
                                                  b200reg_quatro_info* quatro_out);
/* Blocks until the job is done; returns ITS status (the message is then in b200reg_last_error of the calling thread).
 * latency_ms (optional): submit -> completion on the host clock.  A ticket can be waited for once.               */
int b200reg_batch_wait(b200reg_batch* b, int64_t ticket, double* latency_ms);
int b200reg_batch_wait_all(b200reg_batch* b);
/* Loop clouds and LM trace of driver jobs, all three kinds: what b200reg_ctx_set_loop_clouds / b200reg_ctx_set_lm_trace
 * capture on a context, per job.
 *   Settings: the kinds to capture (an OR of B200REG_CLOUD_*) and the tracing flag, both off by default, set from the
 *     submitting thread.  A job copies them at submit, as it copies the store's state, and applies them to its worker's
 *     context for its own run; changing them later does not affect it.
 *   Same bytes: a job's clouds of each kind and its trace equal, byte for byte, what b200reg_loop_clouds / b200reg_lm_trace
 *     return on a context after the synchronous call with the same inputs, mask and tracing -- at every driver depth,
 *     empty rows included (e.g. SOURCE / TARGET of an icpAlignment job), rows in the caller's pair or query order.  A
 *     b200reg_batch_submit_perform_loop_closure job with closest_idx NULL compares with b200reg_fetch_closest_keyframes
 *     followed by b200reg_perform_loop_closure.  Capture changes no result or Quatro record.
 *   Off costs nothing: a job with both settings off allocates nothing more, launches nothing more and keeps nothing.
 *   No carry-over: a worker runs jobs of different settings back to back; each job sees its own outputs only, moved out of
 *     the worker's context (no copy) when it ends.  No new kernel: the same capture and trace run on the worker.
 *   Lifetime: the outputs of a job that captured are readable once b200reg_batch_wait (or _wait_all) has returned for its
 *     ticket, until b200reg_batch_release(ticket) or b200reg_batch_destroy.  Errors inside a job (e.g. a trace or capture
 *     buffer that cannot be allocated) come back from b200reg_batch_wait with their message; such a job keeps nothing.
 *   Getters: the rules of b200reg_loop_clouds / b200reg_lm_trace (CSR over the job's pairs, offsets_out NULL returns the
 *     pair count, a total above `capacity` fills offsets_out only and returns B200REG_ESTATE; a kind that is not one
 *     B200REG_CLOUD_* bit: B200REG_EINVAL).  A ticket never handed out: B200REG_EINVAL.  A ticket not waited for yet, a
 *     job that failed, a kind it did not capture, tracing off at its submit, or a released ticket: B200REG_ESTATE, the
 *     message says which.
 *   Release: B200REG_OK for any waited-for ticket, also one that holds nothing, and again for a released one;
 *     B200REG_ESTATE before its wait; B200REG_EINVAL for a ticket never handed out.                                   */
int b200reg_batch_set_loop_clouds(b200reg_batch* b, int mask);
int b200reg_batch_set_lm_trace(b200reg_batch* b, int enable);
int b200reg_batch_loop_clouds(b200reg_batch* b, int64_t ticket, int kind, int64_t* offsets_out, size_t capacity,
                              float* xyzi_out);
int b200reg_batch_lm_trace(b200reg_batch* b, int64_t ticket, int64_t* offsets_out, size_t capacity,
                           b200reg_lm_trial* trials_out);
/* Quatro matches of driver jobs (b200reg_ctx_set_quatro_matches / b200reg_quatro_matches per job).  The setting is off by
 * default and is copied at submit like the two above.  A job of b200reg_batch_submit_loop_closure or
 * _submit_perform_loop_closure that ran with it on returns, byte for byte, what b200reg_quatro_matches returns on a context
 * after the synchronous call with the same inputs.  The record moves into the job's outputs without a copy and stays
 * readable from b200reg_batch_wait until b200reg_batch_release or b200reg_batch_destroy.  The getter follows the rules of
 * b200reg_quatro_matches and the ticket rules above; an icpAlignment job, or one submitted with recording off, holds no
 * matches (B200REG_ESTATE).                                                                                            */
int b200reg_batch_set_quatro_matches(b200reg_batch* b, int enable);
int b200reg_batch_quatro_matches(b200reg_batch* b, int64_t ticket, int64_t* offsets_out, size_t capacity, int32_t* corr_out,
                                 int32_t* inlier_out, float* src_xyz_out, float* dst_xyz_out);
/* Residuals of driver jobs (b200reg_ctx_set_residuals / b200reg_residuals per job).  The setting is off by default and is
 * copied at submit like the ones above.  A job of any of the three kinds that ran with it on returns, byte for byte, what
 * b200reg_residuals returns on a context after the synchronous call with the same inputs.  The record moves into the
 * job's outputs without a copy and stays readable from b200reg_batch_wait until b200reg_batch_release or
 * b200reg_batch_destroy.  The getter follows the rules of b200reg_residuals and the ticket rules above; a job submitted
 * with recording off holds no residuals (B200REG_ESTATE).                                                              */
int b200reg_batch_set_residuals(b200reg_batch* b, int enable);
int b200reg_batch_residuals(b200reg_batch* b, int64_t ticket, int64_t* offsets_out, size_t capacity, int32_t* nn_out,
                            float* d2_out);
int b200reg_batch_release(b200reg_batch* b, int64_t ticket);
int64_t b200reg_batch_launch_count(const b200reg_batch* b);
int b200reg_batch_depth(const b200reg_batch* b);

/* ---- the ONE collective of the path (SURVEY.md §8(e)): all-gather of the fixed-size result records over NCCL.
 *      Rank 0 makes the id, the caller ships its 128 bytes to the other ranks by any means (MPI, a file, torch.distributed),
 *      every rank calls b200reg_comm_init on its own context.  NCCL is loaded at run time (libnccl.so.2). -------------- */
#define B200REG_UNIQUE_ID_BYTES 128
int b200reg_comm_unique_id(void* id_out128);
int b200reg_comm_init(b200reg_ctx* ctx, const void* id128, int rank, int world);
int b200reg_comm_destroy(b200reg_ctx* ctx);
int b200reg_comm_rank(const b200reg_ctx* ctx);   /* -1 without a communicator */
int b200reg_comm_world(const b200reg_ctx* ctx);  /* 1 without a communicator  */
/* ncclAllGather of n_local records per rank on the context's stream: all_out holds world * n_local records in rank
 * order on EVERY rank (bytes identical for any world size given the same shards).  Without a communicator (world 1)
 * it is a copy.                                                                                                   */
int b200reg_allgather_results(b200reg_ctx* ctx, const b200reg_result* local, int n_local, b200reg_result* all_out);

/* Output cloud of align(): final_transformation_ applied to the source in fp32
 * (lsq_registration_impl.hpp:114).  out_xyz: n x 3 floats (host), original point order.       */
int b200reg_transform_cloud(b200reg_ctx* ctx, const b200reg_cloud* cloud, const float* Tf16, float* out_xyz);

/* ---- debug taps used by the parity tests ------------------------------------------- */
/* Exact k-NN of host queries in a cloud: KdTreeFLANN::nearestKSearch (nanoflann.hpp:140-152), any k >= 1.
 * Queries are (x, y, z [, ...]) records qstride_bytes apart (a multiple of 4, >= 12), nq >= 1 (nq < 2^30 when k >= the
 * cloud size).  idx_out / d2_out: nq x k, each row ascending by (d2, original index) -- equal distances resolve to the lower
 * index; indices refer to the ORIGINAL point order; d2 is ((dx*dx) + dy*dy) + dz*dz in fp32 without FMA.  Slots past the
 * last neighbour hold index -1 and d2 FLT_MAX: k > n, points whose d2 overflows to +inf (never neighbours), and every slot
 * of a query with a NaN coordinate.  A row depends only on its query and the cloud: repeated calls, other batch sizes and
 * other query orders return identical bytes.  k <= 32 runs one thread per query, k > 32 one warp per query with the
 * queries in chunks, so device memory stays bounded (about 16 bytes per result entry of one chunk of max(2^23, cloud size)
 * entries) whatever nq * k is.  k <= 0, NULL pointers and bad strides: B200REG_EINVAL.                                */
int b200reg_knn(b200reg_ctx* ctx, const b200reg_cloud* cloud, const float* queries, size_t nq,
                size_t qstride_bytes, int k, int32_t* idx_out, float* d2_out);
/* Same answer by brute force (every point tested, tiles staged into shared memory by TMA bulk copies): the on-GPU
 * anchor the tree traversal is verified against at full size (100k x 100k).  k in 1..32.                   */
int b200reg_knn_bruteforce(b200reg_ctx* ctx, const b200reg_cloud* cloud, const float* queries, size_t nq,
                           size_t qstride_bytes, int k, int32_t* idx_out, float* d2_out);
/* Fixed-radius search: KdTreeFLANN::radiusSearch (nanoflann.hpp:154-175) for nq host queries at once, CSR output.
 * !! sq_radius is a SQUARED radius, exactly as the reference takes it: radiusSearch hands its `radius` argument unchanged
 * to RadiusResultSet<float, int> (nanoflann.hpp:162), which compares it with squared distances.  Passing 1.5 finds every
 * point with d2 < 1.5f (strict; the double is converted to float first); a PCL user expecting r -> r*r gets a ball of
 * radius sqrt(1.5).  d2 is the same fp32 expression as b200reg_knn's (((dx*dx) + dy*dy) + dz*dz, no FMA).
 * Queries are (x, y, z [, ...]) records qstride_bytes apart (a multiple of 4, >= 12), 1 <= nq < 2^30.
 * Results: the neighbours of query i are idx_out / d2_out [offsets_out[i], offsets_out[i+1]), offsets_out has nq + 1
 * entries; indices refer to the cloud's ORIGINAL order.  sorted != 0: ascending (d2, index) (the reference sorts by d2 with
 * ties unspecified); sorted == 0: ascending index (the reference returns its kd-tree's visit order, which no other index
 * reproduces).  The result is deterministic: repeated calls return identical bytes.
 * idx_out == d2_out == NULL: count only (offsets_out is filled).  If the total exceeds `capacity` (entries of each output)
 * the call fills offsets_out, leaves idx_out / d2_out untouched and returns B200REG_ESTATE, the total in the message.
 * Device memory is bounded: the queries are processed in chunks of ~8M neighbours (or one query, if it has more).   */
int b200reg_radius_search(b200reg_ctx* ctx, const b200reg_cloud* cloud, const float* queries, size_t nq,
                          size_t qstride_bytes, double sq_radius, int sorted, int64_t* offsets_out, size_t capacity,
                          int32_t* idx_out, float* d2_out);
/* The TEASER++ QUATRO solve on n given correspondences: correspondence i joins src_xyz[3i..3i+2] to dst_xyz[3i..3i+2]
 * (host floats).  TIM graph, core-number order, greedy clique, GNC-TLS yaw and TLS translation, exactly as
 * b200reg_quatro_align runs them.  `wide` picks the solver:
 *   0  the global-memory solver of advancedMatching sets up to B200REG_ADV_CORR_CAPACITY (n must not exceed it);
 *   2  the shared-memory solver of optimizedMatching sets (the deployment's), n <= B200REG_CORR_CAPACITY;
 *   any other value: the solver of advancedMatching sets beyond B200REG_ADV_CORR_CAPACITY, any 1 <= n < 2^20.
 * All three give the same clique and iteration count, and T up to the order of their fp64 sums.  info: T, valid,
 * clique_size, gnc_iterations (n_mutual = n_corr = n).  clique_out (optional, n ints): the clique's correspondence
 * indices, ascending.                                                                                           */
int b200reg_quatro_solve_tap(b200reg_ctx* ctx, int n, const float* src_xyz, const float* dst_xyz, int wide,
                             const b200reg_quatro_params* params, b200reg_quatro_info* info, int32_t* clique_out);
/* The feature matcher of b200reg_quatro_align alone, on caller descriptors: for each of `count` pairs, fi[k] (ni[k] x 33
 * host floats) and fj[k] (nj[k] x 33), in the matcher's roles (fi the base of the forward search: 1 <= nj[k] <= ni[k],
 * otherwise B200REG_EINVAL; b200reg_quatro_align swaps its clouds to get there).  An all-zero row is unusable: never a
 * neighbour, never matched.  Distances are fp32 ((e0*e0 + e1*e1) + ...) + e32*e32 without FMA, ties go to the lower row.
 *   nn_out[k]      nj[k]: row of fi nearest to row j of fj, -1 when it is unusable or no usable row lies within the gate
 *                  d2 <= fp32(distance_threshold)^2 (no gate when advanced != 0, or when that square overflows or is NaN)
 *   dis_out[k]     nj[k]: its squared distance (meaningful where nn >= 0)
 *   rnn_out[k]     ni[k]: row of fj nearest to row i of fi where the reverse search ran (optimizedMatching: i is the nn of
 *                  some j within the gate; advancedMatching: of any j), -1 elsewhere
 *   mutual_out[k]  up to nj[k] (i, j) pairs, ascending j: optimizedMatching keeps (i, j) when j is the lowest j whose nn
 *                  is i and rnn(i) == j; advancedMatching when nn(j) = i and rnn(i) == j
 *   n_mutual_out   count: the length of each mutual list (b200reg_quatro_info::n_mutual)                       */
int b200reg_match_tap(b200reg_ctx* ctx, int count, const float* const* fi, const int32_t* ni, const float* const* fj,
                      const int32_t* nj, double distance_threshold, int advanced, int32_t* const* nn_out,
                      float* const* dis_out, int32_t* const* rnn_out, int32_t* const* mutual_out, int32_t* n_mutual_out);
/* normals (n x 3, NaN where fewer than 3 neighbours) and FPFH (n x 33), original point order.            */
int b200reg_get_fpfh(b200reg_ctx* ctx, const b200reg_cloud* cloud, float* normals_out, float* fpfh_out);
/* n x 9 doubles (row-major 3x3 block of the reference's Matrix4d), original point order.          */
int b200reg_get_covariances(b200reg_ctx* ctx, const b200reg_cloud* cloud, double* cov9_out);
/* NanoGICP::linearize at pose T16 (nano_gicp_impl.hpp:213-270): H 6x6 row-major, b, sum of errors,
 * per-source-point correspondence (original target index or -1) and squared distance.             */
int b200reg_linearize(b200reg_ctx* ctx, const b200reg_cloud* src, const b200reg_cloud* tgt, const double* T16,
                      double max_corr_dist, double* H36, double* b6, double* err, int32_t* corr_out,
                      float* sqd_out);
/* NanoGICP::compute_error (nano_gicp_impl.hpp:272-296) in isolation: correspondences and Mahalanobis matrices are
 * taken from ONE linearize at T_lin16 (they stay stale, as in step_lm), then sum e^T M e is evaluated at T_trial16.  */
int b200reg_compute_error(b200reg_ctx* ctx, const b200reg_cloud* src, const b200reg_cloud* tgt, const double* T_lin16,
                          const double* T_trial16, double max_corr_dist, double* err);
/* The LM controller of the solve (step_lm, lsq_registration_impl.hpp:160-208) on n caller-supplied states, one device
 * thread per case, through the same device functions b200reg_gicp_align runs: mode 0 runs what follows a linearize
 * (lambda init, nu = 2, the first trial's step, or lm_failed when lm_max_iterations <= 0); mode 1 prepares one trial from
 * (H, b, lambda) and decides it on yi (accept / reject / converged / out of trials, the lambda and nu rules).       */
int b200reg_lm_step_tap(b200reg_ctx* ctx, int n, const b200reg_lm_case* cases, b200reg_lm_step* out);
/* The spatial index of `count` clouds, built exactly as b200reg_clouds_create builds them (same arguments, same batched
 * launches), read back and released.  Per cloud i of n[i] points:
 *   keys_out[i]    n[i] words: the 30-bit Morton keys in sorted order
 *   pts_out[i]     n[i] x 4 floats: the sorted points, w = the int bits of the original index
 *   rank_out[i]    n[i]: original index -> sorted position
 *   tnodes_out[i]  (n[i] - 1) x 16 floats (may be NULL when n[i] == 1): record r holds both children of internal node r,
 *                  (lo0.xyz, ref0) (hi0.xyz, -) (lo1.xyz, ref1) (hi1.xyz, -), a ref >= 0 naming an internal node and a ref
 *                  < 0 the leaf -1 - ((start << 4) | count); records inside a collapsed leaf are never written
 *   root_ref_out   count: 0 (an internal root) or the leaf reference of a cloud of at most 8 points                    */
int b200reg_index_tap(b200reg_ctx* ctx, int count, const float* const* xyz, const size_t* n, size_t stride_bytes, int on_device,
                      uint32_t* const* keys_out, float* const* pts_out, int32_t* const* rank_out, float* const* tnodes_out,
                      int32_t* root_ref_out);
/* The stable LSD radix sort the index build, the voxel grid, the matcher and the radius search share, on `count` caller
 * arrays of host (key, value) words in one batched call: keys_out[i] / vals_out[i] receive the n[i] pairs ordered by key,
 * equal keys in input order.  key_bits 30 (three 10-bit passes: the order of the low 30 bits, the bits above ride
 * along) or 32 (three 11-bit passes).  1 <= n[i] < 2^30, the most the sort's 30-bit tile counts hold.              */
int b200reg_sort_tap(b200reg_ctx* ctx, int count, const uint32_t* const* keys, const uint32_t* const* vals, const int32_t* n,
                     int key_bits, uint32_t* const* keys_out, uint32_t* const* vals_out);

#ifdef __cplusplus
}
#endif
#endif /* B200REG_H */
