// api_keyframes.cu -- the C ABI around registration: the keyframe store, candidate search, sub-map assembly,
// b200reg_perform_loop_closure and the loop factors.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>

#include "api.cuh"

// Keyframe clouds live in SLABS of their own (plain cudaMalloc, never the context's stream-ordered pool): a store only
// grows, while every registration call takes and returns hundreds of MB of scratch from the pool; 480 KB keyframes carved
// out of the pool's free scratch blocks between two calls fragmented it, and the pool then grew by a fresh block in almost
// every call (profiles/diag_sequence_e2e.py times the steps).
struct KfSlab {
  float4* base = nullptr;
  size_t cap = 0, used = 0;  // points
};
// What a loop-closure attempt reads of the store.  The store keeps the live state; a job of the batch driver
// (b200reg_batch_submit_perform_loop_closure) keeps a copy taken at submit.  Both read keyframes through this one shape.
struct KfState {
  std::vector<float4*> pts;
  std::vector<int> n;
  std::vector<double> poses;   // 16 per keyframe, row-major
  std::vector<double> stamps;
  int size() const { return (int)pts.size(); }
};
// The stream-ordered mark of the latest ingest: recorded on the ingesting context's stream after every add; a job's stream
// waits for it before the job reads a keyframe.  A mark that a job still holds is never recorded again: the next add makes
// a new one.
struct IngestMark {
  cudaEvent_t ev = nullptr;
  ~IngestMark() {
    if (ev) cudaEventDestroy(ev);
  }
};
struct b200reg_keyframes {
  KfState st;
  std::vector<KfSlab> slabs;
  int device = 0;
  std::shared_ptr<IngestMark> ingest;
  std::atomic<int> jobs{0};  // batch-driver jobs that hold a copy of `st` and have not finished
};
constexpr size_t KF_SLAB_POINTS = (size_t)8 << 20;  // 8 Mi points = 128 MB per slab unless reserved otherwise

// room for n more points: the tail of the last slab, else a new slab (cudaMalloc: a rare, synchronous event)
static int kf_alloc(b200reg_keyframes* kf, size_t n, size_t min_slab, float4** out) {
  if (kf->slabs.empty() || kf->slabs.back().cap - kf->slabs.back().used < n) {
    KfSlab sl;
    sl.cap = std::max(n, min_slab);
    CU(cudaMalloc((void**)&sl.base, sl.cap * sizeof(float4)));
    kf->slabs.push_back(sl);
  }
  KfSlab& sl = kf->slabs.back();
  *out = sl.base + sl.used;
  sl.used += n;
  return B200REG_OK;
}

// after the uploads of an add are queued on c's stream: mark them for the jobs that will read the new keyframe
static int mark_ingest(b200reg_ctx* c, b200reg_keyframes* kf) {
  // only this thread hands out marks, so a use count of 1 cannot grow under us: no job holds this mark
  if (!kf->ingest || kf->ingest.use_count() > 1) {
    std::shared_ptr<IngestMark> m(new IngestMark);
    CU(cudaEventCreateWithFlags(&m->ev, cudaEventDisableTiming));
    kf->ingest = m;
  }
  CU(cudaEventRecord(kf->ingest->ev, c->stream));
  return B200REG_OK;
}

static int assemble_clouds(b200reg_ctx* c, const KfState& kf, int count, const int32_t* src_idx, const int32_t* dst_idx,
                           const b200reg_loop_config* cfg, const int32_t* n_keyframes, bool keep_intensity, b200reg_cloud** src_out,
                           b200reg_cloud** dst_out);
static int fetch_closest(b200reg_ctx* c, const KfState& kf, int count, const int32_t* query_idx, double radius, double tdiff,
                         int32_t* closest_out);
static int perform_loop_closure(b200reg_ctx* c, Recording& rec, const KfState& kf, int count, const int32_t* query_idx,
                                const int32_t* closest_idx, const b200reg_loop_config* cfg, b200reg_result* out,
                                b200reg_quatro_info* quatro_out);

// the configuration ranges sub-map assembly refuses (nullptr: none), for the call itself and for a job's submit
static const char* assembly_config_error(const b200reg_loop_config* cfg) {
  if (2 * cfg->num_submap_keyframes + 1 > MAXSEG) return "num_submap_keyframes too large";
  if (!(cfg->voxel_res > 0)) return "voxel_res must be positive";
  return nullptr;
}

extern "C" {

void b200reg_default_loop_config(b200reg_loop_config* cfg) {
  if (!cfg) return;
  cfg->enable_quatro = 1;
  cfg->enable_submap_matching = 0;
  cfg->num_submap_keyframes = 5;
  cfg->reserved = 0;
  cfg->voxel_res = 0.3;
  cfg->loop_detection_radius = 35.0;
  cfg->loop_detection_timediff_threshold = 30.0;
  b200reg_default_gicp_params(&cfg->gicp);
  b200reg_default_quatro_params(&cfg->quatro);
}

int b200reg_keyframes_create(b200reg_ctx* c, b200reg_keyframes** out) {
  if (!c || !out) return fail(B200REG_EINVAL, "bad argument");
  *out = new b200reg_keyframes;
  (*out)->device = c->device;
  return B200REG_OK;
}

int b200reg_keyframes_destroy(b200reg_ctx* c, b200reg_keyframes* kf) {
  if (!kf) return B200REG_OK;
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  if (kf->jobs.load() > 0)
    return fail(B200REG_ESTATE, "batch-driver jobs that read this keyframe store are in flight; wait for them first");
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));  // nothing in flight may still read a keyframe
  for (KfSlab& sl : kf->slabs) CU(cudaFree(sl.base));
  delete kf;
  return B200REG_OK;
}

int b200reg_keyframes_reserve(b200reg_ctx* c, b200reg_keyframes* kf, size_t n_points) {
  if (!c || !kf) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  if (!kf->slabs.empty() && kf->slabs.back().cap - kf->slabs.back().used >= n_points) return B200REG_OK;
  if (n_points == 0) return B200REG_OK;
  KfSlab sl;
  sl.cap = n_points;
  CU(cudaMalloc((void**)&sl.base, sl.cap * sizeof(float4)));
  kf->slabs.push_back(sl);
  return B200REG_OK;
}

int b200reg_keyframes_size(const b200reg_keyframes* kf) { return kf ? (int)kf->st.pts.size() : 0; }

int b200reg_keyframes_add(b200reg_ctx* c, b200reg_keyframes* kf, const float* xyzi, size_t n, size_t stride_bytes, const double* pose16,
                          double timestamp) {
  if (!c || !kf || !xyzi || n == 0 || !pose16 || stride_bytes < 16 || stride_bytes % 4) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  float4* d = nullptr;
  {
    const int rc = kf_alloc(kf, n, KF_SLAB_POINTS, &d);
    if (rc) return rc;
  }
  if (stride_bytes == 16) {  // already packed (x, y, z, intensity): one linear copy (a 2-D copy of n 16-byte rows crawls)
    CU(cudaMemcpyAsync(d, xyzi, n * 16, cudaMemcpyHostToDevice, c->stream));
  } else {  // pcl::PointXYZI (32 B) and friends: upload the records as they are, repack on the device
    Scratch scratch(c);
    float* d_raw = nullptr;
    CU(scratch.upload(&d_raw, xyzi, n * stride_bytes));
    launch_pack_xyzi(d_raw, (int)(stride_bytes / 4), (int)n, d, c->stream);
    c->launches++;
    CU(cudaGetLastError());
  }
  {
    const int rc = mark_ingest(c, kf);
    if (rc) return rc;
  }
  kf->st.pts.push_back(d);
  kf->st.n.push_back((int)n);
  kf->st.poses.insert(kf->st.poses.end(), pose16, pose16 + 16);
  kf->st.stamps.push_back(timestamp);
  return (int)kf->st.pts.size() - 1;
}

namespace {
// inverse of a 4x4 by cofactors (what pose_eig_.inverse() computes for a fixed-size 4x4; row-major in, row-major out)
bool inverse4(const double* m, double* inv) {
  double a[16];
  a[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
  a[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
  a[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
  a[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
  a[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
  a[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
  a[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
  a[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
  a[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
  a[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
  a[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
  a[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
  a[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
  a[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
  a[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
  a[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
  const double det = m[0] * a[0] + m[1] * a[4] + m[2] * a[8] + m[3] * a[12];
  if (det == 0.0) return false;
  for (int i = 0; i < 16; i++) inv[i] = a[i] / det;
  return true;
}
}  // namespace

int b200reg_keyframes_add_world(b200reg_ctx* c, b200reg_keyframes* kf, const float* xyzi_world, size_t n, size_t stride_bytes,
                                const double* pos, const double* q, double timestamp) {
  if (!c || !kf || !xyzi_world || n == 0 || !pos || !q || stride_bytes < 16 || stride_bytes % 4) return fail(B200REG_EINVAL, "bad argument");
  // tf::Matrix3x3(q) = setRotation(q) (tf/LinearMath/Matrix3x3.h; tf itself is not vendored): s = 2 / |q|^2
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double d = x * x + y * y + z * z + w * w;
  if (!(d > 0.0)) return fail(B200REG_EINVAL, "zero quaternion");
  const double sc = 2.0 / d;
  const double xs = x * sc, ys = y * sc, zs = z * sc;
  const double wx = w * xs, wy = w * ys, wz = w * zs, xx = x * xs, xy = x * ys, xz = x * zs, yy = y * ys, yz = y * zs, zz = z * zs;
  const double P[16] = {1.0 - (yy + zz), xy - wz, xz + wy, pos[0], xy + wz, 1.0 - (xx + zz), yz - wx, pos[1],
                        xz - wy, yz + wx, 1.0 - (xx + yy), pos[2], 0.0, 0.0, 0.0, 1.0};
  double Tinv[16];
  if (!inverse4(P, Tinv)) return fail(B200REG_EINVAL, "singular pose");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  float* d_raw = nullptr;
  double* d_T = nullptr;
  float4* d_out = nullptr;
  CU(scratch.upload(&d_raw, xyzi_world, n * stride_bytes));
  CU(scratch.upload(&d_T, Tinv, 128));
  {
    const int rc = kf_alloc(kf, n, KF_SLAB_POINTS, &d_out);
    if (rc) return rc;
  }
  launch_ingest_world(d_raw, (int)(stride_bytes / 4), (int)n, d_T, d_out, s);
  c->launches++;
  CU(cudaGetLastError());
  {
    const int rc = mark_ingest(c, kf);
    if (rc) return rc;
  }
  CU(cudaStreamSynchronize(s));  // Tinv lives on this stack frame; the caller's message buffer may go away
  kf->st.pts.push_back(d_out);
  kf->st.n.push_back((int)n);
  kf->st.poses.insert(kf->st.poses.end(), P, P + 16);
  kf->st.stamps.push_back(timestamp);
  return (int)kf->st.pts.size() - 1;
}

int b200reg_keyframes_get(b200reg_ctx* c, const b200reg_keyframes* kf, int idx, float* xyzi_out, double* pose16_out, double* ts_out) {
  if (!c || !kf || idx < 0 || idx >= (int)kf->st.pts.size()) return fail(B200REG_EINVAL, "bad argument");
  if (pose16_out) memcpy(pose16_out, &kf->st.poses[16 * (size_t)idx], 128);
  if (ts_out) *ts_out = kf->st.stamps[idx];
  if (xyzi_out) {
    CU(cudaSetDevice(c->device));
    CU(cudaMemcpyAsync(xyzi_out, kf->st.pts[idx], (size_t)kf->st.n[idx] * 16, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
  }
  return B200REG_OK;
}

size_t b200reg_keyframes_cloud_size(const b200reg_keyframes* kf, int idx) {
  return (kf && idx >= 0 && idx < (int)kf->st.n.size()) ? (size_t)kf->st.n[idx] : 0;
}

int b200reg_keyframes_set_pose(b200reg_ctx* c, b200reg_keyframes* kf, int idx, const double* pose16) {
  if (!c || !kf || !pose16 || idx < 0 || idx >= (int)kf->st.pts.size()) return fail(B200REG_EINVAL, "bad argument");
  memcpy(&kf->st.poses[16 * (size_t)idx], pose16, 128);
  return B200REG_OK;
}

// ---- result consumption (host arithmetic only) -------------------------------------------------------
namespace {
// poseEigToGtsamPose (utilities.hpp:67-75): tf::Matrix3x3::getRPY (getEulerYPR, solution 1), then gtsam::Rot3::RzRyRx
void pose_rpy_roundtrip(const double* P, double R[9], double t[3]) {
  const double m00 = P[0], m10 = P[4], m20 = P[8], m21 = P[9], m22 = P[10];
  double roll, pitch, yaw;
  if (fabs(m20) >= 1.0) {  // gimbal-lock branch of tf's getEulerYPR (tf is not vendored; restated from
                           // tf/LinearMath/Matrix3x3.h: yaw = 0, roll = atan2(m21, m22) in both sub-cases)
    yaw = 0.0;
    roll = atan2(m21, m22);
    pitch = m20 < 0 ? M_PI / 2.0 : -M_PI / 2.0;
  } else {
    pitch = -asin(m20);
    const double cp = cos(pitch);
    roll = atan2(m21 / cp, m22 / cp);
    yaw = atan2(m10 / cp, m00 / cp);
  }
  const double cx = cos(roll), sx = sin(roll), cy = cos(pitch), sy = sin(pitch), cz = cos(yaw), sz = sin(yaw);
  // Rz(yaw) * Ry(pitch) * Rx(roll)
  R[0] = cz * cy; R[1] = cz * sy * sx - sz * cx; R[2] = cz * sy * cx + sz * sx;
  R[3] = sz * cy; R[4] = sz * sy * sx + cz * cx; R[5] = sz * sy * cx - cz * sx;
  R[6] = -sy;     R[7] = cy * sx;                R[8] = cy * cx;
  t[0] = P[3]; t[1] = P[7]; t[2] = P[11];
}
}  // namespace

int b200reg_loop_factor_from_poses(const double* Tb, const double* Pl, const double* Pc, double score, int valid, int from_idx,
                                   int to_idx, b200reg_loop_factor* out) {
  if (!Tb || !Pl || !Pc || !out) return fail(B200REG_EINVAL, "bad argument");
  double F[16];  // pose_between_eig_ * latest.pose_corrected_eig_ (Matrix4d product)
  for (int r = 0; r < 4; r++)
    for (int cidx = 0; cidx < 4; cidx++) {
      double s = 0;
      for (int k = 0; k < 4; k++) s += Tb[4 * r + k] * Pl[4 * k + cidx];
      F[4 * r + cidx] = s;
    }
  double R1[9], t1[3], R2[9], t2[3];
  pose_rpy_roundtrip(F, R1, t1);
  pose_rpy_roundtrip(Pc, R2, t2);
  // Pose3::between: inverse(from) * to = (R1^T R2, R1^T (t2 - t1))
  double* M = out->measurement;
  for (int r = 0; r < 3; r++) {
    for (int cidx = 0; cidx < 3; cidx++) {
      double s = 0;
      for (int k = 0; k < 3; k++) s += R1[3 * k + r] * R2[3 * k + cidx];
      M[4 * r + cidx] = s;
    }
    double s = 0;
    for (int k = 0; k < 3; k++) s += R1[3 * k + r] * (t2[k] - t1[k]);
    M[4 * r + 3] = s;
  }
  M[12] = M[13] = M[14] = 0.0;
  M[15] = 1.0;
  for (int k = 0; k < 6; k++) out->variances[k] = score;
  out->from_idx = from_idx;
  out->to_idx = to_idx;
  out->valid = valid ? 1 : 0;
  out->reserved = 0;
  return B200REG_OK;
}

int b200reg_loop_factors(b200reg_ctx* c, const b200reg_keyframes* kf, int count, const int32_t* query_idx, const int32_t* closest_idx,
                         const b200reg_result* results, b200reg_loop_factor* out) {
  if (!c || !kf || count <= 0 || !query_idx || !closest_idx || !results || !out) return fail(B200REG_EINVAL, "bad argument");
  const int nk = (int)kf->st.pts.size();
  for (int i = 0; i < count; i++) {
    if (query_idx[i] < 0 || query_idx[i] >= nk || closest_idx[i] >= nk) return fail(B200REG_EINVAL, "keyframe index out of range");
    if (closest_idx[i] < 0) {  // no candidate: the reference returns before any registration (fast_lio_sam_qn.cpp:213-216)
      memset(&out[i], 0, sizeof(b200reg_loop_factor));
      out[i].from_idx = query_idx[i];
      out[i].to_idx = -1;
      continue;
    }
    const int rc = b200reg_loop_factor_from_poses(results[i].pose_between, &kf->st.poses[16 * (size_t)query_idx[i]], &kf->st.poses[16 * (size_t)closest_idx[i]],
                                                  results[i].fitness, results[i].valid, query_idx[i], closest_idx[i], &out[i]);
    if (rc) return rc;
  }
  return B200REG_OK;
}

int b200reg_fetch_closest_keyframes(b200reg_ctx* c, b200reg_keyframes* kf, int count, const int32_t* query_idx, double radius,
                                    double tdiff, int32_t* closest_out) {
  if (!c || !kf || count <= 0 || !query_idx || !closest_out) return fail(B200REG_EINVAL, "bad argument");
  return fetch_closest(c, kf->st, count, query_idx, radius, tdiff, closest_out);
}

int b200reg_assemble_clouds(b200reg_ctx* c, b200reg_keyframes* kf, int count, const int32_t* src_idx, const int32_t* dst_idx,
                            const b200reg_loop_config* cfg, int n_keyframes, b200reg_cloud** src_out, b200reg_cloud** dst_out) {
  if (!kf || count <= 0) return fail(B200REG_EINVAL, "bad argument");
  std::vector<int32_t> nks(count, n_keyframes > 0 ? n_keyframes : (int)kf->st.pts.size());
  return b200reg_assemble_clouds_at(c, kf, count, src_idx, dst_idx, cfg, nks.data(), src_out, dst_out);
}

int b200reg_assemble_clouds_at(b200reg_ctx* c, b200reg_keyframes* kf, int count, const int32_t* src_idx, const int32_t* dst_idx,
                               const b200reg_loop_config* cfg, const int32_t* n_keyframes, b200reg_cloud** src_out,
                               b200reg_cloud** dst_out) {
  if (!kf) return fail(B200REG_EINVAL, "bad argument");
  return assemble_clouds(c, kf->st, count, src_idx, dst_idx, cfg, n_keyframes, false, src_out, dst_out);
}

}  // extern "C"

static int fetch_closest(b200reg_ctx* c, const KfState& kf, int count, const int32_t* query_idx, double radius, double tdiff,
                         int32_t* closest_out) {
  const int nk = kf.size();
  for (int i = 0; i < count; i++)
    if (query_idx[i] < 0 || query_idx[i] >= nk) return fail(B200REG_EINVAL, "query index out of range");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  std::vector<double> pos(3 * (size_t)nk);
  for (int i = 0; i < nk; i++)
    for (int d = 0; d < 3; d++) pos[3 * (size_t)i + d] = kf.poses[16 * (size_t)i + 4 * d + 3];
  double *d_pos = nullptr, *d_st = nullptr;
  int *d_q = nullptr, *d_o = nullptr;
  CU(scratch.upload(&d_pos, pos.data(), pos.size() * 8));
  CU(scratch.upload(&d_st, kf.stamps.data(), (size_t)nk * 8));
  CU(scratch.upload(&d_q, query_idx, (size_t)count * 4));
  CU(scratch.alloc((void**)&d_o, (size_t)count * 4));
  c->launches += launch_fetch_closest(d_pos, d_st, d_q, count, radius, tdiff, d_o, s);
  CU(cudaMemcpyAsync(closest_out, d_o, (size_t)count * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

// b200reg_assemble_clouds_at; keep_intensity: the clouds keep the voxel-mean intensities (b200reg_cloud::inten)
static int assemble_clouds(b200reg_ctx* c, const KfState& kf, int count, const int32_t* src_idx, const int32_t* dst_idx,
                           const b200reg_loop_config* cfg, const int32_t* n_keyframes, bool keep_intensity, b200reg_cloud** src_out,
                           b200reg_cloud** dst_out) {
  if (!c || count <= 0 || !src_idx || !dst_idx || !cfg || !n_keyframes || !src_out || !dst_out)
    return fail(B200REG_EINVAL, "bad argument");
  for (int i = 0; i < count; i++)
    if (n_keyframes[i] <= 0 || n_keyframes[i] > kf.size()) return fail(B200REG_EINVAL, "n_keyframes out of range");
  if (const char* e = assembly_config_error(cfg)) return fail(B200REG_EINVAL, e);
  const int range = cfg->num_submap_keyframes;
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  const int njobs = 2 * count;  // jobs [0,count) = src clouds, [count, 2 count) = dst clouds
  std::vector<AssembleJob> jobs(njobs);
  std::vector<SortDev> sorts(njobs);
  int max_total = 0;
  for (int j = 0; j < njobs; j++) {
    const bool is_src = j < count;
    const int centre = is_src ? src_idx[j] : dst_idx[j - count];
    const int nk = n_keyframes[is_src ? j : j - count];  // keyframes.size() at this pair's tick
    if (centre < 0 || centre >= nk) return fail(B200REG_EINVAL, "keyframe index out of range");
    AssembleJob& J = jobs[j];
    memset(&J, 0, sizeof(J));
    // loop_closure.cpp:68-105: which keyframes are merged
    const bool merged = cfg->enable_submap_matching || (!is_src && !cfg->enable_quatro);
    J.nseg = 0;
    J.seg_off[0] = 0;
    if (merged) {
      for (int i = centre - range; i < centre + range + 1; i++)
        if (i >= 0 && i < nk - 1) {  // the reference excludes the last keyframe (loop_closure.cpp:72,79,100)
          J.seg_kf[J.nseg] = i;
          J.seg_off[J.nseg + 1] = J.seg_off[J.nseg] + kf.n[i];
          J.nseg++;
        }
    } else {
      J.seg_kf[0] = centre;
      J.seg_off[1] = kf.n[centre];
      J.nseg = 1;
    }
    J.total = J.seg_off[J.nseg];
    if (J.total <= 0) return fail(B200REG_EINVAL, "empty merged cloud");
    const size_t n = J.total;
    Layout l;
    const size_t o_m = l.take(n * 16), o_o = l.take(n * 16), o_h = l.take(n * 4), o_b = l.take(32), o_c = l.take(sizeof(AssembleCounters));
    const SortLayout sl(l, l, J.total, 32);
    char* slab = nullptr;
    CU(scratch.alloc((void**)&slab, l.size));
    J.merged = (float4*)(slab + o_m);
    J.out = (float4*)(slab + o_o);
    J.heads = (int*)(slab + o_h);
    J.bbox = (int*)(slab + o_b);
    J.counters = (AssembleCounters*)(slab + o_c);
    sorts[j] = sl.bind(slab, slab);
    CU(cudaMemsetAsync(sorts[j].hist, 0, sl.ws, s));
    max_total = std::max(max_total, J.total);
  }
  const int nkall = kf.size();
  std::vector<KeyframeDev> kd(nkall);
  for (int i = 0; i < nkall; i++) kd[i] = KeyframeDev{kf.pts[i], kf.n[i], 0};
  AssembleJob* d_jobs = nullptr;
  SortDev* d_sorts = nullptr;
  KeyframeDev* d_kf = nullptr;
  double* d_poses = nullptr;
  CU(scratch.upload(&d_jobs, jobs.data(), sizeof(AssembleJob) * njobs));
  CU(scratch.upload(&d_sorts, sorts.data(), sizeof(SortDev) * njobs));
  CU(scratch.upload(&d_kf, kd.data(), sizeof(KeyframeDev) * nkall));
  CU(scratch.upload(&d_poses, kf.poses.data(), 128 * (size_t)nkall));
  {
    ProfScope ps(c, CLS_MISC);
    const float inv_leaf = 1.0f / (float)cfg->voxel_res;
    c->launches += launch_assemble_voxelize(d_jobs, d_sorts, njobs, max_total, d_kf, d_poses, inv_leaf, s);
    for (int j = 0; j < njobs; j++) c->prof_bytes[CLS_MISC] += 68.0 * jobs[j].total;  // 16 in + 16 merged + 36 sort/centroid
  }
  CU(cudaGetLastError());
  std::vector<AssembleCounters> counters(njobs);
  for (int j = 0; j < njobs; j++) CU(cudaMemcpyAsync(&counters[j], jobs[j].counters, sizeof(AssembleCounters), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  // index the voxelised clouds (records are (x, y, z, intensity), 16-byte stride, already on the device)
  std::vector<const float*> ptrs(njobs);
  std::vector<size_t> ns(njobs);
  for (int j = 0; j < njobs; j++) {
    const bool overflow = counters[j].overflow != 0;  // PCL returns the input unchanged in that case
    ptrs[j] = (const float*)(overflow ? jobs[j].merged : jobs[j].out);
    ns[j] = overflow ? (size_t)jobs[j].total : (size_t)counters[j].voxels;
  }
  std::vector<b200reg_cloud*> clouds(njobs, nullptr);
  int rc = clouds_create(c, njobs, ptrs.data(), ns.data(), 16, 1, keep_intensity, clouds.data());
  for (int i = 0; i < count && !rc; i++) {
    src_out[i] = clouds[i];
    dst_out[i] = clouds[count + i];
  }
  return rc;
}

extern "C" {

int b200reg_perform_loop_closure(b200reg_ctx* c, b200reg_keyframes* kf, int count, const int32_t* query_idx, const int32_t* closest_idx,
                                 const b200reg_loop_config* cfg, b200reg_result* out, b200reg_quatro_info* quatro_out) {
  Recording rec(c, REC_ALL);
  if (!c || !kf || count <= 0 || !query_idx || !closest_idx || !cfg || !out) return fail(B200REG_EINVAL, "bad argument");
  return perform_loop_closure(c, rec, kf->st, count, query_idx, closest_idx, cfg, out, quatro_out);
}

}  // extern "C"

// b200reg_perform_loop_closure on a view of the store: the live one, or a batch-driver job's copy.  Its stages run on the
// queries with a candidate, where[k] for stage pair k, and `rec` stores their records renumbered to all queries.
static int perform_loop_closure(b200reg_ctx* c, Recording& rec, const KfState& kf, int count, const int32_t* query_idx,
                                const int32_t* closest_idx, const b200reg_loop_config* cfg, b200reg_result* out,
                                b200reg_quatro_info* quatro_out) {
  LoopCapture cap(c);
  std::vector<int32_t> qs, cs;
  std::vector<int> where;
  for (int i = 0; i < count; i++) {
    out[i] = default_result();  // dummy output whose is_valid is false (loop_closure.cpp:201-204)
    if (quatro_out) memset(&quatro_out[i], 0, sizeof(b200reg_quatro_info));
    if (closest_idx[i] >= 0) {
      qs.push_back(query_idx[i]);
      cs.push_back(closest_idx[i]);
      where.push_back(i);
    }
  }
  if (qs.empty()) return rec.commit(B200REG_OK, count, where);  // no stage runs: every row is empty
  const int m = (int)qs.size();
  // at the time query q was the latest keyframe the vector held q + 1 keyframes (fast_lio_sam_qn.cpp:205-219); a batch
  // replays several ticks, so every pair carries the size its own tick saw (the sub-map bounds of loop_closure.cpp:72,79,100)
  std::vector<int32_t> nks(m);
  for (int k = 0; k < m; k++) nks[k] = qs[k] + 1;
  std::vector<b200reg_cloud*> sc(m, nullptr), dc(m, nullptr);
  int rc = assemble_clouds(c, kf, m, qs.data(), cs.data(), cfg, nks.data(), cap.on(), sc.data(), dc.data());
  if (rc) return rc;
  CloudBag bag(c);
  bag.cl = sc;
  bag.cl.insert(bag.cl.end(), dc.begin(), dc.end());
  if ((rc = cap.clouds(m, sc.data(), dc.data(), true, cfg->enable_quatro != 0))) return rc;
  ResidualSlab rslab(c);
  {
    std::vector<size_t> sn(m);  // the fine stage's source clouds have the sizes of the assembled sources
    for (int k = 0; k < m; k++) sn[k] = (size_t)sc[k]->dev.n;
    if ((rc = rslab.reserve(m, sn.data()))) return rc;
  }
  std::vector<b200reg_result> res(m);
  std::vector<b200reg_quatro_info> qi(m);
  std::vector<float> fine_tf(16 * (size_t)m);  // the fine stage's transform of align()'s output cloud
  if (cfg->enable_quatro) {
    rc = coarse_to_fine_on_clouds(c, m, sc.data(), dc.data(), &cfg->quatro, &cfg->gicp, res.data(), qi.data(), fine_tf.data());
  } else {
    rc = b200reg_gicp_align(c, m, sc.data(), dc.data(), nullptr, &cfg->gicp, res.data());
    for (int k = 0; k < m && !rc; k++) memcpy(&fine_tf[16 * (size_t)k], res[k].Tf, sizeof(res[k].Tf));
  }
  for (int k = 0; k < m && !rc; k++) {
    out[where[k]] = res[k];
    if (quatro_out && cfg->enable_quatro) quatro_out[where[k]] = qi[k];
  }
  if (!rc) rc = cap.finish(cfg->enable_quatro ? qi.data() : nullptr, fine_tf.data());
  return rec.commit(rc, count, where);
}

// ---- b200reg_perform_loop_closure as a job of the batch driver (batch.cu) ------------------------------------------
struct KfJob {
  b200reg_keyframes* kf;
  KfState st;                         // the store at submit
  std::shared_ptr<IngestMark> ingest;  // the last add before submit (null: nothing was ever added)
  std::vector<int32_t> query, closest;  // closest empty: the job runs fetchClosestKeyframeIdx first
  b200reg_loop_config cfg;
  explicit KfJob(b200reg_keyframes* k) : kf(k) { kf->jobs++; }
  ~KfJob() { kf->jobs--; }
};

namespace b200 {

int kf_job_create(b200reg_keyframes* kf, int device, int count, const int32_t* query_idx, const int32_t* closest_idx,
                  const b200reg_loop_config* cfg, std::shared_ptr<KfJob>* out) {
  if (!kf || count <= 0 || !query_idx || !cfg || !out) return fail(B200REG_EINVAL, "bad argument");
  if (kf->device != device) return fail(B200REG_EINVAL, "the keyframe store lives on another device than the batch driver");
  // what the synchronous call refuses: b200reg_fetch_closest_keyframes checks every query, assembly every pair with a
  // candidate (the query's keyframe count q + 1 must exist and hold the candidate)
  const int nk = kf->st.size();
  for (int i = 0; i < count; i++) {
    const int q = query_idx[i];
    if (!closest_idx && (q < 0 || q >= nk)) return fail(B200REG_EINVAL, "query index out of range");
    if (closest_idx && closest_idx[i] >= 0 && (q < 0 || q >= nk || closest_idx[i] > q))
      return fail(B200REG_EINVAL, "keyframe index out of range");
  }
  if (const char* e = assembly_config_error(cfg)) return fail(B200REG_EINVAL, e);
  std::shared_ptr<KfJob> j(new KfJob(kf));
  j->st = kf->st;
  j->ingest = kf->ingest;
  j->query.assign(query_idx, query_idx + count);
  if (closest_idx) j->closest.assign(closest_idx, closest_idx + count);
  j->cfg = *cfg;
  *out = std::move(j);
  return B200REG_OK;
}

int kf_job_run(b200reg_ctx* c, KfJob* j, b200reg_result* out, b200reg_quatro_info* quatro_out) {
  Recording rec(c, REC_ALL);
  CU(cudaSetDevice(c->device));
  if (j->ingest) CU(cudaStreamWaitEvent(c->stream, j->ingest->ev, 0));  // the adds' uploads land before any read
  const int count = (int)j->query.size();
  int rc = B200REG_OK;
  if (j->closest.empty()) {
    j->closest.resize(count);
    rc = fetch_closest(c, j->st, count, j->query.data(), j->cfg.loop_detection_radius, j->cfg.loop_detection_timediff_threshold,
                       j->closest.data());
  }
  if (!rc) rc = perform_loop_closure(c, rec, j->st, count, j->query.data(), j->closest.data(), &j->cfg, out, quatro_out);
  // a failed call may return with its kernels still queued: none may read a keyframe once the job counts as finished
  const cudaError_t e = cudaStreamSynchronize(c->stream);
  if (!rc && e != cudaSuccess) rc = fail(B200REG_ECUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
  return rc;
}

}  // namespace b200
