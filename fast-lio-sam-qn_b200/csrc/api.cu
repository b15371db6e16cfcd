// api.cu -- the C ABI declared in include/b200reg.h: errors, defaults, contexts and profiling, cloud objects and their taps,
// the NCCL collective.  Registration lives in api_gicp.cu / api_quatro.cu, the keyframe store in api_keyframes.cu.
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "api.cuh"

namespace b200 {
static thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

// gicp_step = the whole LM loop of a solve when it runs as one graph launch; with profiling enabled the same kernels are
// launched one by one and timed per kernel: gicp_search / gicp_accum / gicp_control (and gicp_step stays empty)
static const char* kClassNames[NCLS] = {"index_build", "knn_covariance", "gicp_step", "misc", "fpfh", "quatro_match_solve",
                                        "gicp_search", "gicp_accum", "gicp_control"};

cudaEvent_t prof_event(b200reg_ctx* c) {
  cudaEvent_t e;
  if (!c->free_events.empty()) {
    e = c->free_events.back();
    c->free_events.pop_back();
  } else {
    cudaEventCreate(&e);
  }
  return e;
}
static void prof_resolve(b200reg_ctx* c) {
  for (auto& sp : c->pending) {
    float ms = 0.f;
    cudaEventSynchronize(sp.b);
    cudaEventElapsedTime(&ms, sp.a, sp.b);
    c->prof_ms[sp.cls] += ms;
    c->free_events.push_back(sp.a);
    c->free_events.push_back(sp.b);
  }
  c->pending.clear();
}

b200reg_result default_result() {
  b200reg_result r;
  memset(&r, 0, sizeof(r));
  for (int a = 0; a < 16; a += 5) {
    r.T[a] = r.pose_between[a] = 1.0;
    r.Tf[a] = 1.f;
  }
  r.fitness = 1.7976931348623157e308;
  return r;
}

int create_pair_clouds(b200reg_ctx* c, int count, const float* const* src_xyz, const size_t* src_n, const float* const* tgt_xyz,
                       const size_t* tgt_n, size_t stride_bytes, int on_device, bool keep_intensity, CloudBag& bag,
                       b200reg_cloud** src_out, b200reg_cloud** tgt_out) {
  std::vector<const float*> ptrs(src_xyz, src_xyz + count);
  ptrs.insert(ptrs.end(), tgt_xyz, tgt_xyz + count);
  std::vector<size_t> ns(src_n, src_n + count);
  ns.insert(ns.end(), tgt_n, tgt_n + count);
  std::vector<b200reg_cloud*> cl(2 * count, nullptr);
  const int rc = clouds_create(c, 2 * count, ptrs.data(), ns.data(), stride_bytes, on_device, keep_intensity, cl.data());
  if (rc) return rc;
  bag.cl.insert(bag.cl.end(), cl.begin(), cl.end());
  std::copy(cl.begin(), cl.begin() + count, src_out);
  std::copy(cl.begin() + count, cl.end(), tgt_out);
  return B200REG_OK;
}

int sorted_to_original(b200reg_ctx* c, const CloudDev& d, std::vector<int>& orig, std::vector<float4>* pts_out) {
  std::vector<float4> pts(d.n);
  CU(cudaMemcpyAsync(pts.data(), d.pts, (size_t)d.n * 16, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  orig.resize(d.n);
  for (int p = 0; p < d.n; p++) memcpy(&orig[p], &pts[p].w, 4);
  if (pts_out) pts_out->swap(pts);
  return B200REG_OK;
}
}  // namespace b200

extern "C" {

void b200reg_default_gicp_params(b200reg_gicp_params* p) {
  if (!p) return;
  p->k_correspondences = 15;
  p->max_iterations = 32;
  p->max_corr_dist = 52.5;
  p->transformation_eps = 0.01;
  p->rotation_eps = 2e-3;
  p->lm_max_iterations = 10;
  p->regularization = 3;  // PLANE
  p->lm_init_lambda_factor = 1e-9;
  p->icp_score_thr = 1.5;
}

const char* b200reg_last_error(void) { return g_err.c_str(); }
void b200reg_set_last_error(const char* message) { g_err = message ? message : ""; }
const char* b200reg_version(void) { return "b200reg 0.2 (sm_90a)"; }
size_t b200reg_struct_size(int which) {
  switch (which) {
    case 0: return sizeof(b200reg_gicp_params);
    case 1: return sizeof(b200reg_result);
    case 2: return sizeof(b200reg_quatro_params);
    case 3: return sizeof(b200reg_quatro_info);
    case 4: return sizeof(b200reg_loop_config);
    case 5: return sizeof(b200reg_loop_factor);
    case 6: return sizeof(b200reg_lm_trial);
    case 7: return sizeof(b200reg_lm_case);
    case 8: return sizeof(b200reg_lm_step);
    default: return 0;
  }
}

int b200reg_ctx_create(int device, b200reg_ctx** out) {
  if (!out) return fail(B200REG_EINVAL, "out is NULL");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev)
    return fail(B200REG_ENODEV, "no usable CUDA device (this library has no CPU fallback)");
  CU(cudaSetDevice(device));
  CU(quatro_init_device());
  b200reg_ctx* c = new b200reg_ctx;
  c->device = device;
  struct Undo {  // a failure half way must not leak the context
    b200reg_ctx* c;
    bool ok = false;
    ~Undo() {
      if (!ok) b200reg_ctx_destroy(c);
    }
  } undo{c};
  CU(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
  CU(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  c->stream = c->own_stream;
  cudaMemPoolProps props = {};
  props.allocType = cudaMemAllocationTypePinned;
  props.handleTypes = cudaMemHandleTypeNone;
  props.location.type = cudaMemLocationTypeDevice;
  props.location.id = device;
  CU(cudaMemPoolCreate(&c->pool, &props));
  uint64_t thr = UINT64_MAX;
  CU(cudaMemPoolSetAttribute(c->pool, cudaMemPoolAttrReleaseThreshold, &thr));
  CU(cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device));
  undo.ok = true;
  *out = c;
  return B200REG_OK;
}

int b200reg_ctx_destroy(b200reg_ctx* c) {
  if (!c) return B200REG_OK;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->comm) b200reg_comm_destroy(c);
  lm_arena_free(c);
  if (c->own_stream) cudaStreamDestroy(c->own_stream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->pool) cudaMemPoolDestroy(c->pool);
  delete c;
  return B200REG_OK;
}

int b200reg_ctx_set_stream(b200reg_ctx* c, void* s) {
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  c->stream = s ? (cudaStream_t)s : c->own_stream;
  return B200REG_OK;
}

int b200reg_ctx_synchronize(b200reg_ctx* c) {
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  return B200REG_OK;
}

int64_t b200reg_ctx_launch_count(const b200reg_ctx* c) { return c ? c->launches : 0; }

int b200reg_ctx_set_profiling(b200reg_ctx* c, int enable) {
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  CU(cudaSetDevice(c->device));
  prof_resolve(c);
  c->profiling = enable != 0;
  return B200REG_OK;
}

int b200reg_ctx_reset_profile(b200reg_ctx* c) {
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  prof_resolve(c);
  for (int i = 0; i < NCLS; i++) {
    c->prof_ms[i] = 0;
    c->prof_bytes[i] = 0;
    c->prof_launches[i] = 0;
  }
  return B200REG_OK;
}

int b200reg_ctx_get_profile(b200reg_ctx* c, int cls, const char** name, double* ms, double* algo_bytes, int64_t* launches) {
  if (!c || cls < 0 || cls >= NCLS) return fail(B200REG_EINVAL, "bad class");
  CU(cudaSetDevice(c->device));
  prof_resolve(c);
  if (name) *name = kClassNames[cls];
  if (ms) *ms = c->prof_ms[cls];
  if (algo_bytes) *algo_bytes = c->prof_bytes[cls];
  if (launches) *launches = c->prof_launches[cls];
  return B200REG_OK;
}

size_t b200reg_cloud_size(const b200reg_cloud* cl) { return cl ? (size_t)cl->dev.n : 0; }

// ------------------------------------------------------------------------------------------
int b200reg_clouds_create(b200reg_ctx* c, int count, const float* const* xyz, const size_t* n, size_t stride_bytes,
                          int on_device, b200reg_cloud** out) {
  return clouds_create(c, count, xyz, n, stride_bytes, on_device, false, out);
}

}  // extern "C"

int b200::clouds_create(b200reg_ctx* c, int count, const float* const* xyz, const size_t* n, size_t stride_bytes, int on_device,
                        bool keep_intensity, b200reg_cloud** out) {
  if (!c || count <= 0 || !xyz || !n || !out) return fail(B200REG_EINVAL, "bad argument");
  if (stride_bytes < 12 || stride_bytes % 4) return fail(B200REG_EINVAL, "stride_bytes must be a multiple of 4, >= 12");
  for (int i = 0; i < count; i++)
    if (!xyz[i] || n[i] == 0 || n[i] > (size_t)(1u << 26)) return fail(B200REG_EINVAL, "empty or oversized cloud");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  std::vector<CloudDev> descs(count);
  int max_n = 0;
  for (int i = 0; i < count; i++) out[i] = nullptr;
  CloudBag bag(c);  // a failure half way must not leak the clouds already created
  // sort work memory and AABB arrival flags of the whole batch: ONE allocation, ONE memset
  std::vector<size_t> z_ws(count), z_fl(count);
  Layout zl;
  for (int i = 0; i < count; i++) {
    z_ws[i] = zl.take(radix_sort_ws_bytes((int)n[i], 30));
    z_fl[i] = zl.take((size_t)std::max((int)n[i] - 1, 1) * 4);
  }
  char* zeroed = nullptr;
  CU(scratch.alloc((void**)&zeroed, zl.size));
  CU(cudaMemsetAsync(zeroed, 0, zl.size, s));
  for (int i = 0; i < count; i++) {
    b200reg_cloud* cl = new b200reg_cloud;
    bag.cl.push_back(cl);
    CloudDev& d = cl->dev;
    d.n = (int)n[i];
    d.root_ref = d.n <= LEAF ? leaf_ref(0, d.n) : 0;
    d.raw_stride = (int)(stride_bytes / 4);
    const size_t nn = (size_t)std::max(d.n - 1, 1);
    // persistent slab
    Layout pl;
    const size_t o_pts = pl.take((size_t)d.n * sizeof(float4)), o_tn = pl.take(4 * nn * sizeof(float4)),
                 o_cov = pl.take((size_t)6 * d.n * sizeof(double)), o_rank = pl.take((size_t)d.n * sizeof(int));
    const size_t o_int = keep_intensity ? pl.take((size_t)d.n * sizeof(float)) : 0;
    char* slab = nullptr;
    CU(cudaMallocFromPoolAsync((void**)&slab, pl.size, c->pool, s));
    cl->slab = slab;
    if (keep_intensity) cl->inten = (float*)(slab + o_int);
    d.pts = (float4*)(slab + o_pts);
    d.tnodes = (float4*)(slab + o_tn);
    d.cov = (double*)(slab + o_cov);
    d.rank = (int*)(slab + o_rank);
    d.nrm = nullptr;
    d.spfh = nullptr;
    d.fpfh = nullptr;
    d.fproj = nullptr;
    d.fpfh_s = nullptr;
    d.fproj_s = nullptr;
    d.ftile = nullptr;
    d.fcode_s = nullptr;
    // temporary slab (sort buffers, tree scratch, bbox partials, and the raw records when uploading)
    Layout tl;
    const size_t t_k0 = tl.take((size_t)d.n * 4), t_k1 = tl.take((size_t)d.n * 4), t_v0 = tl.take((size_t)d.n * 4),
                 t_v1 = tl.take((size_t)d.n * 4), t_i = tl.take(nn * sizeof(int4)), t_pn = tl.take(nn * 4),
                 t_pl = tl.take((size_t)d.n * 4), t_b = tl.take(6 * BBOX_BLOCKS * sizeof(float)),
                 t_raw = tl.take(on_device ? 0 : (size_t)d.n * stride_bytes);
    char* tmp = nullptr;
    CU(scratch.alloc((void**)&tmp, tl.size));
    d.keys[0] = (uint32_t*)(tmp + t_k0);
    d.keys[1] = (uint32_t*)(tmp + t_k1);
    d.vals[0] = (uint32_t*)(tmp + t_v0);
    d.vals[1] = (uint32_t*)(tmp + t_v1);
    d.hist = (uint32_t*)(zeroed + z_ws[i]);
    d.flags = (uint32_t*)(zeroed + z_fl[i]);
    d.info = (int4*)(tmp + t_i);
    d.parent_node = (int*)(tmp + t_pn);
    d.parent_leaf = (int*)(tmp + t_pl);
    d.bbox = (float*)(tmp + t_b);
    if (on_device) {
      d.raw = xyz[i];
    } else {
      CU(cudaMemcpyAsync(tmp + t_raw, xyz[i], (size_t)d.n * stride_bytes, cudaMemcpyHostToDevice, s));
      d.raw = (const float*)(tmp + t_raw);
    }
    descs[i] = d;
    max_n = std::max(max_n, d.n);
  }
  CloudDev* d_descs = nullptr;
  CU(scratch.upload(&d_descs, descs.data(), sizeof(CloudDev) * count));
  {
    ProfScope ps(c, CLS_BUILD);
    c->launches += launch_index_build(d_descs, count, max_n, s);
    for (int i = 0; i < count; i++) c->prof_bytes[CLS_BUILD] += 36.0 * descs[i].n;  // SURVEY §8(d) K1
  }
  CU(cudaGetLastError());
  if (keep_intensity) {  // from the raw records, while they are still there
    std::vector<float*> inten(count);
    for (int i = 0; i < count; i++) inten[i] = bag.cl[i]->inten;
    float** d_inten = nullptr;
    CU(scratch.upload(&d_inten, inten.data(), sizeof(float*) * count));
    launch_gather_intensity(d_descs, count, max_n, d_inten, s);
    c->launches++;
    CU(cudaGetLastError());
  }
  for (b200reg_cloud* cl : bag.cl) {  // the temporaries are gone once the build has run
    CloudDev& d = cl->dev;
    d.raw = nullptr;
    d.keys[0] = d.keys[1] = d.vals[0] = d.vals[1] = d.hist = d.flags = nullptr;
    d.info = nullptr;
    d.parent_node = d.parent_leaf = nullptr;
    d.bbox = nullptr;
  }
  if (!on_device) CU(cudaStreamSynchronize(s));  // host buffers have been consumed when the call returns (pinned or not)
  std::copy(bag.cl.begin(), bag.cl.end(), out);  // the caller owns the clouds from here on
  bag.cl.clear();
  return B200REG_OK;
}

extern "C" {

int b200reg_cloud_destroy(b200reg_ctx* c, b200reg_cloud* cl) {
  if (!cl) return B200REG_OK;
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  CU(cudaSetDevice(c->device));
  if (cl->slab) CU(cudaFreeAsync(cl->slab, c->stream));
  if (cl->fslab) CU(cudaFreeAsync(cl->fslab, c->stream));
  delete cl;
  return B200REG_OK;
}

// The plain entry point keeps its 1..32 range; b200reg_clouds_covariances_ex takes any k >= 1.
int b200reg_clouds_covariances(b200reg_ctx* c, int count, b200reg_cloud* const* clouds, int k) {
  if (k < 1 || k > 32) return fail(B200REG_EINVAL, "k_correspondences must be in 1..32 (b200reg_clouds_covariances_ex takes any k >= 1)");
  return b200reg_clouds_covariances_ex(c, count, clouds, k, 3);
}

int b200reg_clouds_covariances_ex(b200reg_ctx* c, int count, b200reg_cloud* const* clouds, int k, int method) {
  if (!c || count <= 0 || !clouds) return fail(B200REG_EINVAL, "bad argument");
  if (method < 0 || method > 4) return fail(B200REG_EINVAL, "regularization must be 0..4 (NONE, MIN_EIG, NORMALIZED_MIN_EIG, PLANE, FROBENIUS)");
  if (k < 1) return fail(B200REG_EINVAL, "k_correspondences must be >= 1");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  std::vector<CloudDev> descs;
  int max_n = 0;
  for (int i = 0; i < count; i++) {
    if (!clouds[i]) return fail(B200REG_EINVAL, "NULL cloud");
    if (clouds[i]->has_cov && !clouds[i]->cov_user && clouds[i]->cov_k == k && clouds[i]->cov_method == method) continue;
    bool dup = false;
    for (int j = 0; j < i; j++) dup |= clouds[j] == clouds[i];
    if (dup) continue;
    descs.push_back(clouds[i]->dev);
    max_n = std::max(max_n, clouds[i]->dev.n);
  }
  if (descs.empty()) return B200REG_OK;
  CloudDev* d_descs = nullptr;
  CU(scratch.upload(&d_descs, descs.data(), sizeof(CloudDev) * descs.size()));
  unsigned long long* d_slab = nullptr;  // lists beyond shared memory (k > 256): one per warp, bounded (launchers.cuh)
  if (const size_t slab = covariance_large_slab_bytes((int)descs.size(), max_n, k)) CU(scratch.alloc((void**)&d_slab, slab));
  {
    ProfScope ps(c, CLS_COV);
    int l = launch_covariances(d_descs, (int)descs.size(), max_n, k, method, d_slab, s);
    if (l < 0) return fail(B200REG_EINVAL, "unsupported k");
    c->launches += l;
    for (auto& d : descs) c->prof_bytes[CLS_COV] += 64.0 * d.n;  // SURVEY §8(d) K2
  }
  CU(cudaGetLastError());
  for (int i = 0; i < count; i++) {
    clouds[i]->has_cov = true;
    clouds[i]->cov_user = false;
    clouds[i]->cov_k = k;
    clouds[i]->cov_method = method;
  }
  return B200REG_OK;
}

int b200reg_set_covariances(b200reg_ctx* c, b200reg_cloud* cl, const double* cov9, size_t n) {
  if (!c || !cl || !cov9) return fail(B200REG_EINVAL, "bad argument");
  if (n != (size_t)cl->dev.n) return fail(B200REG_EINVAL, "covariance count differs from the cloud size");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  double* d_cov9 = nullptr;
  CU(scratch.upload(&d_cov9, cov9, n * 72));
  launch_set_covariances(cl->dev, d_cov9, s);
  c->launches++;
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(s));  // the caller's buffer may go away
  cl->has_cov = true;
  cl->cov_user = true;
  return B200REG_OK;
}

int b200reg_transform_cloud(b200reg_ctx* c, const b200reg_cloud* cl, const float* Tf16, float* out_xyz) {
  if (!c || !cl || !Tf16 || !out_xyz) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  float* d_T = nullptr;
  float* d_out = nullptr;
  CU(scratch.upload(&d_T, Tf16, 64));
  CU(scratch.alloc((void**)&d_out, (size_t)cl->dev.n * 12));
  launch_transform_out(cl->dev, d_T, d_out, s);
  c->launches++;
  CU(cudaMemcpyAsync(out_xyz, d_out, (size_t)cl->dev.n * 12, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

// ---- debug taps --------------------------------------------------------------------------
static int knn_impl(b200reg_ctx* c, const b200reg_cloud* cl, const float* queries, size_t nq, size_t qstride_bytes, int k,
                    int32_t* idx_out, float* d2_out, int brute);

int b200reg_knn(b200reg_ctx* c, const b200reg_cloud* cl, const float* queries, size_t nq, size_t qstride_bytes, int k,
                int32_t* idx_out, float* d2_out) {
  return knn_impl(c, cl, queries, nq, qstride_bytes, k, idx_out, d2_out, 0);
}

int b200reg_knn_bruteforce(b200reg_ctx* c, const b200reg_cloud* cl, const float* queries, size_t nq, size_t qstride_bytes, int k,
                           int32_t* idx_out, float* d2_out) {
  return knn_impl(c, cl, queries, nq, qstride_bytes, k, idx_out, d2_out, 1);
}

static int knn_large(b200reg_ctx* c, const b200reg_cloud* cl, const float* queries, size_t nq, size_t qstride_bytes, int k,
                     int32_t* idx_out, float* d2_out);

static int knn_impl(b200reg_ctx* c, const b200reg_cloud* cl, const float* queries, size_t nq, size_t qstride_bytes, int k,
                    int32_t* idx_out, float* d2_out, int brute) {
  if (!c || !cl || !queries || nq == 0 || k <= 0 || !idx_out || !d2_out || qstride_bytes < 12 || qstride_bytes % 4)
    return fail(B200REG_EINVAL, "bad argument (k must be >= 1, qstride_bytes a multiple of 4, >= 12)");
  if (brute && k > 32) return fail(B200REG_EINVAL, "bad argument (the brute-force k-NN takes k in 1..32)");
  if (k > 32) return knn_large(c, cl, queries, nq, qstride_bytes, k, idx_out, d2_out);
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  float* d_q = nullptr;
  int* d_idx = nullptr;
  float* d_d2 = nullptr;
  CU(scratch.upload(&d_q, queries, nq * qstride_bytes));
  CU(scratch.alloc((void**)&d_idx, nq * k * 4));
  CU(scratch.alloc((void**)&d_d2, nq * k * 4));
  if (launch_knn_queries(cl->dev, d_q, (int)nq, (int)(qstride_bytes / 4), k, d_idx, d_d2, s, brute) < 0)
    return fail(B200REG_EINVAL, "unsupported k");
  c->launches++;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(idx_out, d_idx, nq * k * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(d2_out, d_d2, nq * k * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

// k > 32 (knn_large.cu).  The queries run in chunks of consecutive rows holding at most max(kKnnChunk, cloud size) result
// entries (or one row, if k is larger), so the device copy of the output -- and, for lists longer than KL_SMEM_K, the
// per-query slab -- stays bounded whatever nq * k is; each chunk's rows are copied to the caller's buffers.
// k >= n: every point is a neighbour, and the sorted radius search with r2 = +inf lists exactly the points the kernel would
// (d2 < +inf, ascending (d2, index)); its compact rows are spread to stride k and padded with (-1, FLT_MAX) here.
static constexpr int64_t kKnnChunk = int64_t(1) << 23;

static int knn_large(b200reg_ctx* c, const b200reg_cloud* cl, const float* queries, size_t nq, size_t qstride_bytes, int k,
                     int32_t* idx_out, float* d2_out) {
  const int n = cl->dev.n;
  if (k >= n) {
    std::vector<int64_t> off(nq + 1);
    if (const int rc = b200reg_radius_search(c, cl, queries, nq, qstride_bytes, HUGE_VAL, 1, off.data(), nq * (size_t)k, idx_out,
                                             d2_out))
      return rc;
    for (size_t i = nq; i-- > 0;) {  // last row first: row i's source [off[i], off[i+1]) lies at or below its target i * k
      const size_t cnt = (size_t)(off[i + 1] - off[i]);
      std::memmove(idx_out + i * k, idx_out + off[i], cnt * 4);
      std::memmove(d2_out + i * k, d2_out + off[i], cnt * 4);
      std::fill(idx_out + i * k + cnt, idx_out + (i + 1) * k, -1);
      std::fill(d2_out + i * k + cnt, d2_out + (i + 1) * k, 3.402823466e+38f);
    }
    return B200REG_OK;
  }
  const int qs = (int)(qstride_bytes / 4);
  const size_t rows = (size_t)std::max<int64_t>(1, std::max<int64_t>(kKnnChunk, n) / k);
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  ProfScope ps(c, CLS_MISC);
  float* d_q = nullptr;
  int* d_idx = nullptr;
  float* d_d2 = nullptr;
  unsigned long long* d_slab = nullptr;
  const size_t cap = std::min(rows, nq) * (size_t)k;
  CU(scratch.upload(&d_q, queries, nq * qstride_bytes));
  CU(scratch.alloc((void**)&d_idx, cap * 4));
  CU(scratch.alloc((void**)&d_d2, cap * 4));
  if (k > KL_SMEM_K) CU(scratch.alloc((void**)&d_slab, cap * 8));
  for (size_t r0 = 0; r0 < nq; r0 += rows) {
    const size_t nr = std::min(rows, nq - r0);
    c->launches += launch_knn_large(cl->dev, d_q + r0 * qs, (int)nr, qs, k, d_slab, d_idx, d_d2, s);
    CU(cudaGetLastError());
    c->prof_bytes[CLS_MISC] += 16.0 * nr + 8.0 * nr * k;
    CU(cudaMemcpyAsync(idx_out + r0 * k, d_idx, nr * k * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(d2_out + r0 * k, d_d2, nr * k * 4, cudaMemcpyDeviceToHost, s));
  }
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

// Fixed-radius search (radius.cu).  The neighbours of the queries are produced chunk by chunk: a chunk is a run of
// consecutive caller queries with at most kRadiusChunk neighbours (or one query with more), so device memory stays bounded
// by max(kRadiusChunk, cloud size) entries, 28 bytes each, whatever the total, and each chunk's block of the output is
// contiguous on the host.
static constexpr int64_t kRadiusChunk = int64_t(1) << 23;

int b200reg_radius_search(b200reg_ctx* c, const b200reg_cloud* cl, const float* queries, size_t nq, size_t qstride_bytes,
                          double sq_radius, int sorted, int64_t* offsets_out, size_t capacity, int32_t* idx_out, float* d2_out) {
  if (!c || !cl || !queries || !offsets_out || nq == 0 || nq >= ((size_t)1 << 30) || qstride_bytes < 12 || qstride_bytes % 4)
    return fail(B200REG_EINVAL, "bad argument (nq must be 1..2^30-1, qstride_bytes a multiple of 4, >= 12)");
  if ((idx_out == nullptr) != (d2_out == nullptr)) return fail(B200REG_EINVAL, "idx_out and d2_out: both or neither (count only)");
  const float r2 = (float)sq_radius;  // RadiusResultSet<float, int>(radius): converted to float, NOT squared
  const int n = (int)nq, qs = (int)(qstride_bytes / 4);
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  ProfScope ps(c, CLS_MISC);
  float* d_q = nullptr;
  uint32_t *qk[2], *qv[2];
  int* d_cnt = nullptr;
  int64_t* d_off = nullptr;
  char* d_ws = nullptr;  // zeroed sort work memory: query order, then (several chunks) chunk grouping
  void* d_scan = nullptr;
  const size_t sort_ws = radix_sort_ws_bytes(n, 30);
  CU(scratch.upload(&d_q, queries, nq * qstride_bytes));
  for (int b = 0; b < 2; b++) {
    CU(scratch.alloc((void**)&qk[b], nq * 4));
    CU(scratch.alloc((void**)&qv[b], nq * 4));
  }
  CU(scratch.alloc((void**)&d_cnt, nq * 4));
  CU(scratch.alloc((void**)&d_off, (nq + 1) * 8));
  CU(scratch.alloc((void**)&d_scan, radius_scan_ws_bytes(n)));
  CU(scratch.alloc((void**)&d_ws, 2 * sort_ws));
  CU(cudaMemsetAsync(d_ws, 0, 2 * sort_ws, s));
  // Stable sort of (k0, v0) with k1 / v1 as the ping-pong halves; *out = whichever value buffer holds the result.  The radix
  // sort reads its arrays through a device-side descriptor (only n / keys / vals / hist are used).
  auto sort = [&](int m, uint32_t* k0, uint32_t* k1, uint32_t* v0, uint32_t* v1, void* hist, int key_bits, uint32_t** out) -> int {
    CloudDev d = {};
    d.n = m;
    d.keys[0] = k0; d.keys[1] = k1;
    d.vals[0] = v0; d.vals[1] = v1;
    d.hist = (uint32_t*)hist;
    CloudDev* dd = nullptr;
    CU(scratch.upload(&dd, &d, sizeof(d)));
    c->launches += launch_radix_sort(dd, 1, m, key_bits, s);
    *out = radix_sort_result_buf(key_bits) ? v1 : v0;
    return B200REG_OK;
  };
  // 1. queries in the cloud's Morton order, 2. counts, 3. offsets
  c->launches += launch_radius_query_keys(cl->dev, d_q, n, qs, qk[0], qv[0], s);
  uint32_t* order = nullptr;
  if (const int rc = sort(n, qk[0], qk[1], qv[0], qv[1], d_ws, 30, &order)) return rc;
  c->launches += launch_radius_count(cl->dev, d_q, qs, order, n, r2, d_cnt, s);
  c->launches += launch_radius_scan(d_cnt, n, d_off, d_scan, s);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(offsets_out, d_off, (nq + 1) * 8, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  const int64_t total = offsets_out[n];
  if (!idx_out || total == 0) return B200REG_OK;
  if ((uint64_t)total > (uint64_t)capacity)
    return fail(B200REG_ESTATE, "radius search found " + std::to_string(total) + " neighbours, capacity is " + std::to_string(capacity));
  // 4. chunks of consecutive caller queries
  std::vector<int> starts{0};
  int64_t max_entries = 0;
  for (int i = 0, a = 0; i <= n; i++) {
    if (i == n || (offsets_out[i + 1] - offsets_out[a] > kRadiusChunk && i > a)) {
      max_entries = std::max(max_entries, offsets_out[i] - offsets_out[a]);
      if (i == n) break;
      starts.push_back(i);
      a = i;
    }
  }
  const int nchunks = (int)starts.size();
  starts.push_back(n);
  if (max_entries >= (int64_t)INT32_MAX) return fail(B200REG_EINVAL, "one query has 2^31 or more neighbours");
  if (nchunks > 1) {  // group the Morton-ordered queries by chunk (stable: Morton order inside each chunk)
    int* d_starts = nullptr;
    CU(scratch.upload(&d_starts, starts.data(), starts.size() * 4));
    uint32_t* other = order == qv[0] ? qv[1] : qv[0];
    c->launches += launch_radius_chunk_keys(order, n, d_starts, nchunks, qk[0], other, s);
    if (const int rc = sort(n, qk[0], qk[1], other, order, d_ws + sort_ws, 30, &order)) return rc;
  }
  // per chunk: entries, three sort passes' key / value ping-pong, three zeroed sort work areas
  const size_t m = (size_t)max_entries;
  int* e_idx = nullptr;
  float* e_d2 = nullptr;
  uint32_t *e_seg = nullptr, *K[2], *V[2];
  char* ews = nullptr;
  const size_t ews1 = radix_sort_ws_bytes((int)m, 32);
  CU(scratch.alloc((void**)&e_idx, m * 4));
  CU(scratch.alloc((void**)&e_d2, m * 4));
  CU(scratch.alloc((void**)&e_seg, m * 4));
  for (int b = 0; b < 2; b++) {
    CU(scratch.alloc((void**)&K[b], m * 4));
    CU(scratch.alloc((void**)&V[b], m * 4));
  }
  CU(scratch.alloc((void**)&ews, 3 * ews1));
  for (int ci = 0; ci < nchunks; ci++) {
    RadiusChunk ch;
    ch.q0 = ch.r0 = starts[ci];
    ch.nr = starts[ci + 1] - starts[ci];
    ch.base = offsets_out[ch.q0];
    const int me = (int)(offsets_out[starts[ci + 1]] - ch.base);
    if (me == 0) continue;
    ch.e_idx = e_idx; ch.e_d2 = e_d2; ch.e_seg = e_seg; ch.keys = K[0]; ch.vals = V[0];
    CU(cudaMemsetAsync(ews, 0, 3 * ews1, s));
    c->launches += launch_radius_fill(cl->dev, d_q, qs, order, r2, d_off, ch, s);
    // stable LSD passes: original index, (sorted) d2, query -> per query ascending index or ascending (d2, index)
    uint32_t* cur = nullptr;
    if (const int rc = sort(me, K[0], K[1], V[0], V[1], ews, 30, &cur)) return rc;
    if (sorted) {  // d2 >= 0 and never NaN here: its bit pattern orders like the value
      c->launches += launch_radius_rekey(cur, me, (const uint32_t*)e_d2, K[0], s);
      if (const int rc = sort(me, K[0], K[1], cur, cur == V[0] ? V[1] : V[0], ews + ews1, 32, &cur)) return rc;
    }
    c->launches += launch_radius_rekey(cur, me, e_seg, K[0], s);
    if (const int rc = sort(me, K[0], K[1], cur, cur == V[0] ? V[1] : V[0], ews + 2 * ews1, 30, &cur)) return rc;
    c->launches += launch_radius_gather(cur, me, e_idx, e_d2, (int*)K[0], (float*)K[1], s);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(idx_out + ch.base, K[0], (size_t)me * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(d2_out + ch.base, K[1], (size_t)me * 4, cudaMemcpyDeviceToHost, s));
  }
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

int b200reg_get_covariances(b200reg_ctx* c, const b200reg_cloud* cl, double* cov9_out) {
  if (!c || !cl || !cov9_out) return fail(B200REG_EINVAL, "bad argument");
  if (!cl->has_cov) return fail(B200REG_ESTATE, "covariances not computed");
  CU(cudaSetDevice(c->device));
  const int n = cl->dev.n;
  std::vector<double> cov((size_t)n * 6);
  std::vector<int> orig;
  CU(cudaMemcpyAsync(cov.data(), cl->dev.cov, (size_t)n * 48, cudaMemcpyDeviceToHost, c->stream));
  if (const int rc = sorted_to_original(c, cl->dev, orig)) return rc;
  for (int p = 0; p < n; p++) {
    const double* a = &cov[(size_t)p * 6];
    double* m = &cov9_out[(size_t)orig[p] * 9];
    m[0] = a[0]; m[1] = a[1]; m[2] = a[2];
    m[3] = a[1]; m[4] = a[3]; m[5] = a[4];
    m[6] = a[2]; m[7] = a[4]; m[8] = a[5];
  }
  return B200REG_OK;
}

int b200reg_cloud_points(b200reg_ctx* c, const b200reg_cloud* cl, float* xyz_out) {
  if (!c || !cl || !xyz_out) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  std::vector<int> orig;
  std::vector<float4> pts;
  if (const int rc = sorted_to_original(c, cl->dev, orig, &pts)) return rc;
  for (int p = 0; p < cl->dev.n; p++) {
    xyz_out[3 * (size_t)orig[p]] = pts[p].x;
    xyz_out[3 * (size_t)orig[p] + 1] = pts[p].y;
    xyz_out[3 * (size_t)orig[p] + 2] = pts[p].z;
  }
  return B200REG_OK;
}

// ---- the one collective: all-gather of the result records over NCCL (SURVEY §8(e)) ------------------------
namespace {
struct NcclApi {
  void* h = nullptr;
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  std::string err;
};
NcclApi* nccl_api() {  // loaded once per process; a process that already holds libnccl.so.2 (torch) shares that copy
  static NcclApi api;
  static bool tried = false;
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  if (tried) return &api;
  tried = true;
  // 1. a copy this process already holds (e.g. the one a framework bundles and linked first): two NCCL builds under one
  //    soname would starve whichever library loads second of its symbols;  2. $B200REG_NCCL_LIB (the Python binding points
  //    it at the pip-bundled libnccl so that a LATER `import torch` finds the version it was built against);  3. the system's.
  api.h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
  const char* names[] = {getenv("B200REG_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    if (api.h) break;
    if (!n || !*n) continue;
    api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
  }
  if (!api.h) {
    api.err = std::string("cannot load libnccl.so.2: ") + dlerror();
    return &api;
  }
  api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(api.h, "ncclGetUniqueId");
  api.CommInitRank = (decltype(api.CommInitRank))dlsym(api.h, "ncclCommInitRank");
  api.CommDestroy = (decltype(api.CommDestroy))dlsym(api.h, "ncclCommDestroy");
  api.AllGather = (decltype(api.AllGather))dlsym(api.h, "ncclAllGather");
  api.GetErrorString = (decltype(api.GetErrorString))dlsym(api.h, "ncclGetErrorString");
  if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather || !api.GetErrorString) {
    api.err = "libnccl.so.2 lacks a required symbol";
    dlclose(api.h);
    api.h = nullptr;
  }
  return &api;
}
}  // namespace
#define NC(call)                                                                                               \
  do {                                                                                                         \
    ncclResult_t _r = (call);                                                                                  \
    if (_r != ncclSuccess) return fail(B200REG_ENCCL, std::string(#call) + ": " + api->GetErrorString(_r)); \
  } while (0)

static_assert(sizeof(ncclUniqueId) == B200REG_UNIQUE_ID_BYTES, "ncclUniqueId is 128 bytes");

int b200reg_comm_unique_id(void* id_out) {
  if (!id_out) return fail(B200REG_EINVAL, "id_out is NULL");
  NcclApi* api = nccl_api();
  if (!api->h) return fail(B200REG_ENCCL, api->err);
  ncclUniqueId id;
  NC(api->GetUniqueId(&id));
  memcpy(id_out, &id, sizeof(id));
  return B200REG_OK;
}

int b200reg_comm_init(b200reg_ctx* c, const void* id128, int rank, int world) {
  if (!c || !id128 || world < 1 || rank < 0 || rank >= world) return fail(B200REG_EINVAL, "bad argument");
  if (c->comm) return fail(B200REG_ESTATE, "the context already has a communicator");
  NcclApi* api = nccl_api();
  if (!api->h) return fail(B200REG_ENCCL, api->err);
  CU(cudaSetDevice(c->device));
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  NC(api->CommInitRank(&c->comm, world, id, rank));
  c->rank = rank;
  c->world = world;
  return B200REG_OK;
}

int b200reg_comm_destroy(b200reg_ctx* c) {
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  if (!c->comm) return B200REG_OK;
  NcclApi* api = nccl_api();
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  ncclComm_t comm = c->comm;
  c->comm = nullptr;
  c->rank = -1;
  c->world = 1;
  NC(api->CommDestroy(comm));
  return B200REG_OK;
}

int b200reg_comm_rank(const b200reg_ctx* c) { return c ? c->rank : -1; }
int b200reg_comm_world(const b200reg_ctx* c) { return c ? c->world : 1; }

int b200reg_allgather_results(b200reg_ctx* c, const b200reg_result* local, int n_local, b200reg_result* all_out) {
  if (!c || !local || n_local <= 0 || !all_out) return fail(B200REG_EINVAL, "bad argument");
  const size_t bytes = sizeof(b200reg_result) * (size_t)n_local;
  if (!c->comm || c->world == 1) {
    if (all_out != local) memcpy(all_out, local, bytes);
    return B200REG_OK;
  }
  NcclApi* api = nccl_api();
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  char *d_local = nullptr, *d_all = nullptr;
  CU(scratch.upload(&d_local, local, bytes));
  CU(scratch.alloc((void**)&d_all, bytes * c->world));
  NC(api->AllGather(d_local, d_all, bytes, ncclChar, c->comm, s));
  CU(cudaMemcpyAsync(all_out, d_all, bytes * c->world, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

}  // extern "C"
