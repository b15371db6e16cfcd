// api.cuh -- what the host files of the C ABI share (api.cu, api_gicp.cu, api_quatro.cu, api_keyframes.cu): the context and
// cloud objects, error reporting, profiling scopes, stream-ordered scratch memory and the helpers more than one area uses.
// Host orchestration only; every arithmetic step of the path runs in the kernels of index_build.cu / gicp.cu / quatro.cu /
// assemble.cu.  There is no CPU fallback anywhere in this library.
#pragma once
#include <cuda_runtime.h>
#include <nccl.h>  // types only: the library is dlopen()ed in b200reg_comm_*

#include <cstddef>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200reg.h"
#include "internal.cuh"
#include "launchers.cuh"

using namespace b200;

struct KfJob;  // a batch-driver job over the keyframe store (api_keyframes.cu)

namespace b200 {
int fail(int code, const std::string& msg);  // sets b200reg_last_error() and returns code
}  // namespace b200
#define CU(call)                                                                                              \
  do {                                                                                                        \
    cudaError_t _e = (call);                                                                                  \
    if (_e != cudaSuccess)                                                                                    \
      return fail(B200REG_ECUDA, std::string(#call) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + \
                                     std::to_string(__LINE__));                                               \
  } while (0)

enum { CLS_BUILD = 0, CLS_COV = 1, CLS_STEP = 2, CLS_MISC = 3, CLS_FPFH = 4, CLS_MATCH = 5, CLS_SEARCH = 6, CLS_ACCUM = 7, CLS_CTRL = 8, NCLS = 9 };

struct b200reg_ctx {
  int device = 0;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;  // H2D uploads of later chunks overlap the compute of earlier ones
  cudaMemPool_t pool = nullptr;        // per-context pool: reuse never adds dependencies on another context's streams
  int pipeline_chunks = 4;
  int sm_count = 132;
  // persistent arena of the batched LM solve: every kernel argument of the solve's CUDA graph points in here, so the graph is
  // instantiated once and re-launched by every b200reg_gicp_align call until a larger batch makes the arena grow
  struct LmArena {
    int cap = 0;
    PairDev* d_pairs = nullptr;
    PairState* d_states = nullptr;
    LmSched* d_sched = nullptr;  // header + slots[cap]
    double* d_guess = nullptr;   // [16 * cap]
    LmCall* d_call = nullptr;
    LmCall* h_call = nullptr;    // pinned staging
    PairState* h_states = nullptr;  // pinned read-back
    LmGraph graph;
  } lm;
  // LM trace of the most recent call that ran the LM solve (b200reg_ctx_set_lm_trace / b200reg_lm_trace), CSR over the pairs
  // of that call, on the host
  struct LmTrace {
    bool enabled = false;
    bool valid = false;  // false before a traced solve and after an untraced one
    std::vector<int64_t> offsets;  // pairs + 1
    std::vector<b200reg_lm_trial> trials;
  } lm_trace;
  // loop clouds (b200reg_ctx_set_loop_clouds / b200reg_loop_clouds): the kinds the capturing calls record, and the clouds of
  // the most recent such call, CSR over its pairs per kind (slot = log2 of the kind's bit), on the host
  struct LoopClouds {
    int mask = 0;
    int stored = 0;  // kinds held; 0 before a capturing call and after an uncaptured one
    std::vector<int64_t> offsets[4];  // pairs + 1 each
    std::vector<float4> pts[4];       // (x, y, z, intensity)
  } loop_clouds;
  // Quatro matches (b200reg_ctx_set_quatro_matches / b200reg_quatro_matches) of the most recent call that reached the Quatro
  // stage with recording on, CSR over its pairs, on the host.  `words` holds four blocks over all `total` matches, as the
  // capture slab does: corr (2 per match), inlier (1), src xyz (3 float bits), dst xyz (3 float bits)
  struct QuatroMatches {
    bool enabled = false;
    bool valid = false;  // false before a recording call, after one that did not record and after one that failed
    std::vector<int64_t> offsets;  // pairs + 1
    std::vector<int32_t> words;    // 9 per match
  } quatro_matches;
  // residuals (b200reg_ctx_set_residuals / b200reg_residuals) of the most recent call that ran the fine stage with recording
  // on, CSR over its pairs, on the host: per source point in original order, the fitness pass's nearest target point
  // (original index) and fp32 squared distance
  struct Residuals {
    bool enabled = false;
    bool valid = false;  // false before a recording call, after one that did not record and after one that failed
    std::vector<int64_t> offsets;  // pairs + 1
    std::vector<int32_t> nn;
    std::vector<float> d2;
    int32_t* slab = nullptr;  // device rows reserved by the call in flight (ResidualSlab): nn block, then d2 block
    size_t slab_points = 0;
  } residuals;
  // the path's one collective (b200reg_comm_*): NCCL communicator of this rank
  ncclComm_t comm = nullptr;
  int rank = -1, world = 1;
  int64_t launches = 0;
  // optional per-kernel-family timing with CUDA events on the launching stream
  bool profiling = false;
  struct Span { int cls; cudaEvent_t a, b; };
  std::vector<Span> pending;
  std::vector<cudaEvent_t> free_events;
  double prof_ms[NCLS] = {0};
  double prof_bytes[NCLS] = {0};
  int64_t prof_launches[NCLS] = {0};
};

struct b200reg_cloud {
  CloudDev dev;            // device pointers + sizes
  void* slab = nullptr;    // persistent allocation (pts, tnodes, cov, rank)
  void* fslab = nullptr;   // Quatro features (nrm, spfh, fpfh), allocated on demand
  bool has_cov = false;
  bool cov_user = false;   // set by b200reg_set_covariances: never recomputed on demand (nano_gicp_impl.hpp:162-167)
  int cov_k = 0;
  int cov_method = 3;
  bool has_fpfh = false;
  double normal_r = 0, fpfh_r = 0;
  float* inten = nullptr;  // [n] intensities, original order, in `slab`: only clouds created inside a capturing call keep them
};

namespace b200 {

cudaEvent_t prof_event(b200reg_ctx* c);
struct ProfScope {  // brackets the kernels launched while it is alive
  b200reg_ctx* c;
  int cls;
  cudaEvent_t a = nullptr;
  int64_t l0;
  ProfScope(b200reg_ctx* c_, int cls_) : c(c_), cls(cls_), l0(c_->launches) {
    if (c->profiling) {
      a = prof_event(c);
      cudaEventRecord(a, c->stream);
    }
  }
  ~ProfScope() {
    if (c->profiling) {
      cudaEvent_t b = prof_event(c);
      cudaEventRecord(b, c->stream);
      c->pending.push_back({cls, a, b});
      c->prof_launches[cls] += c->launches - l0;
    }
  }
};

// Stream-ordered scratch memory with scope lifetime: everything allocated through it is returned to the context's
// pool when the scope ends -- on every path, including the early error returns of the CU() macro.
struct Scratch {
  b200reg_ctx* c;
  std::vector<void*> ptrs;
  explicit Scratch(b200reg_ctx* c_) : c(c_) {}
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  cudaError_t alloc(void** p, size_t bytes) {
    cudaError_t e = cudaMallocFromPoolAsync(p, bytes ? bytes : 16, c->pool, c->stream);
    if (e == cudaSuccess) ptrs.push_back(*p);
    return e;
  }
  // a device copy of `bytes` of host memory, queued on the context's stream
  template <class T>
  cudaError_t upload(T** p, const void* host, size_t bytes) {
    const cudaError_t e = alloc((void**)p, bytes);
    return e == cudaSuccess ? cudaMemcpyAsync(*p, host, bytes, cudaMemcpyHostToDevice, c->stream) : e;
  }
  ~Scratch() {
    for (void* p : ptrs) cudaFreeAsync(p, c->stream);
  }
};

// scope guard: cloud handles created inside a call are released on EVERY exit path (the CU() macro returns early)
struct CloudBag {
  b200reg_ctx* c;
  std::vector<b200reg_cloud*> cl;
  explicit CloudBag(b200reg_ctx* c_) : c(c_) {}
  ~CloudBag() {
    for (b200reg_cloud* p : cl) b200reg_cloud_destroy(c, p);
  }
};

// Sub-buffers carved out of one allocation, each starting at a 256-byte boundary: take() returns the offset of the next
// one, size is what the whole allocation needs.
struct Layout {
  size_t size = 0;
  size_t take(size_t bytes) {
    const size_t o = size;
    size = (size + bytes + 255) / 256 * 256;
    return o;
  }
};

// The buffers of a radix sort (SortDev) of n keys: keys[2] / vals[2] from `bufs`, the work memory from `zeroed`, a Layout
// whose allocation the caller zeroes (it may be `bufs` itself).  `sorts` > 1 reserves one work area per sort that runs
// over the same buffers; bind(..., k) gives the descriptor with area k.  Offsets first, pointers at bind().
struct SortLayout {
  int n;
  size_t ws;  // bytes of one work area
  size_t o_keys[2], o_vals[2], o_hist;
  SortLayout(Layout& bufs, Layout& zeroed, int n_, int key_bits, int sorts = 1) : n(n_), ws(radix_sort_ws_bytes(n_, key_bits)) {
    for (int b = 0; b < 2; b++) o_keys[b] = bufs.take((size_t)n * 4);
    for (int b = 0; b < 2; b++) o_vals[b] = bufs.take((size_t)n * 4);
    o_hist = zeroed.take(sorts * ws);
  }
  SortDev bind(char* bufs, char* zeroed, int k = 0) const {
    SortDev d;
    d.n = n;
    for (int b = 0; b < 2; b++) {
      d.keys[b] = (uint32_t*)(bufs + o_keys[b]);
      d.vals[b] = (uint32_t*)(bufs + o_vals[b]);
    }
    d.hist = (uint32_t*)(zeroed + o_hist + k * ws);
    return d;
  }
};

// RegistrationOutput's defaults (loop_closure.h:64-70): identity transforms, score_ = DBL_MAX, not valid
b200reg_result default_result();

// b200reg_clouds_create; keep_intensity: each cloud also keeps the intensities of its records (b200reg_cloud::inten);
// keys_out (b200reg_index_tap): n[i] host words per cloud receive its sorted Morton keys before the build's temporaries go
int clouds_create(b200reg_ctx* c, int count, const float* const* xyz, const size_t* n, size_t stride_bytes, int on_device,
                  bool keep_intensity, b200reg_cloud** out, uint32_t* const* keys_out = nullptr);

// The clouds of `count` pairs, built in one batch: the source clouds come first, then the targets.  They go to src_out /
// tgt_out and are owned by `bag`.
int create_pair_clouds(b200reg_ctx* c, int count, const float* const* src_xyz, const size_t* src_n, const float* const* tgt_xyz,
                       const size_t* tgt_n, size_t stride_bytes, int on_device, bool keep_intensity, CloudBag& bag,
                       b200reg_cloud** src_out, b200reg_cloud** tgt_out);

// orig[p] = the original index of the point at sorted position p (the int bits of pts[p].w).  Synchronises the stream, so
// the downloads the caller queued before have landed too.  pts_out, if given, receives the sorted points.
int sorted_to_original(b200reg_ctx* c, const CloudDev& d, std::vector<int>& orig, std::vector<float4>* pts_out = nullptr);

void lm_arena_free(b200reg_ctx* c);  // api_gicp.cu

// b200reg_perform_loop_closure as a job of the batch driver (api_keyframes.cu; batch.cu runs it).  kf_job_create, on the
// submitting thread, refuses what the synchronous call refuses, then copies the arguments, the store's state (keyframe
// count, corrected poses, cloud pointers and sizes) and its latest ingest mark; the store counts the job as in flight
// until the job object is released.  kf_job_run, on a worker, waits on its stream for that mark and runs the same
// attempt as the synchronous call on the worker's context.
int kf_job_create(b200reg_keyframes* kf, int device, int count, const int32_t* query_idx, const int32_t* closest_idx,
                  const b200reg_loop_config* cfg, std::shared_ptr<KfJob>* out);
int kf_job_run(b200reg_ctx* c, KfJob* j, b200reg_result* out, b200reg_quatro_info* quatro_out);

// The stored LM trace belongs to the pairs of the last b200reg_gicp_align.  A caller that ran that solve on a subset of its
// `count` pairs (solve pair k = its pair where[k]; `where` empty when no solve ran) renumbers it to its own pairs; the
// others get no records.  Does nothing but keep the trace invalid when tracing is off.  (api_gicp.cu)
void lm_trace_remap(b200reg_ctx* c, int count, const std::vector<int>& where);

// The copy-out rules of b200reg_lm_trace / b200reg_loop_clouds over one stored trace or set of clouds: a context's, or a
// batch-driver job's (b200reg_batch_lm_trace / b200reg_batch_loop_clouds).  A kind that is not one B200REG_CLOUD_* bit is
// B200REG_EINVAL; a null `tr` / `lc`, an invalid trace or a kind not held is B200REG_ESTATE with the message `none`;
// then the CSR offsets and the capacity rule of include/b200reg.h.  (api_gicp.cu, api_loop_clouds.cu)
int lm_trace_copy(const b200reg_ctx::LmTrace* tr, int64_t* offsets_out, size_t capacity, b200reg_lm_trial* trials_out,
                  const std::string& none);
int loop_clouds_copy(const b200reg_ctx::LoopClouds* lc, int kind, int64_t* offsets_out, size_t capacity, float* xyzi_out,
                     const std::string& none);

// The stored Quatro matches belong to the pairs of the last b200reg_quatro_align.  A caller that ran it on a subset of its
// `count` pairs (Quatro pair k = its pair where[k]; `where` empty when no Quatro stage ran) renumbers them to its own pairs;
// the others get empty rows.  Does nothing but keep them invalid when recording is off.  (api_quatro.cu)
void quatro_matches_remap(b200reg_ctx* c, int count, const std::vector<int>& where);
// The copy-out rules of b200reg_quatro_matches over a context's or a batch-driver job's record (b200reg_batch_quatro_matches):
// a null or invalid record is B200REG_ESTATE with the message `none`; then the CSR offsets and the capacity rule.
int quatro_matches_copy(const b200reg_ctx::QuatroMatches* qm, int64_t* offsets_out, size_t capacity, int32_t* corr_out,
                        int32_t* inlier_out, float* src_xyz_out, float* dst_xyz_out, const std::string& none);

// The stored residuals belong to the pairs of the last b200reg_gicp_align.  A caller that ran that solve on a subset of its
// `count` pairs (solve pair k = its pair where[k]) renumbers them to its own pairs; the others get empty rows.  Does
// nothing but keep them invalid when recording is off.  (api_gicp.cu)
void residuals_remap(b200reg_ctx* c, int count, const std::vector<int>& where);
// The copy-out rules of b200reg_residuals over a context's or a batch-driver job's record (b200reg_batch_residuals): a null
// or invalid record is B200REG_ESTATE with the message `none`; then the CSR offsets and the capacity rule.
int residuals_copy(const b200reg_ctx::Residuals* r, int64_t* offsets_out, size_t capacity, int32_t* nn_out, float* d2_out,
                   const std::string& none);
// The device rows of the residual capture of one b200reg_icp_alignment, b200reg_loop_closure or
// b200reg_perform_loop_closure call, reserved as soon as its source clouds exist, so that a failed allocation costs no
// registration: one row per source point of every pair that can run the fine stage.  The call's b200reg_gicp_align writes
// into them instead of allocating its own.  Returned at the end of the scope; with recording off nothing is allocated.
class ResidualSlab {
 public:
  explicit ResidualSlab(b200reg_ctx* c) : c_(c), scratch_(c) {}
  int reserve(int count, const size_t* src_n);
  ~ResidualSlab() {
    c_->residuals.slab = nullptr;
    c_->residuals.slab_points = 0;
  }

 private:
  b200reg_ctx* c_;
  Scratch scratch_;
};

// LoopClosure::coarseToFineAlignment on cloud handles (api_quatro.cu).  fine_tf16 (optional, count x 16): the fine stage's
// own fp32 final transformation of each pair whose coarse stage is valid (the transform of align()'s output cloud)
int coarse_to_fine_on_clouds(b200reg_ctx* c, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst,
                             const b200reg_quatro_params* qp, const b200reg_gicp_params* gp, b200reg_result* out,
                             b200reg_quatro_info* quatro_out, float* fine_tf16);

// The loop clouds of one call of b200reg_icp_alignment, b200reg_loop_closure or b200reg_perform_loop_closure, over the
// CALLER's pairs (api_loop_clouds.cu).  The constructor discards the stored clouds.  The call then hands over what its
// stages ran on, numbered as the stages saw their pairs: stage pair k is the caller's pair where[k], and this is the one
// place that renumbers them (an empty `where`: stage pair k is the caller's pair k).
//   clouds()  the source and target clouds, as soon as they exist: sizes the device slab for every row that can be present,
//             so that a failed allocation costs no registration;
//   finish()  the coarse stage's infos (nullptr: the call has no Quatro stage; the fine stage ran where they are valid) and
//             the fine stage's fp32 transforms (16 per stage pair): writes every row in one launch and stores the result.
// With capture off every step returns at once: no allocation, no launch.
class LoopCapture {
 public:
  LoopCapture(b200reg_ctx* c, int count);
  bool on() const { return mask_ != 0; }
  int clouds(const std::vector<int>& where, b200reg_cloud* const* src, b200reg_cloud* const* dst, bool src_tgt_rows,
             bool coarse_rows);
  int finish(const b200reg_quatro_info* qi, const float* fine_tf16);

 private:
  b200reg_ctx* c_;
  int count_, mask_;
  Scratch scratch_;
  std::vector<int> where_;
  std::vector<const b200reg_cloud*> src_, dst_;  // per stage pair
  bool src_tgt_rows_ = false;
  float4* slab_[4] = {nullptr, nullptr, nullptr, nullptr};
};

}  // namespace b200
