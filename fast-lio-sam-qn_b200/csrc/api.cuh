// api.cuh -- what the host files of the C ABI share (api.cu, api_gicp.cu, api_quatro.cu, api_keyframes.cu): the context and
// cloud objects, error reporting, profiling scopes, stream-ordered scratch memory and the helpers more than one area uses.
// Host orchestration only; every arithmetic step of the path runs in the kernels of index_build.cu / gicp.cu / quatro.cu /
// assemble.cu.  There is no CPU fallback anywhere in this library.
#pragma once
#include <cuda_runtime.h>
#include <nccl.h>  // types only: the library is dlopen()ed in b200reg_comm_*

#include <cstddef>
#include <cstdint>
#include <initializer_list>
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

namespace b200 {

// One recorded output of a call, CSR over its pairs, on the host: `offsets` (pairs + 1; empty until a stage of the call
// writes the record) and `rows`, the record's columns one block after another, each column a fixed number of bytes per
// row (record_copy's table).  The device slab a stage fills has the same layout, so one copy brings it to the host.
// `rows` keeps its memory from call to call: a stage resizes it in place.
struct CsrRecord {
  std::vector<int64_t> offsets;
  std::vector<char> rows;
  // Stage pair k becomes caller pair where[k] (empty `where`: pair k); every other caller pair, and every pair the
  // record does not hold, gets an empty row.  `where` ascends, as every stage's subset of its caller's pairs does, so the
  // rows keep their order and only the offsets change.
  void remap(int count, const std::vector<int>& where);
};

// The records a call can leave for its caller (include/b200reg.h: b200reg_lm_trace, b200reg_residuals,
// b200reg_quatro_matches, b200reg_loop_clouds), and which of them the most recent recording call that touched them stored
struct Records {
  enum { TRACE, RESIDUALS, MATCHES, CLOUD, N = CLOUD + 4 };  // CLOUD + s: the loop clouds of kind 1 << s (B200REG_CLOUD_*)
  CsrRecord rec[N];
  unsigned held = 0;  // bit r: rec[r] is stored
};
constexpr unsigned REC_TRACE = 1u << Records::TRACE, REC_RESIDUALS = 1u << Records::RESIDUALS, REC_MATCHES = 1u << Records::MATCHES,
                   REC_CLOUDS = 15u << Records::CLOUD, REC_ALL = REC_TRACE | REC_RESIDUALS | REC_MATCHES | REC_CLOUDS;

// The recording settings (b200reg_ctx_set_loop_clouds / _set_lm_trace / _set_quatro_matches / _set_residuals): a
// context's, or the driver's that a batch job copies at its submit
struct Capture {
  int cloud_mask = 0;
  bool lm_trace = false;
  bool quatro_matches = false;
  bool residuals = false;
  bool on() const { return cloud_mask || lm_trace || quatro_matches || residuals; }
  bool wants(int r) const {  // record r (Records) is recorded
    return r == Records::TRACE ? lm_trace : r == Records::RESIDUALS ? residuals : r == Records::MATCHES ? quatro_matches
                                                                                                       : (cloud_mask >> (r - Records::CLOUD) & 1) != 0;
  }
  bool operator!=(const Capture& o) const {
    return cloud_mask != o.cloud_mask || lm_trace != o.lm_trace || quatro_matches != o.quatro_matches || residuals != o.residuals;
  }
};

}  // namespace b200

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
  // the recorded outputs: what to record, what is stored, and whether a recording call is running (Recording)
  Capture capture;
  Records records;
  bool recording = false;
  // device rows reserved for the residuals by the call in flight (ResidualSlab): nn block, then d2 block
  int32_t* residual_slab = nullptr;
  size_t residual_slab_points = 0;
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

// The one lifecycle rule of the records (include/b200reg.h), for an entry point that records.  Constructed on entry,
// before the argument checks, it discards every record in `touches`.  The call's stages then write their records into
// c->records as they run, numbered as they saw their pairs.  commit() stores them, renumbered to the caller's pairs, only
// when the call succeeds, and only those the settings ask for.  A scope opened while another is open (b200reg_gicp_align or
// b200reg_quatro_align as a stage of a larger call) does nothing: the outermost call discards and stores for all of them.
class Recording {
 public:
  Recording(b200reg_ctx* c, unsigned touches);
  ~Recording();
  Recording(const Recording&) = delete;
  Recording& operator=(const Recording&) = delete;
  // rc == B200REG_OK: stores the touched records, stage pair k as the caller's pair where[k] (CsrRecord::remap).  Returns rc.
  int commit(int rc, int count, const std::vector<int>& where = {});

 private:
  b200reg_ctx* c_;
  unsigned touches_ = 0;  // 0: a nested scope
};

// The copy-out rules of every record getter, over a context's records or a batch-driver job's (null: none held): r < 0
// (a loop-cloud kind that is not one B200REG_CLOUD_* bit, cloud_record) is B200REG_EINVAL; a record not held is
// B200REG_ESTATE with the message `none`; offsets_out NULL returns the pair count; then the offsets, the capacity rule of
// include/b200reg.h, and column j of the record into cols[j] unless that is NULL.  (api.cu)
int record_copy(const Records* rs, int r, const std::string& none, int64_t* offsets_out, size_t capacity,
                std::initializer_list<void*> cols);
// Records::CLOUD + log2 of a B200REG_CLOUD_* bit; -1 for anything else
int cloud_record(int kind);

// The device rows of the residual capture of one b200reg_icp_alignment, b200reg_loop_closure or
// b200reg_perform_loop_closure call, reserved as soon as its source clouds exist, so that a failed allocation costs no
// registration: one row per source point of every pair that can run the fine stage.  The call's b200reg_gicp_align writes
// into them instead of allocating its own.  Returned at the end of the scope; with recording off nothing is allocated.
class ResidualSlab {
 public:
  explicit ResidualSlab(b200reg_ctx* c) : c_(c), scratch_(c) {}
  int reserve(int count, const size_t* src_n);
  ~ResidualSlab() {
    c_->residual_slab = nullptr;
    c_->residual_slab_points = 0;
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

// The loop clouds of one call of b200reg_icp_alignment, b200reg_loop_closure or b200reg_perform_loop_closure, numbered as
// its stages saw their pairs (api_loop_clouds.cu); the call's Recording renumbers them to its own pairs.
//   clouds()  the `count` source and target clouds of the stages, as soon as they exist: sizes the device slab for every
//             row that can be present, so that a failed allocation costs no registration;
//   finish()  the coarse stage's infos (nullptr: the call has no Quatro stage; the fine stage ran where they are valid) and
//             the fine stage's fp32 transforms (16 per stage pair): writes every row in one launch and into c->records.
// With capture off every step returns at once: no allocation, no launch.
class LoopCapture {
 public:
  explicit LoopCapture(b200reg_ctx* c) : c_(c), mask_(c->capture.cloud_mask), scratch_(c) {}
  bool on() const { return mask_ != 0; }
  int clouds(int count, b200reg_cloud* const* src, b200reg_cloud* const* dst, bool src_tgt_rows, bool coarse_rows);
  int finish(const b200reg_quatro_info* qi, const float* fine_tf16);

 private:
  b200reg_ctx* c_;
  int mask_;
  Scratch scratch_;
  std::vector<const b200reg_cloud*> src_, dst_;  // per stage pair
  bool src_tgt_rows_ = false;
  float4* slab_[4] = {nullptr, nullptr, nullptr, nullptr};
};

}  // namespace b200
