// api_gicp.cu -- the C ABI of the Nano-GICP path: the context's LM arena, b200reg_gicp_align, b200reg_icp_alignment, the
// residual capture and the linearize / compute_error / LM controller taps.
#include <algorithm>
#include <cstddef>
#include <cstdlib>
#include <cstring>

#include "api.cuh"

// scope guard: events created inside a call are released on EVERY exit path (the CU() macro returns early)
struct EventBag {
  std::vector<cudaEvent_t> ev;
  cudaError_t make(cudaEvent_t* e) {
    const cudaError_t r = cudaEventCreateWithFlags(e, cudaEventDisableTiming);
    if (r == cudaSuccess) ev.push_back(*e);
    return r;
  }
  ~EventBag() {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
  }
};

// ------------------------------------------------------------------------------------------
static GicpParamsDev to_dev(const b200reg_gicp_params& p) {
  GicpParamsDev d;
  d.max_iterations = p.max_iterations;
  d.lm_max_iterations = p.lm_max_iterations;
  d.max_corr_dist2 = p.max_corr_dist * p.max_corr_dist;
  d.transformation_eps = p.transformation_eps;
  d.rotation_eps = p.rotation_eps;
  d.lm_init_lambda_factor = p.lm_init_lambda_factor;
  d.icp_score_thr = p.icp_score_thr;
  return d;
}

// per-pair work buffers of a solve (correspondences, Mahalanobis matrices, accumulate partials): device memory comes from the
// caller's Scratch and goes back with it
static int make_pairs(int count, const b200reg_cloud* const* src, const b200reg_cloud* const* tgt, std::vector<PairDev>& pairs,
                      Scratch& scratch) {
  pairs.resize(count);
  for (int i = 0; i < count; i++) {
    PairDev& p = pairs[i];
    p.src = src[i]->dev;
    p.tgt = tgt[i]->dev;
    const int N = p.src.n;
    Layout l;
    const size_t o_corr = l.take((size_t)N * 4), o_sqd = l.take((size_t)N * 4), o_mah = l.take((size_t)N * 6 * 8),
                 o_par = l.take((size_t)((N + 31) / 32) * NRED * 8);
    char* slab = nullptr;
    CU(scratch.alloc((void**)&slab, l.size));
    p.corr = (int*)(slab + o_corr);
    p.sqd = (float*)(slab + o_sqd);
    p.mahal = (double*)(slab + o_mah);
    p.partial = (double*)(slab + o_par);
  }
  return B200REG_OK;
}

// persistent grids of the step kernels: as many blocks as can be resident (search: 16 per SM at 32 registers, accumulate:
// 8 per SM); blocks beyond the current number of work items exit at once.  8 to 64 blocks per SM: the solve time is flat
// from 32 on
constexpr int LM_BLOCKS_PER_SM = 32;

namespace b200 {
void lm_arena_free(b200reg_ctx* c) {
  auto& a = c->lm;
  lm_graph_destroy(&a.graph);
  if (a.d_pairs) cudaFree(a.d_pairs);
  if (a.d_states) cudaFree(a.d_states);
  if (a.d_sched) cudaFree(a.d_sched);
  if (a.d_guess) cudaFree(a.d_guess);
  if (a.d_call) cudaFree(a.d_call);
  if (a.h_call) cudaFreeHost(a.h_call);
  if (a.h_states) cudaFreeHost(a.h_states);
  a = b200reg_ctx::LmArena();
}

int ResidualSlab::reserve(int count, const size_t* src_n) {
  c_->residual_slab = nullptr;
  c_->residual_slab_points = 0;
  if (!c_->capture.residuals) return B200REG_OK;
  size_t points = 0;
  for (int i = 0; i < count; i++) points += src_n[i];
  void* p = nullptr;
  const cudaError_t e = scratch_.alloc(&p, 8 * points);
  if (e != cudaSuccess)
    return fail(B200REG_ECUDA, "residuals: cannot allocate " + std::to_string(8 * points) + " bytes: " + cudaGetErrorString(e));
  c_->residual_slab = (int32_t*)p;
  c_->residual_slab_points = points;
  return B200REG_OK;
}
}  // namespace b200

// make the arena hold `count` pairs and make sure its graph exists
static int lm_arena_ensure(b200reg_ctx* c, int count) {
  auto& a = c->lm;
  if (count > a.cap) {
    CU(cudaStreamSynchronize(c->stream));  // nothing of an earlier solve may still read the old buffers
    lm_arena_free(c);
    const int cap = std::max(16, count + count / 2);
    CU(cudaMalloc(&a.d_pairs, sizeof(PairDev) * cap));
    CU(cudaMalloc(&a.d_states, sizeof(PairState) * cap));
    CU(cudaMemsetAsync(a.d_states, 0, sizeof(PairState) * cap, c->stream));  // the records travel to the host whole: no stale bytes
    CU(cudaMalloc((void**)&a.d_sched, 64 + sizeof(LmSlot) * (size_t)cap));
    CU(cudaMalloc(&a.d_guess, sizeof(double) * 16 * cap));
    CU(cudaMalloc(&a.d_call, sizeof(LmCall)));
    CU(cudaMallocHost(&a.h_call, sizeof(LmCall)));
    CU(cudaMallocHost(&a.h_states, sizeof(PairState) * cap));
    LmSched hs;
    memset(&hs, 0, sizeof(hs));
    static_assert(sizeof(LmSched) <= 64, "LmSched header");
    hs.slots = (LmSlot*)((char*)a.d_sched + 64);
    CU(cudaMemcpy(a.d_sched, &hs, sizeof(hs), cudaMemcpyHostToDevice));
    a.cap = cap;
  }
  if (!a.graph.exec) {
    const int blocks = c->sm_count * LM_BLOCKS_PER_SM;
    const cudaError_t e = lm_graph_build(&a.graph, a.d_pairs, a.d_states, a.d_guess, a.d_call, a.d_sched, blocks, blocks, lm_slot_cache(a.cap));
    if (e != cudaSuccess) return fail(B200REG_ECUDA, std::string("building the LM graph: ") + cudaGetErrorString(e));
  }
  return B200REG_OK;
}

// One LM step launched from the host: search, accumulate and control over the arena's pairs (the body of the graph's while
// node), each kernel timed in its own profiling family
static void lm_step(b200reg_ctx* c) {
  auto& A = c->lm;
  const int blocks = c->sm_count * LM_BLOCKS_PER_SM;
  {
    ProfScope ps(c, CLS_SEARCH);
    launch_gicp_search(A.d_pairs, A.d_states, blocks, A.d_call, A.d_sched, lm_slot_cache(A.cap), c->stream);
    c->launches++;
  }
  {
    ProfScope ps(c, CLS_ACCUM);
    launch_gicp_accum(A.d_pairs, A.d_states, blocks, A.d_sched, lm_slot_cache(A.cap), c->stream);
    c->launches++;
  }
  {
    ProfScope ps(c, CLS_CTRL);
    launch_gicp_control(A.d_pairs, A.d_states, A.d_call, A.d_sched, c->stream);
    c->launches++;
  }
}

// The linearize / compute_error taps run one pair through the solve's kernels on the arena: this uploads the pair, the
// caller's pose as the guess and the call record, and runs the init kernel; every lm_step() after it is one pass.
static int tap_begin(b200reg_ctx* c, const b200reg_cloud* src, const b200reg_cloud* tgt, const double* T16, double max_corr_dist,
                     std::vector<PairDev>& pairs, Scratch& scratch) {
  int rc;
  if ((rc = make_pairs(1, &src, &tgt, pairs, scratch)) || (rc = lm_arena_ensure(c, 1))) return rc;
  auto& A = c->lm;
  cudaStream_t s = c->stream;
  b200reg_gicp_params p;
  b200reg_default_gicp_params(&p);
  p.max_corr_dist = max_corr_dist;
  LmCall& hc = *A.h_call;
  memset(&hc, 0, sizeof(hc));  // cond_handle 0: the kernels run outside the graph
  hc.count = 1;
  hc.has_guess = 1;
  hc.max_steps = 1 << 30;
  hc.prm = to_dev(p);
  CU(cudaMemcpyAsync(A.d_pairs, pairs.data(), sizeof(PairDev), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(A.d_guess, T16, sizeof(double) * 16, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(A.d_call, A.h_call, sizeof(LmCall), cudaMemcpyHostToDevice, s));
  launch_gicp_init(A.d_pairs, A.d_states, A.d_guess, A.d_call, A.d_sched, s);
  c->launches++;
  return B200REG_OK;
}

extern "C" {

int b200reg_gicp_align(b200reg_ctx* c, int count, b200reg_cloud* const* src, b200reg_cloud* const* tgt,
                       const double* guess16, const b200reg_gicp_params* params, b200reg_result* out) {
  Recording rec(c, REC_TRACE | REC_RESIDUALS);
  if (!c || count <= 0 || !src || !tgt || !params || !out) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  int rc;
  // covariances on demand (nano_gicp_impl.hpp:162-167)
  {
    std::vector<b200reg_cloud*> need;
    for (int i = 0; i < count; i++) {
      if (!src[i] || !tgt[i]) return fail(B200REG_EINVAL, "NULL cloud");
      const int m = params->regularization;
      auto stale = [&](const b200reg_cloud* cl) {
        return !cl->has_cov || (!cl->cov_user && (cl->cov_k != params->k_correspondences || cl->cov_method != m));
      };
      if (stale(src[i])) need.push_back(src[i]);
      if (stale(tgt[i])) need.push_back(tgt[i]);
    }
    if (!need.empty() &&
        (rc = b200reg_clouds_covariances_ex(c, (int)need.size(), need.data(), params->k_correspondences, params->regularization)))
      return rc;
  }
  // residual rows: those the enclosing call reserved (ResidualSlab), else this call's own, before the solve
  std::vector<int64_t> res_offsets;
  ResidualOut res_out{nullptr, nullptr};
  if (c->capture.residuals) {
    res_offsets.assign(count + 1, 0);
    for (int i = 0; i < count; i++) res_offsets[i + 1] = res_offsets[i] + src[i]->dev.n;
    const size_t total = (size_t)res_offsets[count];
    int32_t* slab = c->residual_slab;
    if (!slab || c->residual_slab_points < total) {
      const cudaError_t e = scratch.alloc((void**)&slab, 8 * total);
      if (e != cudaSuccess)
        return fail(B200REG_ECUDA, "residuals: cannot allocate " + std::to_string(8 * total) + " bytes: " + cudaGetErrorString(e));
    }
    res_out.nn = slab;
    res_out.d2 = (float*)(slab + total);
  }
  const GicpParamsDev prm = to_dev(*params);
  std::vector<PairDev> pairs;
  if ((rc = make_pairs(count, src, tgt, pairs, scratch))) return rc;
  if ((rc = lm_arena_ensure(c, count))) return rc;
  auto& A = c->lm;
  // per-call inputs of the graph: pair descriptors, guesses, the call record
  CU(cudaMemcpyAsync(A.d_pairs, pairs.data(), sizeof(PairDev) * count, cudaMemcpyHostToDevice, s));
  if (guess16) CU(cudaMemcpyAsync(A.d_guess, guess16, sizeof(double) * 16 * count, cudaMemcpyHostToDevice, s));
  LmCall& hc = *A.h_call;
  memset(&hc, 0, sizeof(hc));
  hc.count = count;
  hc.has_guess = guess16 ? 1 : 0;
  // worst case: every outer iteration burns lm_max_iterations trials, plus the fitness pass
  hc.max_steps = std::max(params->max_iterations, 0) * (1 + std::max(params->lm_max_iterations, 1)) + 2;
  hc.cond_handle = A.graph.cond_handle;
  hc.prm = prm;
  if (c->capture.lm_trace) {
    // every outer iteration makes at most lm_max_iterations trials (none when that is <= 0): the buffer holds any solve's records
    hc.trace_stride = (long long)std::max(params->max_iterations, 0) * std::max(params->lm_max_iterations, 1);
    const size_t bytes = sizeof(b200reg_lm_trial) * (size_t)hc.trace_stride * count;
    if (bytes) {
      const cudaError_t e = scratch.alloc((void**)&hc.trace, bytes);
      if (e != cudaSuccess)
        return fail(B200REG_ECUDA, "LM trace: cannot allocate " + std::to_string(bytes) + " bytes: " + cudaGetErrorString(e));
    }
  }
  CU(cudaMemcpyAsync(A.d_call, A.h_call, sizeof(LmCall), cudaMemcpyHostToDevice, s));
  static const bool env_no_graph = getenv("B200REG_LM_NO_GRAPH") != nullptr;  // Nsight Compute does not list kernels that run
  const bool no_graph = env_no_graph || c->profiling;                          // inside a conditional graph node
  if (no_graph) {
    // Profiling / ncu aid: the SAME kernels launched one by one, the host polling the schedule (what the while node does
    // on the device), each kernel bracketed by its own CUDA events
    A.h_call->cond_handle = 0;
    CU(cudaMemcpyAsync(A.d_call, A.h_call, sizeof(LmCall), cudaMemcpyHostToDevice, s));
    launch_gicp_init(A.d_pairs, A.d_states, A.d_guess, A.d_call, A.d_sched, s);
    for (;;) {
      LmSched hs;
      CU(cudaMemcpyAsync(&hs, A.d_sched, sizeof(LmSched), cudaMemcpyDeviceToHost, s));
      CU(cudaStreamSynchronize(s));
      if (hs.n_active == 0 || hs.steps > hc.max_steps) break;
      lm_step(c);
    }
    c->launches++;
  } else {
    // init kernel + device-side while loop over {search, accumulate, control}: ONE launch, ONE synchronisation per solve
    ProfScope ps(c, CLS_STEP);
    CU(cudaGraphLaunch(A.graph.exec, s));
  }
  PairState* states = A.h_states;
  CU(cudaMemcpyAsync(states, A.d_states, sizeof(PairState) * count, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(A.h_call, A.d_call, sizeof(LmCall), cudaMemcpyDeviceToHost, s));
  LmSched hsched;
  CU(cudaMemcpyAsync(&hsched, A.d_sched, sizeof(LmSched), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (!no_graph) c->launches += 1 + 3 * (int64_t)hsched.steps;  // init + (search, accumulate, control) per executed step, counted by the device
  if (A.h_call->overrun) return fail(B200REG_ESTATE, "LM state machine did not terminate");
  if (c->capture.lm_trace) {  // pair i's records are the first n_err of its region: one strided copy of the longest, then compacted
    CsrRecord& tr = c->records.rec[Records::TRACE];
    int widest = 0;
    tr.offsets.assign(count + 1, 0);
    for (int i = 0; i < count; i++) {
      tr.offsets[i + 1] = tr.offsets[i] + states[i].n_err;
      widest = std::max(widest, states[i].n_err);
    }
    const size_t rec = sizeof(b200reg_lm_trial);
    std::vector<char> rows(rec * count * widest);
    if (widest > 0) {
      CU(cudaMemcpy2DAsync(rows.data(), rec * widest, hc.trace, rec * hc.trace_stride, rec * widest, count, cudaMemcpyDeviceToHost, s));
      CU(cudaStreamSynchronize(s));
    }
    tr.rows.resize(rec * tr.offsets[count]);
    for (int i = 0; i < count; i++)
      if (states[i].n_err > 0) memcpy(&tr.rows[rec * tr.offsets[i]], &rows[rec * i * widest], rec * states[i].n_err);
  }
  if (c->capture.residuals) {  // the fitness pass's per-point values of every pair, in one launch and one copy
    const size_t total = (size_t)res_offsets[count];
    std::vector<ResidualRow> rows;
    int max_n = 0;
    for (int i = 0; i < count; i++) {
      if (pairs[i].src.n == 0) continue;
      rows.push_back(ResidualRow{pairs[i].src.pts, pairs[i].tgt.pts, pairs[i].corr, pairs[i].sqd, pairs[i].src.n, res_offsets[i]});
      max_n = std::max(max_n, pairs[i].src.n);
    }
    CsrRecord& rs = c->records.rec[Records::RESIDUALS];
    rs.rows.resize(8 * total);  // nn block, then d2 block, as in the slab
    if (!rows.empty()) {
      ResidualRow* d_rows = nullptr;
      CU(scratch.upload(&d_rows, rows.data(), sizeof(ResidualRow) * rows.size()));
      {
        ProfScope ps(c, CLS_MISC);
        launch_residual_rows(d_rows, (int)rows.size(), max_n, res_out, s);
        c->launches++;
        c->prof_bytes[CLS_MISC] += 48.0 * total;  // 16 source + 8 corr / sqd + 16 target in, 8 out
      }
      CU(cudaGetLastError());
      CU(cudaMemcpyAsync(rs.rows.data(), res_out.nn, total * 8, cudaMemcpyDeviceToHost, s));
      CU(cudaStreamSynchronize(s));
    }
    rs.offsets.swap(res_offsets);
  }
  for (int i = 0; i < count; i++) {
    const PairState& st = states[i];
    b200reg_result& r = out[i];
    r = default_result();  // pose_between stays the identity unless the result is valid
    for (int a = 0; a < 3; a++) {
      for (int b = 0; b < 3; b++) r.T[4 * a + b] = st.R[3 * a + b];
      r.T[4 * a + 3] = st.t[a];
    }
    for (int a = 0; a < 12; a++) r.Tf[a] = st.Tf[a];
    if (st.n_lin > 0) memcpy(r.final_hessian, st.H, sizeof(r.final_hessian));
    else for (int a = 0; a < 6; a++) r.final_hessian[7 * a] = 1.0;  // final_hessian_.setIdentity() (lsq_registration_impl.hpp:62)
    r.fitness = st.fitness;
    r.converged = st.converged;
    r.valid = (st.converged && st.fitness < params->icp_score_thr) ? 1 : 0;
    if (r.valid)  // getFinalTransformation().cast<double>() (loop_closure.cpp:133)
      for (int a = 0; a < 12; a++) r.pose_between[a] = (double)st.Tf[a];
    r.iterations = st.nr_iterations;
    r.n_linearize = st.n_lin;
    r.n_error = st.n_err;
    r.lm_failed = st.lm_failed;
    r.status = 0;
    // SURVEY §8(d): K3 136*N per linearize, K4 132*N per compute_error, K5 16*N fitness.  Per kernel: the search reads the
    // 16-byte points and writes the 8-byte correspondence record (24*N of K3; all 16*N of K5), the accumulate pass owns the rest
    const double N = pairs[i].src.n;
    if (no_graph) {
      c->prof_bytes[CLS_SEARCH] += (24.0 * st.n_lin + 16.0) * N;
      c->prof_bytes[CLS_ACCUM] += (112.0 * st.n_lin + 132.0 * st.n_err) * N;
    } else {
      c->prof_bytes[CLS_STEP] += (136.0 * st.n_lin + 132.0 * st.n_err + 16.0) * N;
    }
  }
  return rec.commit(B200REG_OK, count);
}

// the solve of icpAlignment over built clouds, with its loop clouds: FINAL is align()'s output cloud of every pair
static int icp_solve(b200reg_ctx* c, LoopCapture& cap, int count, b200reg_cloud* const* sc, b200reg_cloud* const* tc,
                     const b200reg_gicp_params* params, b200reg_result* out) {
  int rc = cap.clouds(count, sc, tc, false, false);
  if (!rc) rc = b200reg_gicp_align(c, count, sc, tc, nullptr, params, out);
  if (rc || !cap.on()) return rc;
  std::vector<float> fine_tf(16 * (size_t)count);
  for (int i = 0; i < count; i++) memcpy(&fine_tf[16 * (size_t)i], out[i].Tf, sizeof(out[i].Tf));
  return cap.finish(nullptr, fine_tf.data());
}

// one chunk of pairs, raw records already on the device
static int icp_alignment_device(b200reg_ctx* c, LoopCapture& cap, int count, const float* const* src_xyz, const size_t* src_n,
                                const float* const* tgt_xyz, const size_t* tgt_n, size_t stride_bytes,
                                const b200reg_gicp_params* params, b200reg_result* out) {
  CloudBag bag(c);
  std::vector<b200reg_cloud*> sc(count), tc(count);
  int rc = create_pair_clouds(c, count, src_xyz, src_n, tgt_xyz, tgt_n, stride_bytes, 1, cap.on(), bag, sc.data(), tc.data());
  if (!rc) rc = b200reg_clouds_covariances_ex(c, 2 * count, bag.cl.data(), params->k_correspondences, params->regularization);
  if (!rc) rc = icp_solve(c, cap, count, sc.data(), tc.data(), params, out);
  return rc;
}

int b200reg_icp_alignment(b200reg_ctx* c, int count, const float* const* src_xyz, const size_t* src_n,
                          const float* const* tgt_xyz, const size_t* tgt_n, size_t stride_bytes, int on_device,
                          const b200reg_gicp_params* params, b200reg_result* out) {
  Recording rec(c, REC_TRACE | REC_RESIDUALS | REC_CLOUDS);
  if (!c || count <= 0 || !src_xyz || !src_n || !tgt_xyz || !tgt_n || !params || !out)
    return fail(B200REG_EINVAL, "bad argument");
  if (stride_bytes < 12 || stride_bytes % 4) return fail(B200REG_EINVAL, "stride_bytes must be a multiple of 4, >= 12");
  for (int i = 0; i < count; i++)
    if (!src_xyz[i] || !tgt_xyz[i] || src_n[i] == 0 || tgt_n[i] == 0) return fail(B200REG_EINVAL, "empty cloud");
  CU(cudaSetDevice(c->device));
  LoopCapture cap(c);
  ResidualSlab rslab(c);
  if (const int rc = rslab.reserve(count, src_n)) return rc;
  if (on_device)
    return rec.commit(icp_alignment_device(c, cap, count, src_xyz, src_n, tgt_xyz, tgt_n, stride_bytes, params, out), count);
  // Host buffers: all uploads are queued on the copy stream up front, chunk by chunk; the compute stream processes
  // chunk k as soon as its records have landed, so the PCIe time of chunk k+1 hides behind the kernels of chunk k.
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  int want = c->pipeline_chunks;
  if (const char* e = getenv("B200REG_PIPELINE_CHUNKS")) want = atoi(e);
  const int nchunks = std::max(1, std::min(want, count));
  const int per = (count + nchunks - 1) / nchunks;
  Layout staged;
  std::vector<size_t> off_s(count), off_t(count);
  for (int i = 0; i < count; i++) {
    off_s[i] = staged.take(src_n[i] * stride_bytes);
    off_t[i] = staged.take(tgt_n[i] * stride_bytes);
  }
  char* stage = nullptr;
  CU(scratch.alloc((void**)&stage, staged.size));
  std::vector<const float*> sp(count), tp(count);  // each pair's records in the staging buffer
  for (int i = 0; i < count; i++) {
    sp[i] = (const float*)(stage + off_s[i]);
    tp[i] = (const float*)(stage + off_t[i]);
  }
  // Release order on every exit path (reverse declaration order): the clouds first, then the copy stream is drained, and only
  // then does Scratch return the staging buffer to the pool -- an upload may still be writing into it until the drain.
  EventBag events;
  struct CopyDrain {  // the uploads read the caller's buffers: they must have finished whenever this call returns
    cudaStream_t cs;
    ~CopyDrain() { cudaStreamSynchronize(cs); }
  } drain{c->copy_stream};
  cudaEvent_t ready;
  CU(events.make(&ready));
  CU(cudaEventRecord(ready, s));
  CU(cudaStreamWaitEvent(c->copy_stream, ready, 0));
  std::vector<cudaEvent_t> landed;
  for (int k0 = 0; k0 < count; k0 += per) {
    const int k1 = std::min(count, k0 + per);
    for (int i = k0; i < k1; i++) {
      CU(cudaMemcpyAsync(stage + off_s[i], src_xyz[i], src_n[i] * stride_bytes, cudaMemcpyHostToDevice, c->copy_stream));
      CU(cudaMemcpyAsync(stage + off_t[i], tgt_xyz[i], tgt_n[i] * stride_bytes, cudaMemcpyHostToDevice, c->copy_stream));
    }
    cudaEvent_t e;
    CU(events.make(&e));
    CU(cudaEventRecord(e, c->copy_stream));
    landed.push_back(e);
  }
  // index build + covariances chunk by chunk (they only need that chunk's records), then ONE batched LM solve over
  // all pairs: the host never blocks before the solve's first poll, so the GPU stays busy while later chunks land.
  int rc = B200REG_OK;
  int chunk = 0;
  std::vector<b200reg_cloud*> sc(count, nullptr), tc(count, nullptr);
  CloudBag bag(c);
  for (int k0 = 0; k0 < count && !rc; k0 += per, chunk++) {
    const int m = std::min(count, k0 + per) - k0;
    CU(cudaStreamWaitEvent(s, landed[chunk], 0));
    rc = create_pair_clouds(c, m, &sp[k0], &src_n[k0], &tp[k0], &tgt_n[k0], stride_bytes, 1, cap.on(), bag, &sc[k0], &tc[k0]);
    // the chunk's clouds are the last 2 m in the bag
    if (!rc) rc = b200reg_clouds_covariances_ex(c, 2 * m, &bag.cl[bag.cl.size() - 2 * m], params->k_correspondences, params->regularization);
  }
  if (!rc) rc = icp_solve(c, cap, count, sc.data(), tc.data(), params, out);
  return rec.commit(rc, count);  // clouds, events and the copy stream are released / drained by the scope guards
}

int b200reg_linearize(b200reg_ctx* c, const b200reg_cloud* src, const b200reg_cloud* tgt, const double* T16,
                      double max_corr_dist, double* H36, double* b6, double* err, int32_t* corr_out, float* sqd_out) {
  if (!c || !src || !tgt || !T16) return fail(B200REG_EINVAL, "bad argument");
  if (!src->has_cov || !tgt->has_cov) return fail(B200REG_ESTATE, "covariances not computed");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  std::vector<PairDev> pairs;
  int rc;
  if ((rc = tap_begin(c, src, tgt, T16, max_corr_dist, pairs, scratch))) return rc;
  lm_step(c);  // exactly one linearize pass
  PairState st;
  const int N = src->dev.n;
  std::vector<int> corr(N), src_orig, tgt_orig;
  std::vector<float> sqd(N);
  CU(cudaMemcpyAsync(&st, c->lm.d_states, sizeof(PairState), cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(corr.data(), pairs[0].corr, (size_t)N * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(sqd.data(), pairs[0].sqd, (size_t)N * 4, cudaMemcpyDeviceToHost, s));
  if ((rc = sorted_to_original(c, src->dev, src_orig)) || (rc = sorted_to_original(c, tgt->dev, tgt_orig))) return rc;
  if (H36) memcpy(H36, st.H, sizeof(double) * 36);
  if (b6) memcpy(b6, st.b, sizeof(double) * 6);
  if (err) *err = st.y0;
  for (int p = 0; p < N; p++) {
    if (corr_out) corr_out[src_orig[p]] = corr[p] >= 0 ? tgt_orig[corr[p]] : -1;
    if (sqd_out) sqd_out[src_orig[p]] = sqd[p];
  }
  return B200REG_OK;
}

int b200reg_compute_error(b200reg_ctx* c, const b200reg_cloud* src, const b200reg_cloud* tgt, const double* T_lin16,
                          const double* T_trial16, double max_corr_dist, double* err) {
  if (!c || !src || !tgt || !T_lin16 || !T_trial16 || !err) return fail(B200REG_EINVAL, "bad argument");
  if (!src->has_cov || !tgt->has_cov) return fail(B200REG_ESTATE, "covariances not computed");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  std::vector<PairDev> pairs;
  if (const int rc = tap_begin(c, src, tgt, T_lin16, max_corr_dist, pairs, scratch)) return rc;
  lm_step(c);  // linearize: correspondences + Mahalanobis, phase -> TRIAL
  // overwrite the trial pose the LM controller prepared with the caller's
  double Rt[9], tt[3];
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) Rt[3 * a + b] = T_trial16[4 * a + b];
    tt[a] = T_trial16[4 * a + 3];
  }
  PairState* d_st = c->lm.d_states;
  CU(cudaMemcpyAsync((char*)d_st + offsetof(PairState, Rt), Rt, sizeof(Rt), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync((char*)d_st + offsetof(PairState, tt), tt, sizeof(tt), cudaMemcpyHostToDevice, s));
  lm_step(c);  // compute_error at the trial pose
  PairState st;
  CU(cudaMemcpyAsync(&st, d_st, sizeof(PairState), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  *err = st.y_trial;
  return B200REG_OK;
}

int b200reg_lm_step_tap(b200reg_ctx* c, int n, const b200reg_lm_case* cases, b200reg_lm_step* out) {
  if (!c || n <= 0 || !cases || !out) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  b200reg_lm_case* d_cases = nullptr;
  b200reg_lm_step* d_out = nullptr;
  CU(scratch.alloc((void**)&d_cases, sizeof(b200reg_lm_case) * (size_t)n));
  CU(scratch.alloc((void**)&d_out, sizeof(b200reg_lm_step) * (size_t)n));
  CU(cudaMemcpyAsync(d_cases, cases, sizeof(b200reg_lm_case) * (size_t)n, cudaMemcpyHostToDevice, s));
  c->launches += launch_lm_step_tap(d_cases, n, d_out, s);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, d_out, sizeof(b200reg_lm_step) * (size_t)n, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

}  // extern "C"
