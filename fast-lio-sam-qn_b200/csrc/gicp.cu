// gicp.cu -- Nano-GICP on the GPU: k-NN covariances, the fused correspondence + Mahalanobis +
// linearize pass, compute_error, fitness and the Levenberg-Marquardt controller, all batched
// over pairs (blockIdx.y = pair) and driven by a per-pair device-side state machine so that the
// host never synchronises inside an LM iteration.
//
// Reference behaviour being replaced (paths relative to the reference tree's root):
//   third_party/nano_gicp/include/nano_gicp/impl/nano_gicp_impl.hpp
//       calculate_covariances :298-357, update_correspondences :173-211, linearize :213-270,
//       compute_error :272-296
//   third_party/nano_gicp/include/nano_gicp/impl/lsq_registration_impl.hpp
//       computeTransformation :88-115, is_converged :117-127, step_lm :160-208
//   third_party/nano_gicp/include/nano_gicp/gicp/so3.hpp  so3_exp :99-118
//   pcl::Registration::getFitnessScore (call site fast_lio_sam_qn/src/loop_closure.cpp:127)
#include "internal.cuh"
#include "knn.cuh"
#include "launchers.cuh"
#include "smallmath.cuh"

namespace b200 {

// ---------------------------------------------------------------------------------------
// small fp64 helpers (sym3_inverse and the covariance epilogue are in smallmath.cuh)
// ---------------------------------------------------------------------------------------
// R C R^T for symmetric C (packed) and row-major R; packed symmetric result
__device__ __forceinline__ void rcrt(const double R[9], const double c[6], double o[6]) {
  const double C[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
  double RC[3][3];
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) RC[i][j] = R[3 * i] * C[0][j] + R[3 * i + 1] * C[1][j] + R[3 * i + 2] * C[2][j];
  int k = 0;
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = i; j < 3; j++) o[k++] = RC[i][0] * R[3 * j] + RC[i][1] * R[3 * j + 1] + RC[i][2] * R[3 * j + 2];
}

// solve (H + lambda I) x = -b, symmetric 6x6, unpivoted LDL^T
__device__ void solve6(const double H[36], double lambda, const double b[6], double x[6]) {
  double L[6][6], D[6];
  for (int j = 0; j < 6; j++) {
    double dj = H[7 * j] + lambda;
    for (int k = 0; k < j; k++) dj -= L[j][k] * L[j][k] * D[k];
    D[j] = dj;
    for (int i = j + 1; i < 6; i++) {
      double v = H[6 * i + j];
      for (int k = 0; k < j; k++) v -= L[i][k] * L[j][k] * D[k];
      L[i][j] = dj != 0.0 ? v / dj : 0.0;
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) {
    double s = -b[i];
    for (int k = 0; k < i; k++) s -= L[i][k] * y[k];
    y[i] = s;
  }
  for (int i = 0; i < 6; i++) y[i] = D[i] != 0.0 ? y[i] / D[i] : 0.0;
  for (int i = 5; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < 6; k++) s -= L[k][i] * x[k];
    x[i] = s;
  }
}

// so3_exp (so3.hpp:99-118) + Quaternion::toRotationMatrix
__device__ void so3_exp_matrix(const double w[3], double R[9]) {
  double theta_sq = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  double imag, real;
  if (theta_sq < 1e-10) {
    double q4 = theta_sq * theta_sq;
    imag = 0.5 - 1.0 / 48.0 * theta_sq + 1.0 / 3840.0 * q4;
    real = 1.0 - 1.0 / 8.0 * theta_sq + 1.0 / 384.0 * q4;
  } else {
    double theta = sqrt(theta_sq), half = 0.5 * theta;
    imag = sin(half) / theta;
    real = cos(half);
  }
  double qw = real, qx = imag * w[0], qy = imag * w[1], qz = imag * w[2];
  double tx = 2 * qx, ty = 2 * qy, tz = 2 * qz;
  double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

// is_converged (lsq_registration_impl.hpp:117-127): max of (1.0 / eps) * |x| < 1, the reciprocal first as the reference
// writes it (|x| / eps rounds differently at |x| = eps for some eps, e.g. 1e-5).  A NaN anywhere in the step is not
// converged: the reference's maxCoeff of an all-NaN block is NaN and NaN < 1 is false (fmax would drop it).  DESIGN §4.
__device__ bool delta_converged(const PairState* st, const GicpParamsDev& prm) {
  const double ir = 1.0 / prm.rotation_eps, it = 1.0 / prm.transformation_eps;
  double m = 0;
  bool nan = false;
  for (int i = 0; i < 9; i++) {
    const double v = ir * fabs(st->dR[i] - ((i % 4) == 0 ? 1.0 : 0.0));
    nan |= isnan(v);
    m = fmax(m, v);
  }
  for (int i = 0; i < 3; i++) {
    const double v = it * fabs(st->dt[i]);
    nan |= isnan(v);
    m = fmax(m, v);
  }
  return !nan && m < 1.0;
}

// ---------------------------------------------------------------------------------------
// LM controller, executed by ONE thread of the last-arriving block of a pair.
// ---------------------------------------------------------------------------------------
__device__ void lm_prepare_trial(PairState* st) {
  solve6(st->H, st->lambda, st->b, st->d);
  so3_exp_matrix(st->d, st->dR);
  st->dt[0] = st->d[3]; st->dt[1] = st->d[4]; st->dt[2] = st->d[5];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++)
      st->Rt[3 * i + j] = st->dR[3 * i] * st->R[j] + st->dR[3 * i + 1] * st->R[3 + j] + st->dR[3 * i + 2] * st->R[6 + j];
    st->tt[i] = st->dR[3 * i] * st->t[0] + st->dR[3 * i + 1] * st->t[1] + st->dR[3 * i + 2] * st->t[2] + st->dt[i];
  }
  st->phase = PH_TRIAL;
}

__device__ void lm_finish(PairState* st, int converged) {
  st->converged = converged;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) st->Tf[4 * r + c] = (float)st->R[3 * r + c];
    st->Tf[4 * r + 3] = (float)st->t[r];
  }
  st->phase = PH_FITNESS;
}

// One trace record (b200reg_lm_trial): the trial's inputs and outcome, and x0 after the decision.
__device__ void lm_record(b200reg_lm_trial* r, const PairState* st, int trial, int decision, double yi, double rho, double lambda,
                          double nu, const double d[6]) {
  r->outer = st->nr_iterations;
  r->trial = trial;
  r->decision = decision;
  r->reserved = 0;
  r->y0 = st->y0;
  r->yi = yi;
  r->rho = rho;
  r->lambda = lambda;
  r->nu = nu;
  for (int i = 0; i < 6; i++) r->d[i] = d[i];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) r->T[4 * i + j] = st->R[3 * i + j];
    r->T[4 * i + 3] = st->t[i];
  }
}

// trace: this pair's trace region (LmCall::trace), nullptr when tracing is off
__device__ void lm_update(PairState* st, const double* sums, const GicpParamsDev& prm, int phase, int n_src,
                          int* done_counter, b200reg_lm_trial* trace) {  // done_counter = &LmSched::done
  if (phase == PH_LINEARIZE) {
    int k = 0;
    for (int i = 0; i < 6; i++)
      for (int j = i; j < 6; j++) {
        st->H[6 * i + j] = sums[k];
        st->H[6 * j + i] = sums[k];
        k++;
      }
    for (int i = 0; i < 6; i++) st->b[i] = sums[21 + i];
    st->y0 = sums[27];
    st->n_lin++;
    st->nr_iterations = st->outer_it;
    if (st->lambda < 0.0) {  // maxCoeff of |diag H|: a NaN on the diagonal makes lambda NaN, as in the reference
      double mx = 0;
      bool nan = false;
      for (int i = 0; i < 6; i++) {
        nan |= isnan(st->H[7 * i]);
        mx = fmax(mx, fabs(st->H[7 * i]));
      }
      st->lambda = prm.lm_init_lambda_factor * (nan ? (double)NAN : mx);
    }
    st->nu = 2.0;
    st->inner_it = 0;
    if (prm.lm_max_iterations <= 0) {  // step_lm's trial loop runs no trial and returns false: "lm not converged!!"
      st->lm_failed = 1;
      lm_finish(st, 0);
      return;
    }
    lm_prepare_trial(st);
  } else if (phase == PH_TRIAL) {
    const double yi = sums[0];
    st->y_trial = yi;
    st->n_err++;
    double denom = 0;
    for (int i = 0; i < 6; i++) denom += st->d[i] * (st->lambda * st->d[i] - st->b[i]);
    const double rho = (st->y0 - yi) / denom;
    // what the trace records of this trial: the next trial's lm_prepare_trial overwrites d, the decision moves lambda / nu
    const int trial = st->inner_it;
    const double lambda = st->lambda, nu = st->nu;
    double d[6];
    for (int i = 0; i < 6; i++) d[i] = st->d[i];
    int decision;
    if (rho < 0) {
      if (delta_converged(st, prm)) {
        decision = 2;
        lm_finish(st, 1);  // step_lm returns true without touching x0; the caller then sees converged
      } else {
        st->lambda = st->nu * st->lambda;
        st->nu = 2 * st->nu;
        st->inner_it++;
        if (st->inner_it >= prm.lm_max_iterations) {
          decision = 3;
          st->lm_failed = 1;  // "lm not converged!!"
          lm_finish(st, 0);
        } else {
          decision = 0;
          lm_prepare_trial(st);
        }
      }
    } else {
      decision = 1;
      for (int i = 0; i < 9; i++) st->R[i] = st->Rt[i];
      for (int i = 0; i < 3; i++) st->t[i] = st->tt[i];
      const double x = 2 * rho - 1;
      st->lambda = st->lambda * fmax(1.0 / 3.0, 1 - x * x * x);
      if (delta_converged(st, prm)) {
        lm_finish(st, 1);
      } else {
        st->outer_it++;
        if (st->outer_it >= prm.max_iterations) lm_finish(st, 0);
        else st->phase = PH_LINEARIZE;
      }
    }
    if (trace) lm_record(&trace[st->n_err - 1], st, trial, decision, yi, rho, lambda, nu, d);
  } else if (phase == PH_FITNESS) {
    st->fitness = n_src > 0 ? sums[0] / (double)n_src : 0.0;
    st->phase = PH_DONE;
    atomicAdd(done_counter, 1);
  }
}

// Rebuild the slot list from the pairs' phases (one block, any size that is a multiple of 32); ascending pair order.
__device__ void sched_rebuild(const PairDev* pairs, const PairState* states, LmSched* sched, LmCall* call) {
  __shared__ int s_wcnt[32];
  __shared__ int s_carry_cnt, s_stride;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (threadIdx.x == 0) {
    s_carry_cnt = 0;
    s_stride = 0;
  }
  __syncthreads();
  const int n = sched->n_pairs;
  int my_max = 0;
  for (int base = 0; base < n; base += blockDim.x) {
    const int p = base + threadIdx.x;
    int nblk = 0, phase = PH_DONE, seeded = 0;
    if (p < n) {
      nblk = (pairs[p].src.n + STEP_THREADS - 1) / STEP_THREADS;
      my_max = max(my_max, nblk);
      phase = __ldcg(&states[p].phase);
      seeded = __ldcg(&states[p].n_lin) > 0;
    }
    const int act = (p < n && phase != PH_DONE) ? 1 : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, act);
    if (lane == 0) s_wcnt[warp] = __popc(bal);
    __syncthreads();
    int woff = s_carry_cnt;
    for (int w = 0; w < warp; w++) woff += s_wcnt[w];
    if (act) sched->slots[woff + __popc(bal & ((1u << lane) - 1u))] = LmSlot{p, nblk, phase, seeded};
    __syncthreads();
    if (threadIdx.x == 0)
      for (int w = 0; w < nw; w++) s_carry_cnt += s_wcnt[w];
    __syncthreads();
  }
  atomicMax(&s_stride, my_max);
  __syncthreads();
  if (threadIdx.x == 0) {
    sched->stride = s_stride;
    sched->n_active = s_carry_cnt;
    sched->total_items = s_carry_cnt * s_stride;
    sched->arrive = 0;
    int again = s_carry_cnt > 0 ? 1 : 0;
    if (again && sched->steps > call->max_steps) {  // the state machine always terminates; this only guards the device loop
      call->overrun = 1;
      again = 0;
    }
    __threadfence();
    // the while node of the solve's CUDA graph runs the two step kernels again as long as a pair is active
    if (call->cond_handle) cudaGraphSetConditional((cudaGraphConditionalHandle)call->cond_handle, again);
  }
}

__global__ void __launch_bounds__(256) k_gicp_init(const PairDev* pairs, PairState* states, const double* guess_buf, LmCall* call,
                                                    LmSched* sched) {
  const int count = call->count;
  const double* guess16 = call->has_guess ? guess_buf : nullptr;
  const GicpParamsDev prm = call->prm;
  if (threadIdx.x == 0) call->overrun = 0;
  for (int p = threadIdx.x; p < count; p += blockDim.x) {
    PairState* st = &states[p];
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) st->R[3 * i + j] = guess16 ? guess16[16 * p + 4 * i + j] : (i == j ? 1.0 : 0.0);
      st->t[i] = guess16 ? guess16[16 * p + 4 * i + 3] : 0.0;
    }
    st->lambda = -1.0;
    st->nu = 2.0;
    st->y0 = 0.0;
    st->y_trial = 0.0;
    st->fitness = 0.0;
    st->phase = PH_LINEARIZE;
    st->outer_it = 0;
    st->inner_it = 0;
    st->converged = 0;
    st->lm_failed = 0;
    st->n_lin = 0;
    st->n_err = 0;
    st->nr_iterations = 0;
    st->arrive = 0;
    st->pad = 0;
    if (prm.max_iterations <= 0) lm_finish(st, 0);
  }
  if (threadIdx.x == 0) {
    sched->n_pairs = count;
    sched->done = 0;
    sched->steps = 0;
  }
  __threadfence();
  __syncthreads();
  sched_rebuild(pairs, states, sched, call);
}

// ---------------------------------------------------------------------------------------
// K2: 15-NN + covariance + PLANE regularisation (nano_gicp_impl.hpp:298-357); the regularisation is
// cov_regularize_store (smallmath.cuh).
// ---------------------------------------------------------------------------------------
// Seed the heap with the K points around position i in Morton order (cheap, coalesced, usually most of the true
// neighbours: the traversal then starts with a tight bound and only ever inserts improvements) and walk the tree.
// A seed enters on the walk's own rule, d2 <= FLT_MAX: the NaN points (all at key 0, so often among the first points'
// seeds) and points at infinity leave an empty slot, as they are never candidates of the walk.
template <typename Heap, int K>
__device__ __forceinline__ void cov_knn(const CloudDev& c, int i, float4 q, Heap& res) {
  int lo = max(0, i - K / 2), hi = min(c.n - 1, lo + K - 1);
  lo = max(0, hi - (K - 1));
#pragma unroll
  for (int j = 0; j < K; j++) {
    float d = 3.402823466e+38f;
    int pos = -1;
    if (lo + j <= hi) {
      const float4 p = __ldg(&c.pts[lo + j]);
      const float dj = dist2_rn(q.x, q.y, q.z, p.x, p.y, p.z);
      if (dj <= d) {
        d = dj;
        pos = lo + j;
      }
    }
    res.set(j, d, pos);
  }
  res.heapify();
  knn_walk(c, q.x, q.y, q.z, res, nullptr, lo, hi);  // stack in local memory: on chip it ran slower on H100 (DESIGN.md §3)
}

// On-chip traversal stack depth of k_gicp_search (knn_walk, knn.cuh).  From profiles/emulate_stack_depth.py on the bench's
// first pair (DESIGN.md §3): the seeded 1-NN walks stay within 6 entries for 99.8 % of their pushes (the one unseeded pass
// per pair goes 18 deep and spills the rest to local memory).
constexpr int SEARCH_STACK = 6;

// K is the CAPACITY of the result set; k <= K neighbours enter the covariance (the k nearest of the K nearest are the
// k nearest), so every k in 1..32 is served by the next instantiated capacity.  k > 32 runs k_covariance_large
// (knn_large.cu), one warp per point.
// The result set is a max-heap in shared memory (KnnHeap, knn.cuh): the covariance needs the SET of neighbours, not their
// order.  (A sorted list in registers, the earlier design, spent most of its instructions in the insertion chain.)
template <int K>
__global__ void __launch_bounds__(STEP_THREADS, (K <= 16 ? 10 : 4)) k_covariance(const CloudDev* clouds, int k, int method) {
  const CloudDev& c = clouds[blockIdx.y];
  const int i = blockIdx.x * STEP_THREADS + threadIdx.x;
  __shared__ float s_hd[K][STEP_THREADS];
  __shared__ int s_hp[K][STEP_THREADS];
  if (i >= c.n) return;
  const float4 q = c.pts[i];
  int nb[K];  // neighbour positions for the covariance
  {
    KnnHeap<K, STEP_THREADS> res;
    res.hd = &s_hd[0][threadIdx.x];
    res.hp = &s_hp[0][threadIdx.x];
    cov_knn<KnnHeap<K, STEP_THREADS>, K>(c, i, q, res);
    if (res.ev == res.worst()) {  // cold: an entry tied at the final cut may have been evicted for a higher index (KnnHeap);
                                  // the exact search rewrites the same shared-memory columns, which the pops below read
      KnnHeap<K, STEP_THREADS, true> ex;
      ex.hd = res.hd;
      ex.hp = res.hp;
      cov_knn<KnnHeap<K, STEP_THREADS, true>, K>(c, i, q, ex);
    }
    int m = K;
    while (m > k) m = res.pop(m, c.pts);  // k < K: drop the K - k farthest
#pragma unroll
    for (int j = 0; j < K; j++) nb[j] = res.p(j);
  }
  // two passes over the K neighbours (second pass hits L1) instead of parking 3K doubles in registers
  double mx = 0, my = 0, mz = 0;
#pragma unroll
  for (int j = 0; j < K; j++) {
    if (j < k && nb[j] >= 0) {
      const float4 p = __ldg(&c.pts[nb[j]]);
      mx += (double)p.x; my += (double)p.y; mz += (double)p.z;
    }
  }
  mx /= k; my /= k; mz /= k;
  double cxx = 0, cxy = 0, cxz = 0, cyy = 0, cyz = 0, czz = 0;
#pragma unroll
  for (int j = 0; j < K; j++) {
    if (j < k && nb[j] >= 0) {
      const float4 p = __ldg(&c.pts[nb[j]]);
      const double dx = (double)p.x - mx, dy = (double)p.y - my, dz = (double)p.z - mz;
      cxx += dx * dx; cxy += dx * dy; cxz += dx * dz; cyy += dy * dy; cyz += dy * dz; czz += dz * dz;
    }
  }
  const double ik = 1.0 / k;
  cxx *= ik; cxy *= ik; cxz *= ik; cyy *= ik; cyz *= ik; czz *= ik;
  cov_regularize_store(c.cov + (size_t)i * 6, cxx, cxy, cxz, cyy, cyz, czz, method);
}

// ---------------------------------------------------------------------------------------
// K3/K4/K5: one LM step = two kernels over the device-side schedule of (active pair, 128-point block) work items
// (LmSched, internal.cuh), both persistent (work items are strided over the grid):
//   k_gicp_search  pairs in PH_LINEARIZE / PH_FITNESS: q = T_f p in fp32, exact 1-NN in the target tree (seeded with the
//                  previous correspondence), correspondence gate; writes corr / sqd.            [update_correspondences,
//                  32 registers, 16 blocks per SM: the walk is a chain of dependent L1/L2 loads,   getFitnessScore's search]
//                  so it runs at full occupancy instead of sharing the fp64 kernel's 64-register budget
//   k_gicp_accum   PH_LINEARIZE: M = (C_B + R C_A R^T)^-1, e, J, accumulate H (21), b (6), e^T M e        [linearize]
//                  PH_TRIAL:     e^T M e at the trial pose with the stale correspondences / M         [compute_error]
//                  PH_FITNESS:   sum of the 1-NN d^2                                               [getFitnessScore]
//                  Block partials go to HBM; the last block of a pair sums them in a fixed order (deterministic, SURVEY
//                  App. A.6) and runs the LM controller; the last block of the STEP rebuilds the schedule from the pairs'
//                  new phases -- no host round trip per iteration, finished pairs cost nothing from the next step on.
// ---------------------------------------------------------------------------------------
// The step's slot list in shared memory: the first n_cached entries (dynamic shared memory of lm_slot_cache(arena
// capacity) entries, sized where the kernels are launched), beyond that straight from global memory.  A context that runs
// 16-pair jobs (arena of 24 pairs) caches 384 B instead of reserving LM_SMEM_SLOTS (8 KB) per block: the rest of the
// SM's L1 / shared memory stays L1.
struct SlotView {
  const LmSlot* g;
  const LmSlot* sh;
  int n_cached;
  __device__ __forceinline__ LmSlot get(int k) const { return k < n_cached ? sh[k] : g[k]; }
};
__device__ __forceinline__ void load_slots(const LmSched* sched, int n_active, int n_cached, LmSlot* sh) {
  const int4* src = reinterpret_cast<const int4*>(sched->slots);
  int4* dst = reinterpret_cast<int4*>(sh);
  for (int k = threadIdx.x; k < min(n_active, n_cached); k += blockDim.x) dst[k] = __ldcg(&src[k]);
  __syncthreads();
}

__global__ void __launch_bounds__(STEP_THREADS, 16) k_gicp_search(const PairDev* pairs, const PairState* states, const LmCall* call,
                                                                const LmSched* sched, int n_cached) {
  __shared__ float s_Tf[12];
  __shared__ int2 s_stack[SEARCH_STACK][STEP_THREADS];
  extern __shared__ __align__(16) LmSlot s_slots[];  // [n_cached]
  const double max_corr_dist2 = call->prm.max_corr_dist2;
  const int total_items = sched->total_items;
  const int n_active = sched->n_active;
  const int stride = sched->stride;
  if ((int)blockIdx.x >= total_items) return;
  load_slots(sched, n_active, n_cached, s_slots);
  const SlotView slots{sched->slots, s_slots, n_cached};
  for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int slot = item / stride, blk = item - slot * stride;
    const LmSlot sl = slots.get(slot);
    const int phase = sl.phase;
    if (blk >= sl.nblk || (phase != PH_LINEARIZE && phase != PH_FITNESS)) continue;  // block-uniform
    const PairState* st = &states[sl.pair];
    const PairDev& P = pairs[sl.pair];
    const bool seeded = sl.seeded != 0;  // P.corr holds the previous linearization's correspondences
    __syncthreads();
    if (threadIdx.x < 12) {
      const int r = threadIdx.x / 4, cc = threadIdx.x % 4;
      s_Tf[threadIdx.x] = phase == PH_FITNESS ? st->Tf[threadIdx.x] : (float)(cc < 3 ? st->R[3 * r + cc] : st->t[r]);
    }
    __syncthreads();
    const int i = blk * STEP_THREADS + threadIdx.x;
    if (i >= P.src.n) continue;
    const float4 p = P.src.pts[i];
    float qx, qy, qz;
    if (phase == PH_LINEARIZE) {
      // trans_f * p, summation order ((r0 x + r1 y) + r2 z) + t, no fma (SURVEY App. A.4)
      qx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_Tf[0], p.x), __fmul_rn(s_Tf[1], p.y)), __fmul_rn(s_Tf[2], p.z)), s_Tf[3]);
      qy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_Tf[4], p.x), __fmul_rn(s_Tf[5], p.y)), __fmul_rn(s_Tf[6], p.z)), s_Tf[7]);
      qz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s_Tf[8], p.x), __fmul_rn(s_Tf[9], p.y)), __fmul_rn(s_Tf[10], p.z)), s_Tf[11]);
    } else {  // pcl::transformPointCloud fp32 order x*c0 + (y*c1 + (z*c2 + c3))
      qx = __fadd_rn(__fmul_rn(s_Tf[0], p.x), __fadd_rn(__fmul_rn(s_Tf[1], p.y), __fadd_rn(__fmul_rn(s_Tf[2], p.z), s_Tf[3])));
      qy = __fadd_rn(__fmul_rn(s_Tf[4], p.x), __fadd_rn(__fmul_rn(s_Tf[5], p.y), __fadd_rn(__fmul_rn(s_Tf[6], p.z), s_Tf[7])));
      qz = __fadd_rn(__fmul_rn(s_Tf[8], p.x), __fadd_rn(__fmul_rn(s_Tf[9], p.y), __fadd_rn(__fmul_rn(s_Tf[10], p.z), s_Tf[11])));
    }
    KnnSet<1> res;
    res.init();
    if (seeded) {  // last iteration's correspondence is almost always still the nearest point: start with its bound
      const int pp = P.corr[i];
      if (pp >= 0) {
        const float4 t = __ldg(&P.tgt.pts[pp]);
        res.d[0] = dist2_rn(qx, qy, qz, t.x, t.y, t.z);
        res.p[0] = pp;
      }
    }
    knn_walk<SEARCH_STACK, STEP_THREADS>(P.tgt, qx, qy, qz, res, &s_stack[0][threadIdx.x]);
    P.sqd[i] = res.d[0];
    // PH_FITNESS keeps the ungated nearest position: nothing reads corr after that pass but the residual capture
    P.corr[i] = (phase == PH_FITNESS || (double)res.d[0] < max_corr_dist2) ? res.p[0] : -1;
  }
}

// Accumulate kernel: NO barrier, NO atomic, NO fence.  A work item is still a 128-point block of a pair, but every warp
// reduces its own 32 points and writes its own partial row (28 doubles for a linearize pass, 1 otherwise); the controller
// kernel sums the rows in a fixed order.  (Round 1 and the first version of this round reduced per block and let the
// last-arriving block of a pair run the controller: four __syncthreads, a __threadfence and an atomic round trip per item
// made the streaming phases barrier- and latency-bound, ncu: barrier 7.9 / long-scoreboard 17 stalled warps per issue.)
// 4 blocks per SM (up to 128 registers): the linearize pass holds the 28 fp64 values plus the inputs of M, J and e and
// needs 116 registers.  Under the 64-register cap of 8 blocks per SM it spilled 324 B per thread, more than the pass's
// own loads, and ran 1.7x longer (DESIGN.md §3); 6 blocks (80 registers) still spill 84 B.
__global__ void __launch_bounds__(STEP_THREADS, 4) k_gicp_accum(const PairDev* pairs, const PairState* states, const LmSched* sched,
                                                               int n_cached) {
  extern __shared__ __align__(16) LmSlot s_slots[];  // [n_cached]
  const int total_items = sched->total_items;
  const int n_active = sched->n_active;
  const int stride = sched->stride;
  if ((int)blockIdx.x >= total_items) return;
  load_slots(sched, n_active, n_cached, s_slots);
  const SlotView slots{sched->slots, s_slots, n_cached};
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int slot = item / stride, blk = item - slot * stride;
    const LmSlot sl = slots.get(slot);
    if (blk >= sl.nblk) continue;  // a shorter pair's padding item
    const PairDev& P = pairs[sl.pair];
    const PairState* st = &states[sl.pair];
    const int N = P.src.n;
    const int phase = sl.phase;
    const int i0 = blk * STEP_THREADS + warp * 32;  // this warp's 32 points
    if (i0 >= N) continue;
    const int i = i0 + lane;
    double* row = P.partial + (size_t)(blk * (STEP_THREADS / 32) + warp) * NRED;
    // pose of this phase: x0 for the linearize pass, the trial pose for compute_error (same address for the whole warp)
    double T[12];
    if (phase != PH_FITNESS) {
      const double* Rp = phase == PH_TRIAL ? st->Rt : st->R;
      const double* tp = phase == PH_TRIAL ? st->tt : st->t;
#pragma unroll
      for (int r = 0; r < 3; r++) {
#pragma unroll
        for (int c = 0; c < 3; c++) T[4 * r + c] = Rp[3 * r + c];
        T[4 * r + 3] = tp[r];
      }
    }
    if (phase == PH_LINEARIZE) {
      double v[NRED];
#pragma unroll
      for (int k = 0; k < NRED; k++) v[k] = 0.0;
      const int pos = i < N ? P.corr[i] : -1;  // this step's k_gicp_search
      if (pos >= 0) {
        const float4 p = P.src.pts[i];
        const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
        double ca[6], cb[6], rcr[6], M[6];
        const double2* pa = reinterpret_cast<const double2*>(P.src.cov + (size_t)i * 6);
        const double2* pb = reinterpret_cast<const double2*>(P.tgt.cov + (size_t)pos * 6);
#pragma unroll
        for (int k = 0; k < 3; k++) {
          double2 a = pa[k], b = __ldg(&pb[k]);
          ca[2 * k] = a.x; ca[2 * k + 1] = a.y;
          cb[2 * k] = b.x; cb[2 * k + 1] = b.y;
        }
        rcrt(R, ca, rcr);
#pragma unroll
        for (int k = 0; k < 6; k++) rcr[k] += cb[k];
        sym3_inverse(rcr, M);
        double2* pm = reinterpret_cast<double2*>(P.mahal + (size_t)i * 6);
        pm[0] = make_double2(M[0], M[1]);
        pm[1] = make_double2(M[2], M[3]);
        pm[2] = make_double2(M[4], M[5]);
        const float4 pbt = __ldg(&P.tgt.pts[pos]);
        const double ax = p.x, ay = p.y, az = p.z;
        const double ta[3] = {R[0] * ax + R[1] * ay + R[2] * az + T[3], R[3] * ax + R[4] * ay + R[5] * az + T[7],
                              R[6] * ax + R[7] * ay + R[8] * az + T[11]};
        const double e[3] = {(double)pbt.x - ta[0], (double)pbt.y - ta[1], (double)pbt.z - ta[2]};
        const double Mf[3][3] = {{M[0], M[1], M[2]}, {M[1], M[3], M[4]}, {M[2], M[4], M[5]}};
        double Me[3];
#pragma unroll
        for (int r = 0; r < 3; r++) Me[r] = Mf[r][0] * e[0] + Mf[r][1] * e[1] + Mf[r][2] * e[2];
        // J = [skew(T a) | -I]
        const double J[3][6] = {{0.0, -ta[2], ta[1], -1.0, 0.0, 0.0}, {ta[2], 0.0, -ta[0], 0.0, -1.0, 0.0}, {-ta[1], ta[0], 0.0, 0.0, 0.0, -1.0}};
        double MJ[3][6];
#pragma unroll
        for (int r = 0; r < 3; r++)
#pragma unroll
          for (int c = 0; c < 6; c++) MJ[r][c] = Mf[r][0] * J[0][c] + Mf[r][1] * J[1][c] + Mf[r][2] * J[2][c];
        int k = 0;
#pragma unroll
        for (int r = 0; r < 6; r++)
#pragma unroll
          for (int c = r; c < 6; c++) v[k++] = J[0][r] * MJ[0][c] + J[1][r] * MJ[1][c] + J[2][r] * MJ[2][c];
#pragma unroll
        for (int r = 0; r < 6; r++) v[21 + r] = J[0][r] * Me[0] + J[1][r] * Me[1] + J[2][r] * Me[2];
        v[27] = e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2];
      }
      // 28 values at once with a transposing butterfly: at step m every lane keeps half of its values and trades the other
      // half, so after 5 steps lane L holds the warp total of value L (31 shuffles of doubles instead of 28 * 5)
      double w[32];
#pragma unroll
      for (int k = 0; k < 32; k++) w[k] = k < NRED ? v[k] : 0.0;
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) {
        const bool up = (lane & m) != 0;
#pragma unroll
        for (int k = 0; k < m; k++) {
          const double keep = up ? w[k + m] : w[k];
          const double send = up ? w[k] : w[k + m];
          w[k] = keep + __shfl_xor_sync(0xffffffffu, send, m);
        }
      }
      if (lane < NRED) row[lane] = w[0];
    } else {
      double x = 0.0;
      if (i < N) {
        if (phase == PH_TRIAL) {
          const int pos = P.corr[i];
          if (pos >= 0) {
            const float4 p = P.src.pts[i];
            const float4 pbt = __ldg(&P.tgt.pts[pos]);
            const double ax = p.x, ay = p.y, az = p.z;
            const double e0 = (double)pbt.x - (T[0] * ax + T[1] * ay + T[2] * az + T[3]);
            const double e1 = (double)pbt.y - (T[4] * ax + T[5] * ay + T[6] * az + T[7]);
            const double e2 = (double)pbt.z - (T[8] * ax + T[9] * ay + T[10] * az + T[11]);
            const double2* pm = reinterpret_cast<const double2*>(P.mahal + (size_t)i * 6);
            const double2 m01 = pm[0], m23 = pm[1], m45 = pm[2];
            const double Me0 = m01.x * e0 + m01.y * e1 + m23.x * e2;
            const double Me1 = m01.y * e0 + m23.y * e1 + m45.x * e2;
            const double Me2 = m23.x * e0 + m45.x * e1 + m45.y * e2;
            x = e0 * Me0 + e1 * Me1 + e2 * Me2;
          }
        } else {  // PH_FITNESS: the 1-NN d^2 this step's k_gicp_search found
          x = (double)P.sqd[i];
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
      if (lane == 0) row[0] = x;
    }
  }
}

// Controller kernel: one block per active pair (strided over a fixed grid) sums the pair's partial rows in a FIXED order
// (32 interleaved chains per column, then a fixed 32-way add: deterministic, SURVEY App. A.6) and runs the LM state machine;
// the last block to finish rebuilds the schedule and sets the loop condition of the solve's while node.
constexpr int CTRL_THREADS = 1024;  // 32 interleaved chains per column: the row sums are latency chains, not bandwidth
__global__ void __launch_bounds__(CTRL_THREADS) k_gicp_control(const PairDev* pairs, PairState* states, LmCall* call, LmSched* sched) {
  __shared__ double s_red[CTRL_THREADS / 32][NRED];
  __shared__ bool s_last;
  const int n_active = sched->n_active;
  const int j = threadIdx.x & 31, g = threadIdx.x >> 5;
  for (int slot = blockIdx.x; slot < n_active; slot += gridDim.x) {
    const LmSlot sl = sched->slots[slot];
    const PairDev& P = pairs[sl.pair];
    const int N = P.src.n;
    const int nrows = (N + 31) / 32;
    const int nred = sl.phase == PH_LINEARIZE ? NRED : 1;
    double x = 0;
    if (j < nred)
      for (int r = g; r < nrows; r += CTRL_THREADS / 32) x += __ldcg(&P.partial[(size_t)r * NRED + j]);
    __syncthreads();
    if (j < NRED) s_red[g][j] = x;
    __syncthreads();
    if (threadIdx.x == 0) {
      double sums[NRED];
      for (int k = 0; k < nred; k++) {
        double s = 0;
        for (int w = 0; w < CTRL_THREADS / 32; w++) s += s_red[w][k];
        sums[k] = s;
      }
      b200reg_lm_trial* trace = call->trace ? call->trace + (size_t)sl.pair * call->trace_stride : nullptr;
      lm_update(&states[sl.pair], sums, call->prm, sl.phase, N, &sched->done, trace);
    }
  }
  // ---- end of the step: the last block to get here rebuilds the schedule from the pairs' new phases
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(&sched->arrive, 1u);
    s_last = (prev == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x == 0) sched->steps++;
  __syncthreads();
  sched_rebuild(pairs, states, sched, call);
}

// ---------------------------------------------------------------------------------------
// debug tap: k-NN of arbitrary queries, results as ORIGINAL indices
// ---------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(STEP_THREADS) k_knn_queries(CloudDev c, const float* q, int nq, int qstride, int kout, int* idx_out,
                                                               float* d2_out) {
  int i = blockIdx.x * STEP_THREADS + threadIdx.x;
  if (i >= nq) return;
  const float* qq = q + (size_t)i * qstride;
  KnnSet<K> res;
  res.init();
  knn_walk(c, qq[0], qq[1], qq[2], res);  // a debug tap: the stack stays in local memory
#pragma unroll
  for (int j = 0; j < K; j++) {
    if (j < kout) {
      idx_out[(size_t)i * kout + j] = res.p[j] >= 0 ? __float_as_int(c.pts[res.p[j]].w) : -1;
      d2_out[(size_t)i * kout + j] = res.d[j];
    }
  }
}

// ---------------------------------------------------------------------------------------
// debug tap: brute-force exact k-NN, the on-GPU anchor the LBVH traversal is checked against at full size
// (SURVEY.md §7 step 4a).  One query per thread; the cloud streams through shared memory in 8 KB tiles staged by
// TMA bulk copies (mbarrier double buffer); all lanes read the same staged point (broadcast, conflict free).
// ---------------------------------------------------------------------------------------
constexpr int BF_TILE = 512;

__device__ __forceinline__ unsigned bf_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

template <int K>
__global__ void __launch_bounds__(STEP_THREADS) k_knn_brute(CloudDev c, const float* q, int nq, int qstride, int kout, int* idx_out,
                                                            float* d2_out) {
  __shared__ __align__(128) float4 tile[2][BF_TILE];
  __shared__ __align__(8) unsigned long long full[2];
  const int i = blockIdx.x * STEP_THREADS + threadIdx.x;
  const bool active = i < nq;
  const float* qq = q + (size_t)(active ? i : 0) * qstride;
  const float qx = qq[0], qy = qq[1], qz = qq[2];
  KnnSet<K> res;
  res.init();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bf_smem_u32(&full[0])), "r"(1));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bf_smem_u32(&full[1])), "r"(1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int ntiles = (c.n + BF_TILE - 1) / BF_TILE;
  auto issue = [&](int t) {
    const unsigned bytes = (unsigned)min(BF_TILE, c.n - t * BF_TILE) * 16u;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bf_smem_u32(&full[t & 1])), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(bf_smem_u32(tile[t & 1])),
                 "l"(c.pts + (size_t)t * BF_TILE), "r"(bytes), "r"(bf_smem_u32(&full[t & 1]))
                 : "memory");
  };
  if (threadIdx.x == 0) issue(0);
  for (int t = 0; t < ntiles; t++) {
    if (threadIdx.x == 0 && t + 1 < ntiles) issue(t + 1);
    unsigned ok = 0;
    while (!ok)
      asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                   : "=r"(ok)
                   : "r"(bf_smem_u32(&full[t & 1])), "r"((unsigned)((t >> 1) & 1))
                   : "memory");
    const int cnt = min(BF_TILE, c.n - t * BF_TILE);
    if (active) {
      for (int j = 0; j < cnt; j++) {
        const float4 p = tile[t & 1][j];
        const float d2 = dist2_rn(qx, qy, qz, p.x, p.y, p.z);
        if (!(d2 > res.worst())) res.offer(d2, t * BF_TILE + j, c.pts);
      }
    }
    __syncthreads();
  }
  if (active) {
#pragma unroll
    for (int j = 0; j < K; j++) {
      if (j < kout) {
        idx_out[(size_t)i * kout + j] = res.p[j] >= 0 ? __float_as_int(c.pts[res.p[j]].w) : -1;
        d2_out[(size_t)i * kout + j] = res.d[j];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// debug tap: the LM controller (lm_prepare_trial / lm_update, the functions the solve runs) on caller-supplied states,
// one thread per case (b200reg_lm_step_tap)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_lm_step_tap(const b200reg_lm_case* cases, int n, b200reg_lm_step* out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const b200reg_lm_case& c = cases[k];
  GicpParamsDev prm;  // the fields lm_update reads
  prm.max_iterations = c.params.max_iterations;
  prm.lm_max_iterations = c.params.lm_max_iterations;
  prm.max_corr_dist2 = 0.0;
  prm.transformation_eps = c.params.transformation_eps;
  prm.rotation_eps = c.params.rotation_eps;
  prm.lm_init_lambda_factor = c.params.lm_init_lambda_factor;
  prm.icp_score_thr = 0.0;
  PairState st;
  memset(&st, 0, sizeof(st));
  for (int i = 0; i < 9; i++) st.R[i] = c.R[i];
  for (int i = 0; i < 3; i++) st.t[i] = c.t[i];
  st.lambda = c.lambda;
  st.nu = c.nu;
  st.outer_it = c.outer_it;
  st.inner_it = c.inner_it;
  st.nr_iterations = c.outer_it;
  st.phase = PH_LINEARIZE;
  double sums[NRED];
  int q = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) sums[q++] = c.H[6 * i + j];  // the upper triangle, as k_gicp_control hands it over
  for (int i = 0; i < 6; i++) sums[21 + i] = c.b[i];
  sums[27] = c.y0;
  b200reg_lm_step& o = out[k];
  memset(&o, 0, sizeof(o));
  if (c.mode == 0) {
    lm_update(&st, sums, prm, PH_LINEARIZE, 0, nullptr, nullptr);
  } else {
    for (int i = 0; i < 36; i++) st.H[i] = c.H[i];
    for (int i = 0; i < 6; i++) st.b[i] = c.b[i];
    st.y0 = c.y0;
    lm_prepare_trial(&st);
  }
  // the trial this call prepared (a rejection prepares the next one: these are the values before the decision)
  for (int i = 0; i < 6; i++) o.d[i] = st.d[i];
  for (int i = 0; i < 9; i++) {
    o.dR[i] = st.dR[i];
    o.Rt[i] = st.Rt[i];
  }
  for (int i = 0; i < 3; i++) {
    o.dt[i] = st.dt[i];
    o.tt[i] = st.tt[i];
  }
  o.has_trial = st.phase == PH_TRIAL;
  if (c.mode != 0 && o.has_trial) {
    const double yi[1] = {c.yi};
    lm_update(&st, yi, prm, PH_TRIAL, 0, nullptr, &o.record);
  }
  o.lambda = st.lambda;
  o.nu = st.nu;
  o.phase = st.phase;
  o.converged = st.converged;
  o.lm_failed = st.lm_failed;
  o.outer_it = st.outer_it;
  o.inner_it = st.inner_it;
  for (int i = 0; i < 9; i++) o.R[i] = st.R[i];
  for (int i = 0; i < 3; i++) o.t[i] = st.t[i];
}

int launch_lm_step_tap(const b200reg_lm_case* d_cases, int n, b200reg_lm_step* d_out, cudaStream_t s) {
  if (n <= 0) return 0;
  k_lm_step_tap<<<(n + 127) / 128, 128, 0, s>>>(d_cases, n, d_out);
  return 1;
}

// setSourceCovariances / setTargetCovariances: caller's 3x3 blocks (original order) -> packed symmetric, sorted order
__global__ void __launch_bounds__(256) k_set_covariances(CloudDev c, const double* cov9) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.n) return;
  const double* m = cov9 + (size_t)__float_as_int(c.pts[i].w) * 9;
  double* o = c.cov + (size_t)i * 6;
  o[0] = m[0]; o[1] = m[1]; o[2] = m[2]; o[3] = m[4]; o[4] = m[5]; o[5] = m[8];  // upper triangle of the row-major block
}

// output cloud: final fp32 transform in the pcl::transformPointCloud order, ORIGINAL point order
__global__ void __launch_bounds__(256) k_transform_out(CloudDev c, const float* Tf, float* out3) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.n) return;
  const float4 p = c.pts[i];
  const size_t o = (size_t)__float_as_int(p.w) * 3;
  const float3 q = transform_out_point(Tf, p.x, p.y, p.z);
  out3[o] = q.x;
  out3[o + 1] = q.y;
  out3[o + 2] = q.z;
}

// residual capture (b200reg_residuals): the fitness pass's per-point values of every pair of a call, scattered from sorted
// source position to ORIGINAL source index; the nearest target position becomes the target point's original index
__global__ void __launch_bounds__(256) k_residual_rows(const ResidualRow* rows, ResidualOut out) {
  const ResidualRow& R = rows[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R.n) return;
  const long long o = R.off + __float_as_int(R.spts[i].w);
  const int p = R.corr[i];
  out.nn[o] = p >= 0 ? __float_as_int(R.tpts[p].w) : -1;
  out.d2[o] = R.sqd[i];
}

// ---------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------
void launch_residual_rows(const ResidualRow* d_rows, int count, int max_n, ResidualOut out, cudaStream_t s) {
  k_residual_rows<<<dim3((max_n + 255) / 256, count), 256, 0, s>>>(d_rows, out);
}

int launch_covariances(const CloudDev* d_clouds, int count, int max_n, int k, int method, unsigned long long* slab, cudaStream_t s) {
  dim3 grid((max_n + STEP_THREADS - 1) / STEP_THREADS, count);
  if (k < 1 || method < 0 || method > 4) return -1;
  if (k > 32) return launch_covariance_large(d_clouds, count, max_n, k, method, slab, s);
  if (k <= 8) k_covariance<8><<<grid, STEP_THREADS, 0, s>>>(d_clouds, k, method);
  else if (k <= 15) k_covariance<15><<<grid, STEP_THREADS, 0, s>>>(d_clouds, k, method);
  else if (k <= 20) k_covariance<20><<<grid, STEP_THREADS, 0, s>>>(d_clouds, k, method);
  else k_covariance<32><<<grid, STEP_THREADS, 0, s>>>(d_clouds, k, method);
  return 1;
}

void launch_gicp_init(const PairDev* pairs, PairState* states, const double* d_guess, LmCall* call, LmSched* sched, cudaStream_t s) {
  k_gicp_init<<<1, 256, 0, s>>>(pairs, states, d_guess, call, sched);
}

// One LM step over every still-active pair = search + accumulate + controller.  blocks_*: persistent grid sizes (work
// items are strided over them); the kernels are correct for any value >= 1.
constexpr int CTRL_BLOCKS = 64;
void launch_gicp_search(const PairDev* pairs, const PairState* states, int blocks, const LmCall* call, const LmSched* sched, int n_cached,
                        cudaStream_t s) {
  k_gicp_search<<<blocks, STEP_THREADS, sizeof(LmSlot) * n_cached, s>>>(pairs, states, call, sched, n_cached);
}
void launch_gicp_accum(const PairDev* pairs, const PairState* states, int blocks, const LmSched* sched, int n_cached, cudaStream_t s) {
  k_gicp_accum<<<blocks, STEP_THREADS, sizeof(LmSlot) * n_cached, s>>>(pairs, states, sched, n_cached);
}
void launch_gicp_control(const PairDev* pairs, PairState* states, LmCall* call, LmSched* sched, cudaStream_t s) {
  k_gicp_control<<<CTRL_BLOCKS, CTRL_THREADS, 0, s>>>(pairs, states, call, sched);
}

// The whole solve as ONE CUDA graph: init kernel, then a WHILE node whose body is the three step kernels; the controller's
// last block sets the loop condition (cudaGraphSetConditional) from the device-side schedule.  The host launches
// the graph once per solve and synchronises once -- no polling, no chunking (round 1 polled a counter every 8 launches).
// All kernel arguments are pointers into the context's persistent LM arena, so the executable graph is reused by every call
// until the arena grows.
cudaError_t lm_graph_build(LmGraph* g, const PairDev* pairs, PairState* states, const double* guess, LmCall* call, LmSched* sched,
                           int blocks_search, int blocks_accum, int n_cached) {
  cudaError_t e;
  if ((e = cudaGraphCreate(&g->graph, 0)) != cudaSuccess) return e;
  cudaGraphNode_t n_init, n_while, n_search, n_accum, n_ctrl;
  {
    void* args[] = {(void*)&pairs, (void*)&states, (void*)&guess, (void*)&call, (void*)&sched};
    cudaKernelNodeParams kp = {};
    kp.func = (void*)k_gicp_init;
    kp.gridDim = dim3(1);
    kp.blockDim = dim3(256);
    kp.kernelParams = args;
    if ((e = cudaGraphAddKernelNode(&n_init, g->graph, nullptr, 0, &kp)) != cudaSuccess) return e;
  }
  cudaGraphConditionalHandle h;
  if ((e = cudaGraphConditionalHandleCreate(&h, g->graph, 1, cudaGraphCondAssignDefault)) != cudaSuccess) return e;
  g->cond_handle = (unsigned long long)h;
  cudaGraphNodeParams wp = {};
  wp.type = cudaGraphNodeTypeConditional;
  wp.conditional.handle = h;
  wp.conditional.type = cudaGraphCondTypeWhile;
  wp.conditional.size = 1;
  if ((e = cudaGraphAddNode(&n_while, g->graph, &n_init, 1, &wp)) != cudaSuccess) return e;
  cudaGraph_t body = wp.conditional.phGraph_out[0];
  const PairState* cstates = states;
  const LmCall* ccall = call;
  const LmSched* csched = sched;
  {
    void* args[] = {(void*)&pairs, (void*)&cstates, (void*)&ccall, (void*)&csched, (void*)&n_cached};
    cudaKernelNodeParams kp = {};
    kp.func = (void*)k_gicp_search;
    kp.gridDim = dim3(blocks_search);
    kp.blockDim = dim3(STEP_THREADS);
    kp.sharedMemBytes = sizeof(LmSlot) * n_cached;
    kp.kernelParams = args;
    if ((e = cudaGraphAddKernelNode(&n_search, body, nullptr, 0, &kp)) != cudaSuccess) return e;
  }
  {
    void* args[] = {(void*)&pairs, (void*)&cstates, (void*)&csched, (void*)&n_cached};
    cudaKernelNodeParams kp = {};
    kp.func = (void*)k_gicp_accum;
    kp.gridDim = dim3(blocks_accum);
    kp.blockDim = dim3(STEP_THREADS);
    kp.sharedMemBytes = sizeof(LmSlot) * n_cached;
    kp.kernelParams = args;
    if ((e = cudaGraphAddKernelNode(&n_accum, body, &n_search, 1, &kp)) != cudaSuccess) return e;
  }
  {
    void* args[] = {(void*)&pairs, (void*)&states, (void*)&call, (void*)&sched};
    cudaKernelNodeParams kp = {};
    kp.func = (void*)k_gicp_control;
    kp.gridDim = dim3(CTRL_BLOCKS);
    kp.blockDim = dim3(CTRL_THREADS);
    kp.kernelParams = args;
    if ((e = cudaGraphAddKernelNode(&n_ctrl, body, &n_accum, 1, &kp)) != cudaSuccess) return e;
  }
  return cudaGraphInstantiate(&g->exec, g->graph, 0);
}

void lm_graph_destroy(LmGraph* g) {
  if (g->exec) cudaGraphExecDestroy(g->exec);
  if (g->graph) cudaGraphDestroy(g->graph);
  g->exec = nullptr;
  g->graph = nullptr;
  g->cond_handle = 0;
}

int launch_knn_queries(const CloudDev& c, const float* d_q, int nq, int qstride, int k, int* idx, float* d2, cudaStream_t s, int brute) {
  dim3 grid((nq + STEP_THREADS - 1) / STEP_THREADS);
  if (brute) {
    if (k == 1) k_knn_brute<1><<<grid, STEP_THREADS, 0, s>>>(c, d_q, nq, qstride, k, idx, d2);
    else if (k <= 15) k_knn_brute<15><<<grid, STEP_THREADS, 0, s>>>(c, d_q, nq, qstride, k, idx, d2);
    else if (k <= 32) k_knn_brute<32><<<grid, STEP_THREADS, 0, s>>>(c, d_q, nq, qstride, k, idx, d2);
    else return -1;
    return 1;
  }
  if (k == 1) k_knn_queries<1><<<grid, STEP_THREADS, 0, s>>>(c, d_q, nq, qstride, k, idx, d2);
  else if (k <= 8) k_knn_queries<8><<<grid, STEP_THREADS, 0, s>>>(c, d_q, nq, qstride, k, idx, d2);
  else if (k <= 15) k_knn_queries<15><<<grid, STEP_THREADS, 0, s>>>(c, d_q, nq, qstride, k, idx, d2);
  else if (k <= 20) k_knn_queries<20><<<grid, STEP_THREADS, 0, s>>>(c, d_q, nq, qstride, k, idx, d2);
  else if (k <= 32) k_knn_queries<32><<<grid, STEP_THREADS, 0, s>>>(c, d_q, nq, qstride, k, idx, d2);
  else return -1;
  return 1;
}

void launch_set_covariances(const CloudDev& c, const double* d_cov9, cudaStream_t s) {
  k_set_covariances<<<(c.n + 255) / 256, 256, 0, s>>>(c, d_cov9);
}

void launch_transform_out(const CloudDev& c, const float* d_Tf, float* d_out3, cudaStream_t s) {
  k_transform_out<<<(c.n + 255) / 256, 256, 0, s>>>(c, d_Tf, d_out3);
}

}  // namespace b200
