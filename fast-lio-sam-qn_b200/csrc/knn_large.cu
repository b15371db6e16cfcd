// knn_large.cu -- exact k-NN for k > 32 (b200reg_knn): one WARP per query.
//
// Replaces KdTreeFLANN::nearestKSearch (third_party/nano_gicp/include/nano_gicp/nanoflann.hpp:140-152) for any k.  The
// k <= 32 kernels (k_knn_queries in gicp.cu) keep their result set in registers, one thread per query; 33 to thousands of
// entries per thread fit neither registers nor a per-thread shared-memory heap (8 k bytes per thread).  Here the 32 lanes of
// a warp share one query:
//   * the result list is sorted 64-bit keys (bits(d2) << 32) | original index.  d2 is >= +0 (or NaN), so the unsigned order
//     of the keys IS the (d2, lower original index) order of SURVEY.md App. A.3: one integer compare, no tie path.  The list
//     starts as k copies of KL_PAD = (FLT_MAX, index -1), which is also what an unfilled slot reports, exactly as the k <= 32
//     path pads; a point is a candidate iff its key is below the current k-th key (so d2 = +inf or NaN never enters);
//   * the walk is knn_walk's (knn.cuh): the same LBVH records, dist2_rn for points, box_dist2_rn for boxes, the near child
//     first, the far child pushed unless its bound is strictly greater than the k-th d2, at most MAX_STACK entries (one push
//     per record, as knn_walk).  The stack is spread over the lanes' registers (entry e on lane e & 31), so it needs no
//     shared memory and no synchronisation;
//   * a leaf step takes up to four leaves -- the one reached plus leaves waiting on top of the stack -- one point per lane;
//   * lanes whose key beats the k-th key are ballot-compacted into a 64-entry staging buffer.  When it could overflow, and
//     once at the end, the warp sorts it (bitonic, one compare-exchange per lane and stage) and merges it into the list:
//     every entry's new position is its rank in the other sequence plus its own index (merge path), entries that land at k
//     or beyond drop out.  The new bound is entry k - 1;
//   * lists of up to KL_SMEM_K entries live in shared memory, longer ones in a per-query slab of device scratch: the same
//     code on a different pointer, so both tiers give identical answers.
// A query with a NaN coordinate has no neighbours (every d2 would be NaN): its row is all padding, as on the k <= 32 path; the
// kernel does not walk the tree for it.
// The answer is the k smallest keys of the cloud, a set that does not depend on the walk order: chunking, query order and
// repeated calls return identical bytes.
// k_covariance_large (b200reg_clouds_covariances_ex, k > 32) runs the same walk for every point of its clouds and sums the
// moments of the list it leaves.
#include <algorithm>
#include <climits>

#include "knn.cuh"
#include "launchers.cuh"
#include "smallmath.cuh"

namespace b200 {

constexpr int KL_WARPS = 4;  // queries per block
constexpr int KL_THREADS = 32 * KL_WARPS;
constexpr int KL_STAGE = 64;  // staging buffer; flushed when the next leaf step (<= 32 candidates) could overflow it
constexpr unsigned long long KL_PAD = (0x7F7FFFFFull << 32) | 0xFFFFFFFFull;  // (FLT_MAX, -1)
constexpr unsigned KL_FULL = 0xffffffffu;
static_assert(MAX_STACK == 64, "the register stack holds two entries per lane");
static_assert(LEAF <= 8, "a leaf step gives each of four leaves eight lanes");

// number of entries of the ascending a[0..n) below v
__device__ __forceinline__ int kl_below(const unsigned long long* a, int n, unsigned long long v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Exact k-NN of one query into list[0..k) (ascending keys).  Called by all 32 lanes of a warp; control flow is warp-uniform.
__device__ __forceinline__ void kl_walk(const CloudDev& c, float qx, float qy, float qz, int k, unsigned long long* list,
                                        unsigned long long* stage) {
  const float4* __restrict__ pts = c.pts;
  const float4* __restrict__ tn = c.tnodes;
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  unsigned long long kth = KL_PAD;
  float wd = __uint_as_float((unsigned)(KL_PAD >> 32));  // d2 of the k-th key: the pruning bound
  int ns = 0;                                            // staged candidates
  int sr0 = 0, sr1 = 0;                                  // stack entry e: ref and bound on lane e & 31, register e >> 5
  float sd0 = 0.f, sd1 = 0.f;
  int sp = 0;
  auto push = [&](int r, float d) {
    if (lane == (sp & 31)) {
      if (sp < 32) { sr0 = r; sd0 = d; }
      else { sr1 = r; sd1 = d; }
    }
    sp++;
  };
  auto stack_ref = [&](int e) { return __shfl_sync(KL_FULL, e < 32 ? sr0 : sr1, e & 31); };
  auto stack_d = [&](int e) { return __shfl_sync(KL_FULL, e < 32 ? sd0 : sd1, e & 31); };
  auto flush = [&]() {
    for (int i = ns + lane; i < KL_STAGE; i += 32) stage[i] = ~0ull;
    __syncwarp();
#pragma unroll
    for (int size = 2; size <= KL_STAGE; size <<= 1) {
#pragma unroll
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        const int i = 2 * stride * (lane / stride) + (lane % stride), j = i + stride;
        const unsigned long long a = stage[i], b = stage[j];
        if ((a > b) == ((i & size) == 0)) {
          stage[i] = b;
          stage[j] = a;
        }
        __syncwarp();
      }
    }
    // new position of a staged key: its index + the list entries below it (computed on the old list)
    const unsigned long long s0 = stage[lane], s1 = stage[lane + 32];
    const int p0 = lane < ns ? lane + kl_below(list, k, s0) : k;
    const int p1 = lane + 32 < ns ? lane + 32 + kl_below(list, k, s1) : k;
    const int lo = __shfl_sync(KL_FULL, p0, 0);  // list entries below the smallest staged key stay where they are
    __syncwarp();
    // list entry j moves up by the staged keys below it; top chunk first, so no entry is overwritten before it is read
    for (int hi = k; hi > lo; hi -= 32) {
      const int j = hi - 1 - lane;
      unsigned long long v = 0;
      int dst = k;
      if (j >= lo) {
        v = list[j];
        dst = j + kl_below(stage, KL_STAGE, v);
      }
      __syncwarp();
      if (dst < k) list[dst] = v;
      __syncwarp();
    }
    if (p0 < k) list[p0] = s0;
    if (p1 < k) list[p1] = s1;
    __syncwarp();
    kth = list[k - 1];
    wd = __uint_as_float((unsigned)(kth >> 32));
    ns = 0;
    __syncwarp();  // every lane has read the stage before it is refilled
  };

  int ref = c.root_ref;
  float dnode = 0.f;
  for (;;) {
    bool alive = !(dnode > wd);
    while (alive && ref >= 0) alive = near_far_step(load_node(tn, ref), qx, qy, qz, wd, ref, dnode, push);
    if (alive) {  // leaf step: this leaf and up to three more from the top of the stack
      int l1 = 0, l2 = 0, l3 = 0, nl = 1;
      while (nl < 4 && sp > 0) {
        const float d = stack_d(sp - 1);
        if (d > wd) {  // pruned for good: the bound only shrinks
          sp--;
          continue;
        }
        const int r = stack_ref(sp - 1);
        if (r >= 0) break;
        sp--;
        if (nl == 1) l1 = r;
        else if (nl == 2) l2 = r;
        else l3 = r;
        nl++;
      }
      const int t = lane >> 3, j = lane & 7;
      const LeafSpan leaf = leaf_span(t == 0 ? ref : t == 1 ? l1 : t == 2 ? l2 : l3);
      const int base = leaf.base, cnt = leaf.count;
      unsigned long long key = 0;
      bool take = false;
      if (t < nl && j < cnt) {
        const float4 p = __ldg(&pts[base + j]);
        key = ((unsigned long long)__float_as_uint(dist2_rn(qx, qy, qz, p.x, p.y, p.z)) << 32) | (unsigned)__float_as_int(p.w);
        take = key < kth;
      }
      const unsigned m = __ballot_sync(KL_FULL, take);
      if (take) stage[ns + __popc(m & lt)] = key;
      ns += __popc(m);
      if (ns > KL_STAGE - 32) {
        __syncwarp();
        flush();
      }
    }
    bool found = false;
    while (sp > 0) {
      sp--;
      const float d = stack_d(sp);
      if (!(d > wd)) {
        ref = stack_ref(sp);
        dnode = d;
        found = true;
        break;
      }
    }
    if (!found) break;
  }
  if (ns > 0) {
    __syncwarp();
    flush();
  }
}

// warp w of block b answers query b * KL_WARPS + w; SMEM_LIST: the list lives in shared memory (k <= KL_SMEM_K), else in
// slab[query * k ...]
template <bool SMEM_LIST>
__global__ void __launch_bounds__(KL_THREADS) k_knn_large(const __grid_constant__ CloudDev c, const float* q, int nq, int qstride, int k,
                                                          unsigned long long* slab, int* idx_out, float* d2_out) {
  __shared__ unsigned long long s_list[SMEM_LIST ? KL_WARPS * KL_SMEM_K : 1];
  __shared__ unsigned long long s_stage[KL_WARPS][KL_STAGE];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * KL_WARPS + warp;
  if (row >= nq) return;  // the whole warp
  unsigned long long* list = SMEM_LIST ? s_list + warp * KL_SMEM_K : slab + (size_t)row * k;
  const float* qq = q + (size_t)row * qstride;
  const float qx = qq[0], qy = qq[1], qz = qq[2];
  for (int j = lane; j < k; j += 32) list[j] = KL_PAD;
  __syncwarp();
  if (!(isnan(qx) || isnan(qy) || isnan(qz))) kl_walk(c, qx, qy, qz, k, list, s_stage[warp]);
  __syncwarp();
  for (int j = lane; j < k; j += 32) {
    const unsigned long long key = list[j];
    idx_out[(size_t)row * k + j] = (int)(unsigned)key;
    d2_out[(size_t)row * k + j] = __uint_as_float((unsigned)(key >> 32));
  }
}

// ---------------------------------------------------------------------------------------
// k > 32 covariances (nano_gicp_impl.hpp:298-357): one warp per point
// ---------------------------------------------------------------------------------------
// Work item it = cloud * max_n + point covers every cloud of the call in one launch; items past a cloud's size are skipped,
// and the items are strided over the grid's warps.  The neighbour list of a point is its m = min(k, n) nearest points of
// its own cloud (itself included), found by kl_walk: ascending (d2, original index), all of the cloud once k >= n.  A warp
// reuses one list for all its items: in shared memory when m <= KL_SMEM_K, else at slab + (global warp) * lstride.
// The moments follow the oracle's operation order (oracle_gicp.cpp:214-232, the reference's rowwise().mean() and
// / k_correspondences_), so the unregularised covariance is bit-identical to it wherever the lists agree: lanes 0..2 each
// sum one coordinate in list order and divide by k; lanes 0..5 then each sum one product (xa - ma) (xb - mb) in list order
// and divide by k -- fp64, no FMA, the divisor k even when fewer than k points exist.  (A lane-parallel tree sum would be
// faster but would not be that order.)  Lane 0 regularises and stores.
template <bool SMEM_LIST>
__global__ void __launch_bounds__(KL_THREADS) k_covariance_large(const CloudDev* clouds, int max_n, long long items, int k, int method,
                                                                 unsigned long long* slab, int lstride) {
  __shared__ unsigned long long s_list[SMEM_LIST ? KL_WARPS * KL_SMEM_K : 1];
  __shared__ unsigned long long s_stage[KL_WARPS][KL_STAGE];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long gw = (long long)blockIdx.x * KL_WARPS + warp;
  unsigned long long* list = SMEM_LIST ? s_list + warp * KL_SMEM_K : slab + gw * lstride;
  // the covariance term of lane t < 6: (xx, xy, xz, yy, yz, zz)
  const int ta = lane < 3 ? 0 : lane < 5 ? 1 : 2, tb = lane < 3 ? lane : lane < 5 ? lane - 2 : 2;
  const double dk = (double)k;
  for (long long it = gw; it < items; it += (long long)gridDim.x * KL_WARPS) {
    const CloudDev& c = clouds[it / max_n];
    const int i = (int)(it % max_n);
    if (i >= c.n) continue;  // the whole warp
    const int m = min(k, c.n);
    const float4 q = c.pts[i];
    for (int j = lane; j < m; j += 32) list[j] = KL_PAD;
    __syncwarp();
    if (!(isnan(q.x) || isnan(q.y) || isnan(q.z))) kl_walk(c, q.x, q.y, q.z, m, list, s_stage[warp]);
    __syncwarp();
    // original index -> sorted position, in place; padding (no neighbour) keeps index -1
    for (int j = lane; j < m; j += 32) {
      const unsigned o = (unsigned)list[j];
      if (o != 0xFFFFFFFFu) list[j] = (unsigned)c.rank[o];
    }
    __syncwarp();
    const float* __restrict__ pf = reinterpret_cast<const float*>(c.pts);
    double mean = 0.0;
    if (lane < 3) {
      for (int j = 0; j < m; j++) {
        const unsigned p = (unsigned)list[j];
        if (p != 0xFFFFFFFFu) mean = __dadd_rn(mean, (double)__ldg(&pf[4 * (size_t)p + lane]));
      }
      mean = __ddiv_rn(mean, dk);
    }
    const double mx = __shfl_sync(KL_FULL, mean, 0), my = __shfl_sync(KL_FULL, mean, 1), mz = __shfl_sync(KL_FULL, mean, 2);
    double acc = 0.0;
    if (lane < 6) {
      const double ma = ta == 0 ? mx : ta == 1 ? my : mz, mb = tb == 0 ? mx : tb == 1 ? my : mz;
      for (int j = 0; j < m; j++) {
        const unsigned p = (unsigned)list[j];
        if (p == 0xFFFFFFFFu) continue;
        const double da = __dsub_rn((double)__ldg(&pf[4 * (size_t)p + ta]), ma);
        const double db = __dsub_rn((double)__ldg(&pf[4 * (size_t)p + tb]), mb);
        acc = __dadd_rn(acc, __dmul_rn(da, db));
      }
      acc = __ddiv_rn(acc, dk);
    }
    double cv[6];
#pragma unroll
    for (int t = 0; t < 6; t++) cv[t] = __shfl_sync(KL_FULL, acc, t);
    if (lane == 0) cov_regularize_store(c.cov + (size_t)i * 6, cv[0], cv[1], cv[2], cv[3], cv[4], cv[5], method);
    __syncwarp();  // every lane has read the list before the next item refills it
  }
}

// ---------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------
int launch_knn_large(const CloudDev& c, const float* d_q, int nq, int qstride, int k, unsigned long long* slab, int* idx, float* d2,
                     cudaStream_t s) {
  const int grid = (nq + KL_WARPS - 1) / KL_WARPS;
  if (k <= KL_SMEM_K) k_knn_large<true><<<grid, KL_THREADS, 0, s>>>(c, d_q, nq, qstride, k, slab, idx, d2);
  else k_knn_large<false><<<grid, KL_THREADS, 0, s>>>(c, d_q, nq, qstride, k, slab, idx, d2);
  return 1;
}

// k_covariance_large's grid: one warp per item, capped for slab lists so that the slab stays within KL_COV_SLAB_BYTES
// (but holds at least one block's lists).
static int cov_large_blocks(int count, int max_n, int k) {
  const long long items = (long long)count * max_n, lstride = std::min(k, max_n);
  long long blocks = (items + KL_WARPS - 1) / KL_WARPS;
  if (lstride > KL_SMEM_K) blocks = std::min(blocks, std::max(1LL, (long long)(KL_COV_SLAB_BYTES / (KL_WARPS * lstride * 8))));
  return (int)std::min(blocks, (long long)INT_MAX);
}

size_t covariance_large_slab_bytes(int count, int max_n, int k) {
  const int lstride = std::min(k, max_n);
  if (lstride <= KL_SMEM_K) return 0;
  return (size_t)cov_large_blocks(count, max_n, k) * KL_WARPS * lstride * 8;
}

int launch_covariance_large(const CloudDev* d_clouds, int count, int max_n, int k, int method, unsigned long long* slab,
                            cudaStream_t s) {
  const int lstride = std::min(k, max_n), grid = cov_large_blocks(count, max_n, k);
  const long long items = (long long)count * max_n;
  if (lstride <= KL_SMEM_K) k_covariance_large<true><<<grid, KL_THREADS, 0, s>>>(d_clouds, max_n, items, k, method, slab, lstride);
  else k_covariance_large<false><<<grid, KL_THREADS, 0, s>>>(d_clouds, max_n, items, k, method, slab, lstride);
  return 1;
}

}  // namespace b200
