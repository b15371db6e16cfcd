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
#include "knn.cuh"
#include "launchers.cuh"

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
__global__ void __launch_bounds__(KL_THREADS) k_knn_large(CloudDev c, const float* q, int nq, int qstride, int k,
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
// host launcher
// ---------------------------------------------------------------------------------------
int launch_knn_large(const CloudDev& c, const float* d_q, int nq, int qstride, int k, unsigned long long* slab, int* idx, float* d2,
                     cudaStream_t s) {
  const int grid = (nq + KL_WARPS - 1) / KL_WARPS;
  if (k <= KL_SMEM_K) k_knn_large<true><<<grid, KL_THREADS, 0, s>>>(c, d_q, nq, qstride, k, slab, idx, d2);
  else k_knn_large<false><<<grid, KL_THREADS, 0, s>>>(c, d_q, nq, qstride, k, slab, idx, d2);
  return 1;
}

}  // namespace b200
