// knn.cuh -- exact k-NN traversal of the implicit AABB tree (device functions).
//
// Replaces KdTreeFLANN::nearestKSearch -> findNeighbors -> searchLevel + KNNResultSet
// (third_party/nano_gicp/include/nano_gicp/nanoflann.hpp:140-152;
//  .../impl/nanoflann_impl.hpp:1229-1250, 1354-1418, 151-214).
//
// Exactness contract (SURVEY.md App. A.3):
//   * point distance is the reference's fp32 expression ((dx*dx) + dy*dy) + dz*dz with
//     diff = query - point and NO fma contraction (nanoflann_impl.hpp:441-449), spelled with
//     __fsub_rn/__fmul_rn/__fadd_rn so nvcc cannot fuse it;
//   * the box lower bound uses the SAME operation sequence on the clamped per-axis gap, so by
//     monotonicity of IEEE rounding it never exceeds the fp32 distance of any point inside
//     the box; subtrees are skipped only when bound > current worst (strict), so candidates at
//     exactly the worst distance are still examined;
//   * ties on d2 resolve to the lower ORIGINAL index (the deterministic rule of App. A.3).
#pragma once
#include "internal.cuh"

namespace b200 {

__device__ __forceinline__ float dist2_rn(float qx, float qy, float qz, float px, float py, float pz) {
  float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ float box_dist2_rn(float qx, float qy, float qz, float4 lo, float4 hi) {
  float dx = fmaxf(fmaxf(__fsub_rn(lo.x, qx), __fsub_rn(qx, hi.x)), 0.f);
  float dy = fmaxf(fmaxf(__fsub_rn(lo.y, qy), __fsub_rn(qy, hi.y)), 0.f);
  float dz = fmaxf(fmaxf(__fsub_rn(lo.z, qz), __fsub_rn(qz, hi.z)), 0.f);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ int orig_index(const float4* __restrict__ pts, int pos) {
  return pos < 0 ? 0x7FFFFFFF : __float_as_int(__ldg(&pts[pos].w));
}

// Result set of K entries kept ascending in registers (fully unrolled; no dynamic indexing).
template <int K>
struct KnnSet {
  float d[K];
  int p[K];  // sorted POSITION in the cloud (original index is pts[p].w)
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int j = 0; j < K; j++) {
      d[j] = 3.402823466e+38f;
      p[j] = -1;
    }
  }
  __device__ __forceinline__ float worst() const { return d[K - 1]; }
  // Insert a candidate with cd <= worst().  Hot path: strict '<' chain of branch-free selects; the candidate lands
  // AFTER entries of equal distance.  Exact ties (measure ~0 on real data) are repaired by one unrolled upward bubble
  // pass in a cold branch -- written without taking the address of the arrays, so that the result set provably stays
  // in registers (an out-of-line repair taking pointers forced it into local memory: LDL/STL
  // in the hot loop).  A candidate that ties with the current worst replaces it only if its original
  // index is lower (the (d2, index) rule of SURVEY.md App. A.3).
  __device__ __forceinline__ void offer(float cd, int cp, const float4* __restrict__ pts) {
    bool tie = false;
    if (cd == d[K - 1]) {  // ties with the worst entry: decide by original index
      if (!(orig_index(pts, cp) < orig_index(pts, p[K - 1]))) return;
      d[K - 1] = cd;
      p[K - 1] = cp;
      tie = true;
    } else {
      bool placed = false;  // once the candidate is in, everything below simply shifts down by one (a carried entry must
                            // never leapfrog its equal-distance peers: it is the lowest index of its run)
#pragma unroll
      for (int j = 0; j < K; j++) {
        const bool lt = placed || cd < d[j];
        tie |= (!placed && cd == d[j]);
        placed = lt;
        const float td = d[j];
        const int tp = p[j];
        d[j] = lt ? cd : td;
        p[j] = lt ? cp : tp;
        cd = lt ? td : cd;
        cp = lt ? tp : cp;
      }
    }
    if (tie) {  // cold: the new entry sits below its equal-distance peers; bubble it up by original index
#pragma unroll
      for (int j = K - 1; j > 0; j--) {
        if (d[j] == d[j - 1] && p[j] >= 0 && orig_index(pts, p[j]) < orig_index(pts, p[j - 1])) {
          const int t = p[j];
          p[j] = p[j - 1];
          p[j - 1] = t;
        }
      }
    }
  }
  // distance of leaf slot j out of the register-resident dl[]: a select chain (no dynamic register indexing)
  __device__ __forceinline__ float leaf_distance(const float (&dl)[LEAF], int j, const float4* __restrict__, int, float, float, float) const {
    float dj = dl[0];
#pragma unroll
    for (int t = 1; t < LEAF; t++) dj = (j == t) ? dl[t] : dj;
    return dj;
  }
};

// The K best candidates as a binary MAX-heap in shared memory, one column per thread ([slot][thread]: the bank is the
// thread, so the divergent, dynamically indexed accesses of a sift-down are conflict free).  For consumers that need the
// SET of neighbours and the current worst distance, not their order (the covariance pass); the result set no longer
// occupies 2K registers.
// The heap is ordered by DISTANCE ONLY: the hot sift-down is strict float compares and nothing else (the first version
// carried the (d2, original index) rule through every compare and cost as much as the register insertion chain it
// replaced).  The tie rule matters in exactly one place --
// a candidate at EXACTLY the current worst distance -- and is resolved there, cold: among the entries tied at that
// distance the one with the highest original index is the true worst; the candidate overwrites it in place (same
// distance: the heap stays a heap) iff its own index is lower.
template <int K, int stride, bool EXACT = false>
struct KnnHeap {
  float* hd;   // column base: slot j at hd[j * stride] (stride = threads per block, a compile-time constant)
  int* hp;
  float wd;    // cached root distance
  float ev;    // distance of the entry evicted last (-1: none); see offer
  // a leaf candidate's distance is recomputed from the (L1-resident) point instead of being selected out of eight registers
  __device__ __forceinline__ float leaf_distance(const float (&)[LEAF], int, const float4* __restrict__ pts, int pos, float qx, float qy,
                                                 float qz) const {
    const float4 q = __ldg(&pts[pos]);
    return dist2_rn(qx, qy, qz, q.x, q.y, q.z);
  }
  __device__ __forceinline__ float worst() const { return wd; }
  __device__ __forceinline__ float d(int j) const { return hd[j * stride]; }
  __device__ __forceinline__ int p(int j) const { return hp[j * stride]; }
  __device__ __forceinline__ void set(int j, float dd, int pp) {
    hd[j * stride] = dd;
    hp[j * stride] = pp;
  }
  // sink (cd, cp) from slot i to its place among the first m slots; distance order only
  __device__ __forceinline__ void sift(int i, float cd, int cp, int m) {
#pragma unroll 1
    for (;;) {
      const int l = 2 * i + 1;
      if (l >= m) break;
      float dc = d(l);
      int ch = l;
      if (l + 1 < m) {
        const float dr = d(l + 1);
        if (dr > dc) {
          dc = dr;
          ch = l + 1;
        }
      }
      if (!(dc > cd)) break;
      set(i, dc, p(ch));
      i = ch;
    }
    set(i, cd, cp);
  }
  // slots 0..K-1 hold arbitrary entries: make them a heap (Floyd)
  __device__ __forceinline__ void heapify() {
#pragma unroll 1
    for (int i = K / 2 - 1; i >= 0; i--) sift(i, d(i), p(i), K);
    wd = d(0);
    ev = -1.f;
  }
  // sift from the root of a PERFECT tree (K = 2^m - 1: every internal slot has two children), levels unrolled: no bounds
  // checks, the first level's slots are immediates
  template <int LEVELS>
  __device__ __forceinline__ void sift_root_perfect(float cd, int cp) {
    int i = 0;
#pragma unroll
    for (int lv = 0; lv < LEVELS; lv++) {
      const int l = 2 * i + 1;
      const float dl = d(l), dr = d(l + 1);
      const int ch = dr > dl ? l + 1 : l;
      const float dc = fmaxf(dl, dr);
      if (!(dc > cd)) break;
      set(i, dc, p(ch));
      i = ch;
    }
    set(i, cd, cp);
  }
  // Among the first m slots, move the entry that is worst under the full (d2, original index) order to the root: of the
  // entries tied at the root's distance, the one with the highest original index (same distance: the heap stays a heap).
  __device__ __forceinline__ void root_to_true_worst(int m, const float4* __restrict__ pts) {
    const float top = d(0);
    int victim = 0, vidx = orig_index(pts, p(0));
#pragma unroll 1
    for (int j = 1; j < m; j++)
      if (d(j) == top) {
        const int oi = orig_index(pts, p(j));
        if (oi > vidx) {
          vidx = oi;
          victim = j;
        }
      }
    if (victim != 0) {
      const int t = p(0);
      hp[0] = p(victim);
      hp[victim * stride] = t;
    }
  }
  // candidate with cd <= worst()
  __device__ __forceinline__ void offer(float cd, int cp, const float4* __restrict__ pts) {
    if (cd == wd) {  // cold: the (d2, original index) rule among everything tied at the worst distance
      int worst_slot = -1, worst_idx = -1;
#pragma unroll 1
      for (int j = 0; j < K; j++)
        if (d(j) == cd) {
          const int oi = orig_index(pts, p(j));
          if (oi > worst_idx) {
            worst_idx = oi;
            worst_slot = j;
          }
        }
      if (orig_index(pts, cp) < worst_idx) hp[worst_slot * stride] = cp;
      return;
    }
    // The root is evicted.  If another entry ties with it (then a child of the root does), the one to evict is the highest
    // original index among them, not whichever entry the distance-only heap put at the root.  EXACT does that at every
    // eviction; the hot instantiation only records the distance evicted last (evictions only ever lower it), and the
    // caller redoes the search with EXACT when that equals the final worst distance -- the only case in which an entry of
    // the final tie group can have been dropped (exact ties at the cut: lattices, duplicates).
    if (EXACT) {
      if (d(1) == wd || d(2) == wd) root_to_true_worst(K, pts);
    } else {
      ev = wd;
    }
    if (K == 15) sift_root_perfect<3>(cd, cp);
    else if (K == 31) sift_root_perfect<4>(cd, cp);
    else sift(0, cd, cp, K);
    wd = d(0);
  }
  // Remove the worst entry under the full (d2, original index) order from a heap holding m entries; returns m - 1.
  // Only used when fewer neighbours than the capacity are wanted (k < K): cold.
  __device__ __forceinline__ int pop(int m, const float4* __restrict__ pts) {
    root_to_true_worst(m, pts);  // the root's entry is dropped
    const float ld = d(m - 1);
    const int lp = p(m - 1);
    sift(0, ld, lp, m - 1);
    return m - 1;
  }
};

// One descent step of the best-first k-NN walks (knn_walk here, kl_walk in knn_large.cu): order record n's two children
// by their box bound (child 1 first only if strictly nearer), hand the far child to push(ref, bound) unless its bound is
// strictly greater than the current worst distance w, and move to the near child.  Returns false when the near child is
// pruned as well.
template <typename Push>
__device__ __forceinline__ bool near_far_step(const NodeRec& n, float qx, float qy, float qz, float w, int& ref, float& dnode, Push&& push) {
  const float d0 = box_dist2_rn(qx, qy, qz, n.lo0, n.hi0);
  const float d1 = box_dist2_rn(qx, qy, qz, n.lo1, n.hi1);
  int nref = n.ref0(), fref = n.ref1();
  float nd = d0, fd = d1;
  if (d1 < d0) {
    nref = n.ref1(); fref = n.ref0(); nd = d1; fd = d0;
  }
  if (!(fd > w)) push(fref, fd);
  ref = nref;
  dnode = nd;
  return !(nd > w);
}

// Exact K-NN of (qx,qy,qz) in cloud c.  One thread per query; Morton-sorted queries keep
// neighbouring lanes on neighbouring paths (coherent loads, low divergence).
// The traversal stack holds (ref, bound) entries.  The first S live (8 B each) in a shared-memory column of the calling
// thread, sh = &column[0][threadIdx.x] of a __shared__ int2[S][stride] ([slot][thread]: the bank is the thread, as in
// KnnHeap, so the divergent pushes and pops of a warp are conflict free); entries S.. go to local-memory arrays that a walk
// only touches when it goes deeper than S (profiles/emulate_stack_depth.py: how deep the walks of each kernel go).
// S = 0 (sh unused): the whole stack in local memory, where every push and pop is an STL/LDL through L1.
template <int S = 0, int stride = 1, typename Res>
__device__ __forceinline__ void knn_walk(const CloudDev& c, float qx, float qy, float qz, Res& res, int2* sh = nullptr, int skip_lo = 1,
                                         int skip_hi = 0) {
  const float4* __restrict__ pts = c.pts;
  const float4* __restrict__ tn = c.tnodes;  // read once: c may be a reference into global memory (clouds[blockIdx.y])
  int stack_ref[MAX_STACK - S];
  float stack_d[MAX_STACK - S];
  int sp = 0;
  int ref = c.root_ref;
  float dnode = 0.f;
  for (;;) {
    bool alive = !(dnode > res.worst());
    while (alive && ref >= 0)  // internal node: both children's boxes live in one 64-B record
      alive = near_far_step(load_node(tn, ref), qx, qy, qz, res.worst(), ref, dnode, [&](int r, float d) {
        if (sp < S) {
          sh[sp * stride] = make_int2(r, __float_as_int(d));
        } else {
          stack_ref[sp - S] = r;
          stack_d[sp - S] = d;
        }
        sp++;
      });
    if (alive) {  // leaf: up to LEAF consecutive points
      const LeafSpan leaf = leaf_span(ref);
      const int base = leaf.base, cnt = leaf.count;
      float dl[LEAF];
      unsigned mask = 0;
      const float w0 = res.worst();
#pragma unroll
      for (int j = 0; j < LEAF; j++) {
        const float4 p = __ldg(&pts[base + (j < cnt ? j : 0)]);
        dl[j] = dist2_rn(qx, qy, qz, p.x, p.y, p.z);
        // d <= w, not !(d > w): a point with a NaN coordinate (NaN d2) is never a candidate (KnnHeap::offer would evict
        // its root for one)
        if (j < cnt && dl[j] <= w0 && !(base + j >= skip_lo && base + j <= skip_hi)) mask |= 1u << j;
      }
      // ONE insertion site per leaf: candidates are fed in slot order through a select chain
      while (mask) {
        const int j = __ffs(mask) - 1;
        mask &= mask - 1;
        const float dj = res.leaf_distance(dl, j, pts, base + j, qx, qy, qz);
        if (dj <= res.worst()) res.offer(dj, base + j, pts);
      }
    }
    bool found = false;
    while (sp > 0) {
      sp--;
      const float d = sp < S ? __int_as_float(sh[sp * stride].y) : stack_d[sp - S];
      if (!(d > res.worst())) {
        ref = sp < S ? sh[sp * stride].x : stack_ref[sp - S];
        dnode = d;
        found = true;
        break;
      }
    }
    if (!found) break;
  }
}

// Fixed-radius search with a WARP-SHARED traversal and deferred, lockstep processing of the hits.
// Why per warp (profiles/README.md): with the callback inside a per-thread traversal the SPFH kernel ran with 4.75 of 32
// lanes active; collecting hits per thread and processing them warp-convergently brought that to 12.7, but the SASS
// profile still had half of all instructions in the private traversals at 4-7 active lanes (lanes fill their buffers at
// different rates and wait; a bigger buffer cost more occupancy than it won).  The 32 queries of a warp are
// Morton-neighbours, so their balls overlap almost completely; the warp therefore walks the tree once.
//
// radius_descend_warp is that one walk: a node is entered if ANY active lane's own exact box test passes (box bound
// < r2; a subtree whose bound is >= r2 holds no point with d2 < r2, so no lane misses anything), the stack is
// warp-uniform, and leaf(base, count) runs warp-uniformly for every leaf reached.  Control flow is warp-uniform
// throughout; the order of the leaves is deterministic for a given cloud.
// Must be called by every thread of the warp.  wstack: MAX_STACK ints private to the warp.
template <typename L>
__device__ __forceinline__ void radius_descend_warp(const CloudDev& c, bool active, float qx, float qy, float qz, float r2, int* wstack,
                                                    L&& leaf) {
  const float4* __restrict__ tn = c.tnodes;  // read once, as in knn_walk
  constexpr unsigned FULL = 0xffffffffu;
  int sp = 0;
  int ref = c.root_ref;
  for (;;) {
    while (ref >= 0) {
      const NodeRec n = load_node(tn, ref);
      const bool in0 = __any_sync(FULL, active && box_dist2_rn(qx, qy, qz, n.lo0, n.hi0) < r2);
      const bool in1 = __any_sync(FULL, active && box_dist2_rn(qx, qy, qz, n.lo1, n.hi1) < r2);
      if (in0 && in1) {
        wstack[sp++] = n.ref1();  // every lane writes the same value
        ref = n.ref0();
      } else if (in0) {
        ref = n.ref0();
      } else if (in1) {
        ref = n.ref1();
      } else {
        ref = 0x7FFFFFFF;  // dead end
        break;
      }
    }
    if (ref < 0) {
      const LeafSpan s = leaf_span(ref);
      leaf(s.base, s.count);
    }
    if (sp == 0) break;
    __syncwarp();  // the pushes of this round are visible to every lane ...
    ref = wstack[--sp];
    __syncwarp();  // ... and every lane has popped before the slot can be pushed again
  }
}

// The shared walk with PER-LANE hit lists: every lane tests every point of a visited leaf against its own query and
// collects its own hits, and whenever some lane's buffer could overflow the whole warp processes what it has collected,
// in lockstep: f(position, d2) on the owner lane, in the order of the warp's walk.  Each lane receives exactly its own
// neighbour set in a fixed order (k_fpfh's fp32 sums depend on it).
// Must be called by every thread of the warp.  spos (and sd2 unless nullptr): [BUF][blockDim.x]; wstack: MAX_STACK
// ints private to the warp.
template <int BUF, typename F>
__device__ __forceinline__ void radius_visit_warp(const CloudDev& c, bool active, float qx, float qy, float qz, float r2, int* spos,
                                                  float* sd2, int* wstack, F&& f) {
  const float4* __restrict__ pts = c.pts;
  const int tid = threadIdx.x, stride = blockDim.x;
  constexpr unsigned FULL = 0xffffffffu;
  int cnt = 0;
  auto flush = [&]() {
    const int most = __reduce_max_sync(FULL, cnt);
    for (int e = 0; e < most; e++)
      if (e < cnt) f(spos[e * stride + tid], sd2 ? sd2[e * stride + tid] : 0.f);
    cnt = 0;
  };
  if (!__any_sync(FULL, active)) return;
  radius_descend_warp(c, active, qx, qy, qz, r2, wstack, [&](int base, int n) {
    for (int j = 0; j < n; j++) {
      const float4 p = __ldg(&pts[base + j]);
      const float d2 = dist2_rn(qx, qy, qz, p.x, p.y, p.z);
      if (active && d2 < r2) {
        spos[cnt * stride + tid] = base + j;
        if (sd2) sd2[cnt * stride + tid] = d2;
        cnt++;
      }
    }
    if (__any_sync(FULL, cnt > BUF - LEAF)) flush();
  });
  flush();
}

// The shared walk with the hits of all 32 queries POOLED in one per-warp ring and processed 32 at a time by
// whichever lane is free: f(owner_lane, position) runs for entry e on lane e.  For per-pair work whose result is
// order-independent (integer histograms in shared memory) this keeps every lane busy -- with per-lane hit lists the
// lockstep processing leaves lanes idle (the lanes of a warp fill their lists at different rates).
// on_hit(position) runs on the OWNER lane when the hit is found (cheap bookkeeping such as a neighbour count).
// ring: RV_RING unsigned per warp.  Must be called by every thread of the warp; control flow is warp-uniform.
constexpr int RV_RING = 64;
template <typename H, typename F>
__device__ __forceinline__ void radius_visit_warp_pooled(const CloudDev& c, bool active, float qx, float qy, float qz, float r2,
                                                         unsigned* ring, int* wstack, H&& on_hit, F&& f) {
  const float4* __restrict__ pts = c.pts;
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  int head = 0, tail = 0;  // warp-uniform: entries [head, tail) of the ring are pending
  auto process = [&](int take) {
    if (lane < take) {
      const unsigned e = ring[(head + lane) & (RV_RING - 1)];
      f((int)(e & 31u), (int)(e >> 5));
    }
    head += take;
    __syncwarp();
  };
  if (!__any_sync(FULL, active)) return;
  radius_descend_warp(c, active, qx, qy, qz, r2, wstack, [&](int base, int n) {
    for (int j = 0; j < n; j++) {
      const float4 p = __ldg(&pts[base + j]);
      const bool hit = active && dist2_rn(qx, qy, qz, p.x, p.y, p.z) < r2;
      const unsigned m = __ballot_sync(FULL, hit);
      if (hit) {
        ring[(tail + __popc(m & lt)) & (RV_RING - 1)] = ((unsigned)(base + j) << 5) | (unsigned)lane;
        on_hit(base + j);
      }
      tail += __popc(m);
      if (tail - head >= 32) {  // at most 31 + 32 pending: the ring never overflows
        __syncwarp();
        process(32);
      }
    }
  });
  __syncwarp();
  if (tail > head) process(tail - head);
}

}  // namespace b200
