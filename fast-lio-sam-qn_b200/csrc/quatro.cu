// quatro.cu -- the Quatro half of the loop-closure path as batched GPU kernels (blockIdx.y = cloud / pair).
// Compiled with -fmad=false: the fp32 feature arithmetic follows a fixed operation order (see the oracle).
//
// Reference behaviour being replaced (paths relative to the reference tree's root; PCL / FLANN / TEASER++ semantics per
// SURVEY.md App. B because those libraries are not vendored):
//   Q1 k_normals        pcl::NormalEstimation, radius 0.9, viewpoint (0,0,0)       third_party/Quatro/src/fpfh.cc:27-32
//   Q2 k_spfh           FPFHEstimationOMP::computePointSPFHSignature                fpfh.cc:35-39
//   Q3 k_fpfh           FPFHEstimationOMP::weightPointSPFHSignature                 fpfh.cc:35-39
//      k_fcode / k_fgather               the matcher's view: descriptors in filter-space Morton order, identical records collapsed, boxed per 64-record tile
//   Q4 k_feat_nn        FLANN KDTreeSingleIndex exact 1-NN in 33-D (both directions) third_party/Quatro/src/matcher.cc:378-399, 597-636
//      k_first_hit / k_mutual            gate + first-hit reverse search + mutual check   matcher.cc:412-455
//      k_cloud_sum / k_cloud_scale       Matcher::normalizePoints                         matcher.cc:58-116
//      k_tuple_trials / k_tuple_select   tuple test (<= 100 ncorr trials, stop at > max)  matcher.cc:461-538
//      k_adv_select                      Matcher::advancedMatching tail (sort + unique)   matcher.cc:118-356
//   Q5 k_teaser_solve   RobustRegistrationSolver::solve, QUATRO + PMC_HEU           call site third_party/Quatro/src/quatro_module.cc:69-76
//      k_big_*                           the same solve over a global-memory workspace for > 512 correspondences
// Deliberate definitions where the reference is seed- or race-dependent are listed in oracle/oracle_quatro.cpp.
#include "internal.cuh"
#include "fpfh_basis.cuh"
#include "knn.cuh"
#include "launchers.cuh"
#include "smallmath.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------------
// Q1 normals
// ------------------------------------------------------------------------------------------------
constexpr int RV_BUF = 16;     // per-lane hit buffer of the warp-shared walk (radius_visit_warp), positions only
constexpr int RV_BUF_D2 = 16;  // ... when the distance travels with the position (k_fpfh)

__global__ void __launch_bounds__(STEP_THREADS) k_normals(const CloudDev* clouds, float r2) {
  const CloudDev& c = clouds[blockIdx.y];
  const int i = blockIdx.x * STEP_THREADS + threadIdx.x;
  __shared__ int spos[RV_BUF * STEP_THREADS];
  __shared__ int wstack[STEP_THREADS / 32][MAX_STACK];
  const bool inrange = i < c.n;
  const float4 p = inrange ? c.pts[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  double m0 = 0, m1 = 0, m2 = 0, c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, c5 = 0;
  int cnt = 0;
  // the fp64 moments are the heavy part: accumulate them warp-convergently (same neighbour order as the traversal)
  radius_visit_warp<RV_BUF>(c, inrange, p.x, p.y, p.z, r2, spos, nullptr, wstack[threadIdx.x >> 5], [&](int pos, float) {
    const float4 q = __ldg(&c.pts[pos]);
    const double x = (double)q.x - (double)p.x, y = (double)q.y - (double)p.y, z = (double)q.z - (double)p.z;
    m0 += x; m1 += y; m2 += z;
    c0 += x * x; c1 += x * y; c2 += x * z; c3 += y * y; c4 += y * z; c5 += z * z;
    cnt++;
  });
  if (!inrange) return;
  if (cnt < 3) {
    c.nrm[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const double inv = 1.0 / (double)cnt;
  m0 *= inv; m1 *= inv; m2 *= inv;
  double n[3];
  sym3_smallest_evec(c0 * inv - m0 * m0, c1 * inv - m0 * m1, c2 * inv - m0 * m2, c3 * inv - m1 * m1, c4 * inv - m1 * m2,
                     c5 * inv - m2 * m2, n);
  float nx = (float)n[0], ny = (float)n[1], nz = (float)n[2];
  const float cos_theta = ((0.f - p.x) * nx + (0.f - p.y) * ny) + (0.f - p.z) * nz;  // flipNormalTowardsViewpoint, vp = 0
  if (cos_theta < 0.f) {
    nx = -nx; ny = -ny; nz = -nz;
  }
  c.nrm[i] = make_float4(nx, ny, nz, 1.f);
}

// pcl::computePairFeatures in fp32 with the oracle's operation order
__device__ __forceinline__ bool pair_features(const float4& p1, const float4& n1, const float4& p2, const float4& n2, float& f1,
                                              float& f2, float& f3) {
  float d0 = p2.x - p1.x, d1 = p2.y - p1.y, d2 = p2.z - p1.z;
  const float f4 = sqrtf((d0 * d0 + d1 * d1) + d2 * d2);
  if (f4 == 0.f) return false;
  float a0 = n1.x, a1 = n1.y, a2 = n1.z, b0 = n2.x, b1 = n2.y, b2 = n2.z;
  const float angle1 = ((a0 * d0 + a1 * d1) + a2 * d2) / f4;
  const float angle2 = ((b0 * d0 + b1 * d1) + b2 * d2) / f4;
  if (fabsf(angle1) < fabsf(angle2)) {
    float t;
    t = a0; a0 = b0; b0 = t;
    t = a1; a1 = b1; b1 = t;
    t = a2; a2 = b2; b2 = t;
    d0 = -d0; d1 = -d1; d2 = -d2;
    f3 = -angle2;
  } else {
    f3 = angle1;
  }
  float v0 = d1 * a2 - d2 * a1, v1 = d2 * a0 - d0 * a2, v2 = d0 * a1 - d1 * a0;
  const float vn = sqrtf((v0 * v0 + v1 * v1) + v2 * v2);
  if (vn == 0.f) return false;
  v0 /= vn; v1 /= vn; v2 /= vn;
  const float w0 = a1 * v2 - a2 * v1, w1 = a2 * v0 - a0 * v2, w2 = a0 * v1 - a1 * v0;
  f2 = (v0 * b0 + v1 * b1) + v2 * b2;
  f1 = atan2f((w0 * b0 + w1 * b1) + w2 * b2, (a0 * b0 + a1 * b1) + a2 * b2);
  return true;
}

__device__ __forceinline__ int bin11(float v) {
  const int h = (int)floorf(v);
  return h < 0 ? 0 : (h > 10 ? 10 : h);
}

// ------------------------------------------------------------------------------------------------
// Q2 SPFH: per-point 33-bin integer histogram in shared memory (bin-major: the column is the point's thread).  The
// (point, neighbour) pairs of a warp are pooled and processed 32 at a time by whichever lane is free
// (radius_visit_warp_pooled); the increments are integer shared-memory atomics, so the order does not matter.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(STEP_THREADS) k_spfh(const CloudDev* clouds, float r2) {
  const CloudDev& c = clouds[blockIdx.y];
  const int i = blockIdx.x * STEP_THREADS + threadIdx.x;
  __shared__ unsigned int hist[FDIM][STEP_THREADS];  // 32-bit: an un-voxelised cloud can hold > 65535 neighbours in the radius
  __shared__ float4 s_p[STEP_THREADS], s_n[STEP_THREADS];
  __shared__ unsigned ring[STEP_THREADS / 32][RV_RING];
  __shared__ int wstack[STEP_THREADS / 32][MAX_STACK];
#pragma unroll
  for (int k = 0; k < FDIM; k++) hist[k][threadIdx.x] = 0;
  const bool inrange = i < c.n;
  const float4 p = inrange ? c.pts[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 np = inrange ? c.nrm[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  s_p[threadIdx.x] = p;
  s_n[threadIdx.x] = np;
  __syncwarp();
  int cnt = 0;
  const float d_pi = 1.0f / (2.0f * 3.14159265358979323846f);
  const int wbase = threadIdx.x & ~31, ibase = blockIdx.x * STEP_THREADS + wbase;
  radius_visit_warp_pooled(
      c, inrange && np.w != 0.f, p.x, p.y, p.z, r2, ring[threadIdx.x >> 5], wstack[threadIdx.x >> 5], [&](int) { cnt++; },
      [&](int owner, int pos) {
        if (pos == ibase + owner) return;
        const float4 nq = __ldg(&c.nrm[pos]);
        if (nq.w == 0.f) return;
        const float4 q = __ldg(&c.pts[pos]);
        float f1, f2, f3;
        if (!pair_features(s_p[wbase + owner], s_n[wbase + owner], q, nq, f1, f2, f3)) return;
        const int col = wbase + owner;
        atomicAdd(&hist[bin11(11.0f * ((f1 + 3.14159265358979323846f) * d_pi))][col], 1u);
        atomicAdd(&hist[11 + bin11(11.0f * ((f2 + 1.0f) * 0.5f))][col], 1u);
        atomicAdd(&hist[22 + bin11(11.0f * ((f3 + 1.0f) * 0.5f))][col], 1u);
      });
  __syncwarp();
  if (!inrange) return;
  float* out = c.spfh + (size_t)i * FPAD;
  const float incr = cnt >= 2 ? 100.0f / (float)(cnt - 1) : 0.f;
#pragma unroll
  for (int k = 0; k < FDIM; k++) out[k] = (float)hist[k][threadIdx.x] * incr;
  out[33] = 0.f; out[34] = 0.f; out[35] = 0.f;
}

// ------------------------------------------------------------------------------------------------
// Q3 FPFH: sum SPFH(q)/d2 over the neighbours, each 11-bin block rescaled to 100
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(STEP_THREADS) k_fpfh(const CloudDev* clouds, float r2) {
  const CloudDev& c = clouds[blockIdx.y];
  const int i = blockIdx.x * STEP_THREADS + threadIdx.x;
  __shared__ int spos[RV_BUF_D2 * STEP_THREADS];
  __shared__ float sd2[RV_BUF_D2 * STEP_THREADS];
  __shared__ int wstack[STEP_THREADS / 32][MAX_STACK];
  const bool inrange = i < c.n;
  const float4 p = inrange ? c.pts[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  float h[FDIM];
#pragma unroll
  for (int k = 0; k < FDIM; k++) h[k] = 0.f;
  radius_visit_warp<RV_BUF_D2>(c, inrange && c.nrm[inrange ? i : 0].w != 0.f, p.x, p.y, p.z, r2, spos, sd2, wstack[threadIdx.x >> 5], [&](int pos, float d2) {
    if (d2 == 0.f) return;
    const float w = 1.0f / d2;
    const float4* s4 = reinterpret_cast<const float4*>(c.spfh + (size_t)pos * FPAD);
    float s[FPAD];
#pragma unroll
    for (int k = 0; k < 9; k++) {
      const float4 v = __ldg(&s4[k]);
      s[4 * k] = v.x; s[4 * k + 1] = v.y; s[4 * k + 2] = v.z; s[4 * k + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < FDIM; k++) h[k] = __fmaf_rn(s[k], w, h[k]);  // one rounding per term instead of two
  });
  if (!inrange) return;
  // block sums taken once at the end (the reference adds them up pair by pair; neither order is privileged, and the
  // neighbour order already differs from the kd-tree's)
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int k = 0; k < 11; k++) {
    s0 += h[k];
    s1 += h[11 + k];
    s2 += h[22 + k];
  }
  const float sc0 = s0 != 0.f ? 100.0f / s0 : 0.f, sc1 = s1 != 0.f ? 100.0f / s1 : 0.f, sc2 = s2 != 0.f ? 100.0f / s2 : 0.f;
  float* out = c.fpfh + (size_t)i * FPAD;
  bool any = false;
#pragma unroll
  for (int k = 0; k < FDIM; k++) {
    const float v = h[k] * (k < 11 ? sc0 : (k < 22 ? sc1 : sc2));
    out[k] = v;
    any |= (v != 0.f);
  }
  out[33] = p.w;  // original index (int bits)
  out[34] = any ? 1.f : 0.f;
  // the matcher's filter coordinates (fpfh_basis.cuh): projections on three fixed orthonormal directions and the norm of
  // the residual, computed from the residual VECTOR (no cancellation of large sums); plus a hash of the record's bits
  float x[FDIM];
  float c0 = 0.f, c1 = 0.f, c2 = 0.f;
  uint32_t hsh = 0x811C9DC5u;
#pragma unroll
  for (int k = 0; k < FDIM; k++) {
    const float v = h[k] * (k < 11 ? sc0 : (k < 22 ? sc1 : sc2));
    hsh = (hsh ^ __float_as_uint(v)) * 0x01000193u;
    hsh ^= hsh >> 15;
    x[k] = v - FB_MU[k];
    c0 += x[k] * FB_U[0][k];
    c1 += x[k] * FB_U[1][k];
    c2 += x[k] * FB_U[2][k];
  }
  float rr = 0.f;
#pragma unroll
  for (int k = 0; k < FDIM; k++) {
    const float e = x[k] - ((c0 * FB_U[0][k] + c1 * FB_U[1][k]) + c2 * FB_U[2][k]);
    rr += e * e;
  }
  out[35] = __uint_as_float(hsh);
  c.fproj[i] = make_float4(c0, c1, c2, sqrtf(rr));
}

// ------------------------------------------------------------------------------------------------
// Q4 exact 33-D nearest neighbour, brute force with TMA-bulk staged base tiles
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok = 0;
  while (!ok) {
    asm volatile(
        "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}

constexpr int NN_THREADS = 128;  // 4 warps, each owning 32 queries (measured: 64 and 32 threads per block are slower)
constexpr int NN_TILE = 64;      // base descriptors per smem tile: 64 * 144 B = 9216 B per cp.async.bulk
constexpr int NN_QCAP = 96;      // per-warp survivor queue (drained whenever it holds >= 32 entries)

// ---- filter-space ordering of the descriptors (the matcher's view) ------------------------------------------------
// fixed quantiser of the filter coordinates (half-ranges from the spread of real descriptors; outliers clamp -- the code
// only orders the records, exactness never depends on it)
__device__ __forceinline__ uint32_t fcode_of(const float4 f) {
  const int q0 = min(127, max(0, (int)((f.x + 60.f) * (128.f / 120.f)))), q1 = min(127, max(0, (int)((f.y + 40.f) * (128.f / 80.f)))),
            q2 = min(127, max(0, (int)((f.z + 30.f) * (128.f / 60.f)))), q3 = min(127, max(0, (int)(f.w * (128.f / 60.f))));
  uint32_t c = 0;
#pragma unroll
  for (int b = 0; b < 7; b++)
    c |= (((uint32_t)q0 >> b) & 1u) << (4 * b) | (((uint32_t)q1 >> b) & 1u) << (4 * b + 1) | (((uint32_t)q2 >> b) & 1u) << (4 * b + 2) |
         (((uint32_t)q3 >> b) & 1u) << (4 * b + 3);
  return c;
}
// sort key of sorted position p: 28-bit Morton code of the four filter coordinates, then 4 hash bits so that bitwise
// identical descriptors (planar patches all produce the same histogram) end up next to each other; unusable
// descriptors go to the end
__global__ void __launch_bounds__(256) k_fcode(const CloudDev* clouds) {
  const CloudDev& c = clouds[blockIdx.y];
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.n) return;
  const float4 tail = *reinterpret_cast<const float4*>(c.fpfh + (size_t)p * FPAD + 32);  // slots 32..35
  const bool ok = tail.z != 0.f;
  c.keys[0][p] = ok ? ((fcode_of(c.fproj[p]) << 4) | (__float_as_uint(tail.w) & 15u)) : 0xFFFFFFFFu;
  c.vals[0][p] = (uint32_t)p;
}
// gather the records into code order, collapse runs of bitwise identical descriptors and box every tile of NN_TILE
// records in filter space.  One 64-thread block per tile.
//   A run (consecutive identical records inside one tile) keeps its first record as a BASE record, carrying the run's
//   lowest original index in slot 35 -- exactly what the lowest-index tie rule would pick among them; the others get
//   flag 2: still queries, never candidates.  Runs that a tile border or a hash collision splits simply keep two heads.
__global__ void __launch_bounds__(NN_TILE) k_fgather(const CloudDev* clouds) {
  const CloudDev& c = clouds[blockIdx.y];
  const int t = blockIdx.x;
  if (t * NN_TILE >= c.n) return;
  const int r = t * NN_TILE + threadIdx.x;
  __shared__ int s_p[NN_TILE];
  __shared__ int s_same[NN_TILE];
  __shared__ int s_min[NN_TILE];
  float lo[4] = {INFINITY, INFINITY, INFINITY, INFINITY}, hi[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  float4 rec[9];
#pragma unroll
  for (int k = 0; k < 9; k++) rec[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 fp = make_float4(0.f, 0.f, 0.f, 0.f);
  int p = -1;
  bool usable = false;
  if (r < c.n) {
    p = (int)c.vals[1][r];  // radix_sort_result_buf()
    const float4* s4 = reinterpret_cast<const float4*>(c.fpfh + (size_t)p * FPAD);
#pragma unroll
    for (int k = 0; k < 9; k++) rec[k] = s4[k];
    fp = c.fproj[p];
    usable = rec[8].z != 0.f;  // slot 34
  }
  s_p[threadIdx.x] = usable ? p : -1;
  s_min[threadIdx.x] = __float_as_int(rec[8].y);  // own original index
  __syncthreads();
  bool same = false;
  if (usable && threadIdx.x > 0 && s_p[threadIdx.x - 1] >= 0) {
    const float4* q4 = reinterpret_cast<const float4*>(c.fpfh + (size_t)s_p[threadIdx.x - 1] * FPAD);
    const float4 qt = q4[8];
    same = __float_as_uint(qt.w) == __float_as_uint(rec[8].w) && __float_as_uint(qt.x) == __float_as_uint(rec[8].x);  // hash, slot 32
    for (int k = 0; same && k < 8; k++) {
      const float4 v = q4[k];
      same = __float_as_uint(v.x) == __float_as_uint(rec[k].x) && __float_as_uint(v.y) == __float_as_uint(rec[k].y) &&
             __float_as_uint(v.z) == __float_as_uint(rec[k].z) && __float_as_uint(v.w) == __float_as_uint(rec[k].w);
    }
  }
  s_same[threadIdx.x] = same ? 1 : 0;
  __syncthreads();
  if (same) {
    int h = threadIdx.x - 1;
    while (s_same[h]) h--;  // s_same[0] == 0
    atomicMin(&s_min[h], __float_as_int(rec[8].y));
  }
  __syncthreads();
  if (r < c.n) {
    rec[8].z = !usable ? 0.f : (same ? 2.f : 1.f);
    rec[8].w = __int_as_float(s_min[threadIdx.x]);  // base index: the run's lowest original index (heads), own otherwise
    float4* d4 = reinterpret_cast<float4*>(c.fpfh_s + (size_t)r * FPAD);
#pragma unroll
    for (int k = 0; k < 9; k++) d4[k] = rec[k];
    c.fproj_s[r] = fp;
    c.fcode_s[r] = c.keys[1][r];
    if (usable && !same) {
      lo[0] = hi[0] = fp.x; lo[1] = hi[1] = fp.y; lo[2] = hi[2] = fp.z; lo[3] = hi[3] = fp.w;
    }
  }
  __shared__ float red[2][8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int d = 0; d < 4; d++) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
    float* w = red[threadIdx.x >> 5];
#pragma unroll
    for (int d = 0; d < 4; d++) {
      w[d] = lo[d];
      w[4 + d] = hi[d];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // a tile without base records keeps lo = +inf: its lower bound is +inf, nobody visits it
    c.ftile[2 * t] = make_float4(fminf(red[0][0], red[1][0]), fminf(red[0][1], red[1][1]), fminf(red[0][2], red[1][2]), fminf(red[0][3], red[1][3]));
    c.ftile[2 * t + 1] = make_float4(fmaxf(red[0][4], red[1][4]), fmaxf(red[0][5], red[1][5]), fmaxf(red[0][6], red[1][6]), fmaxf(red[0][7], red[1][7]));
  }
}

// filter test of one record: squared distance of the filter coordinates
__device__ __forceinline__ float filt_lb(const float4& q, const float4& b) {
  const float e0 = q.x - b.x, e1 = q.y - b.y, e2 = q.z - b.z, e3 = q.w - b.w;
  return __fmaf_rn(e3, e3, __fmaf_rn(e2, e2, __fmaf_rn(e1, e1, e0 * e0)));  // a filter, not a parity-relevant value: fused
}
// lower bound of the filter's record test over every record of a tile: distance from the query's coordinates to the
// tile's box.  Same operation order as the record test and rounding is monotone, so box_lb <= record lower bound.
__device__ __forceinline__ float tile_lb(const float4& q, const float4& lo, const float4& hi) {
  const float e0 = fmaxf(fmaxf(lo.x - q.x, q.x - hi.x), 0.f), e1 = fmaxf(fmaxf(lo.y - q.y, q.y - hi.y), 0.f),
              e2 = fmaxf(fmaxf(lo.z - q.z, q.z - hi.z), 0.f), e3 = fmaxf(fmaxf(lo.w - q.w, q.w - hi.w), 0.f);
  return __fmaf_rn(e3, e3, __fmaf_rn(e2, e2, __fmaf_rn(e1, e1, e0 * e0)));
}
// acceptance threshold of the filter for a query whose best squared distance so far is `best`.  The filter value is a
// true lower bound of the distance up to fp32 rounding of the coordinates (worst case 2.4e-3 in distance for |a - mu| <=
// 173, measured 7e-5: profiles/emulate_projected_bound_margin.py) and of the refine's sum (4e-6 relative).
__device__ __forceinline__ float filt_bound(float best) {
  const float sb = sqrtf(best) * 1.00001f + 4e-3f;
  return sb * sb;
}

// Exact 33-D 1-NN by filter-and-refine over filter-ordered tiles.
//  * Both clouds are held in the order of the Morton code of their four filter coordinates (k_fcode / k_fgather), so the
//    128 queries of a block are similar and a base tile of 64 records is a small box in filter space; bitwise identical
//    base records are collapsed to one candidate per run (k_fgather).
//  * A block starts at the base tile nearest to its own queries (binary search of the code) and sweeps up, then down:
//    good matches are found in the first tiles and the bound is tight from then on.
//  * Per tile: every lane tests ITS query against the tile box (one test instead of 64); tiles nobody in the block
//    needs are not even fetched (block-wide OR of per-thread need masks, taken per chunk of visits), tiles are fetched
//    by cp.async.bulk (TMA) one ahead.
//  * Per (needed query, tile): the 32 lanes test 32+32 records against the projected lower bound
//    sum_i (u_i.(a - b))^2 + (|r_a| - |r_b|)^2 <= |a - b|^2 (fpfh_basis.cuh), ballot-compact the survivors into a
//    per-warp queue, and refine 32 queued pairs at a time with the full fp32 distance in the oracle's operation order.
// Exact: both bounds are true lower bounds applied with a margin against rounding; ties go to the lower original index
// through the packed (d2 bits, index) 64-bit minimum, so the visiting order does not matter.
// mode 0: queries = fj, base = fi; writes nn/dis by ORIGINAL j
// mode 1: queries = the fi points that were hit (first_j != INT_MAX), base = fj; writes rnn by ORIGINAL i
__global__ void __launch_bounds__(NN_THREADS) k_feat_nn(const MatchDev* pairs, int mode, float thr2) {
  const MatchDev& P = pairs[blockIdx.y];
  const CloudDev& Q = mode == 0 ? P.fj : P.fi;
  const CloudDev& B = mode == 0 ? P.fi : P.fj;
  const int nq = Q.n;
  const int q0 = blockIdx.x * NN_THREADS;
  if (q0 >= nq) return;
  __shared__ __align__(128) float tile[2][NN_TILE * FPAD];
  __shared__ __align__(16) float4 tnorm[2][NN_TILE];
  __shared__ __align__(16) float4 sqn[NN_THREADS / 32][32];
  __shared__ unsigned long long sbest[NN_THREADS / 32][32];
  __shared__ int sbound[NN_THREADS / 32][32];  // filt_bound(best d2) as int bits (positive floats order like ints): atomicMin
  __shared__ unsigned short queue[NN_THREADS / 32][NN_QCAP];
  __shared__ __align__(8) unsigned long long full[2];
  __shared__ unsigned s_need[3];  // block-level need masks of the current / next chunks of tile visits
  __shared__ int s_t0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float lim = __int_as_float(__float_as_int(thr2) + 1);  // nextafter(thr2, +inf): d2 == thr2 still qualifies
  // stage this thread's query (row `lane` of its warp)
  const int qi = q0 + threadIdx.x;
  int qorig = -1;
  bool qok = false;
  float4 qn = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    const bool inrange = qi < nq;
    const float4* q4 = reinterpret_cast<const float4*>(Q.fpfh_s + (size_t)(inrange ? qi : 0) * FPAD);
    const float4 last = inrange ? q4[8] : make_float4(0.f, 0.f, 0.f, 0.f);  // slots 32..35
    qorig = __float_as_int(last.y);
    qok = inrange && last.z != 0.f;
    if (inrange) qn = Q.fproj_s[qi];
    // reverse search: i was reached from j0 = first_j[i] at distance dis[j0], and the metric is symmetric, so that
    // very pair is a valid starting candidate -- the filter is tight from the first tile on
    unsigned long long init = ((unsigned long long)__float_as_uint(lim) << 32) | 0xFFFFFFFFull;
    if (mode == 1 && qok) {
      const int j0 = P.first_j[qorig];
      if (j0 == 0x7FFFFFFF) qok = false;  // nobody asked for this point
      else init = ((unsigned long long)__float_as_uint(P.dis[j0]) << 32) | (unsigned)j0;
    }
    sqn[warp][lane] = qn;
    sbest[warp][lane] = init;
    sbound[warp][lane] = __float_as_int(filt_bound(fminf(lim, __uint_as_float((unsigned)(init >> 32)))));
    if (threadIdx.x < 3) s_need[threadIdx.x] = 0u;
  }
  if (!__syncthreads_or(qok ? 1 : 0)) {  // nothing to search for in this block
    if (mode == 0 && qi < nq && qorig >= 0) {
      P.nn[qorig] = -1;
      P.dis[qorig] = lim;
    }
    return;
  }
  const int nb = B.n;
  const int ntiles = (nb + NN_TILE - 1) / NN_TILE;
  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // first tile: where the code of the block's middle query would sit in the base order
    const uint32_t code = Q.fcode_s[min(nq - 1, q0 + NN_THREADS / 2)];
    int lo = 0, hi = nb;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (B.fcode_s[mid] < code) lo = mid + 1;
      else hi = mid;
    }
    s_t0 = min(ntiles - 1, lo / NN_TILE);
  }
  __syncthreads();
  const int t0 = s_t0, up = ntiles - t0;
  auto visit = [&](int k) { return k < up ? t0 + k : t0 - 1 - (k - up); };
  const float4* boxes = B.ftile;
  // does this thread's query still need tile t?  (lo = +inf when the tile has no base record)
  auto my_need = [&](int t) {
    if (!qok) return false;
    const float4 lo4 = __ldg(&boxes[2 * t]), hi4 = __ldg(&boxes[2 * t + 1]);
    return tile_lb(qn, lo4, hi4) <= __int_as_float(sbound[warp][lane]);
  };
  // First visit index >= k whose tile somebody in the block needs (ntiles if none).  The decision is taken for a CHUNK
  // of visits at a time (every thread tests its query against the chunk's boxes with its current bound, one block-wide
  // OR per chunk instead of one barrier per tile); the bound only tightens afterwards, so the mask is a superset and the
  // warps re-test at the visit.  The first chunks are short: a forward search starts with the gate as its bound.
  // Always at least one barrier per call: it also orders "every warp is done with the buffer about to be refilled"
  // before the refill.
  int cbase = 0, clen = 0, cslot = 0;
  unsigned cmask = 0u;
  auto next_needed = [&](int k) {
    bool synced = false;
    for (;;) {
      if (k >= ntiles) {
        if (!synced) __syncthreads();
        return ntiles;
      }
      if (k >= cbase + clen) {  // open the chunk that starts at visit k
        const int len = min(ntiles - k, clen == 0 ? 2 : (clen == 2 ? 6 : 32));
        unsigned m = 0u;
        if (qok) {
          const float bnd = __int_as_float(sbound[warp][lane]);
          for (int j = 0; j < len; j++) {
            const int t = visit(k + j);
            const float4 lo4 = __ldg(&boxes[2 * t]), hi4 = __ldg(&boxes[2 * t + 1]);
            if (tile_lb(qn, lo4, hi4) <= bnd) m |= 1u << j;
          }
        }
        m = __reduce_or_sync(0xffffffffu, m);
        if (lane == 0 && m) atomicOr(&s_need[cslot], m);
        __syncthreads();
        synced = true;
        cmask = s_need[cslot];
        cbase = k;
        clen = len;
        // the slot of the chunk after next is cleared now: its atomicOr's come after the NEXT chunk's barrier
        if (threadIdx.x == 0) s_need[(cslot + 2) % 3] = 0u;
        cslot = (cslot + 1) % 3;
      }
      const unsigned rem = cmask >> (k - cbase);
      if (rem) {
        if (!synced) __syncthreads();
        return k + __ffs(rem) - 1;
      }
      k = cbase + clen;
    }
  };
  auto issue = [&](int t, int buf) {
    const int cnt = min(NN_TILE, nb - t * NN_TILE);
    const unsigned bytes = (unsigned)cnt * FPAD * 4, nbytes = (unsigned)cnt * 16;
    mbar_expect_tx(&full[buf], bytes + nbytes);
    bulk_g2s(tile[buf], B.fpfh_s + (size_t)t * NN_TILE * FPAD, bytes, &full[buf]);
    bulk_g2s(tnorm[buf], B.fproj_s + (size_t)t * NN_TILE, nbytes, &full[buf]);
  };
  int qn_count = 0;  // entries in this warp's queue (warp-uniform)
  // refine up to 32 queued (query, record) pairs: one per lane
  auto drain = [&](const float* tb, int take) {
    if (lane < take) {
      const unsigned e = queue[warp][lane];
      const int ql = e >> 8, r = e & 255;
      // the query records stay in global memory (18 KB per block: L1-resident); shared memory is what limits the occupancy
      const float4* a4 = reinterpret_cast<const float4*>(Q.fpfh_s + (size_t)min(nq - 1, q0 + warp * 32 + ql) * FPAD);
      const float4* b4 = reinterpret_cast<const float4*>(tb + r * FPAD);
      float d = 0.f;
      float4 x, y;
#pragma unroll
      for (int k = 0; k < 8; k++) {
        x = __ldg(&a4[k]);
        y = b4[k];
        float e0;
        e0 = x.x - y.x; d += e0 * e0;
        e0 = x.y - y.y; d += e0 * e0;
        e0 = x.z - y.z; d += e0 * e0;
        e0 = x.w - y.w; d += e0 * e0;
      }
      x = __ldg(&a4[8]);
      y = b4[8];
      {
        const float e0 = x.x - y.x;
        d += e0 * e0;
      }
      // most refined pairs do not beat the current best (near-duplicate descriptors): look before the atomic
      const unsigned long long cand = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)__float_as_int(y.w);  // slot 35
      if (d < lim && cand < sbest[warp][ql]) {
        atomicMin(&sbest[warp][ql], cand);
        atomicMin(&sbound[warp][ql], __float_as_int(filt_bound(d)));
      }
    }
    __syncwarp();
    // compact the rest of the queue to the front
    const int rest = qn_count - take;
    unsigned short mv0 = 0, mv1 = 0;
    if (lane < rest) mv0 = queue[warp][take + lane];
    if (lane + 32 < rest) mv1 = queue[warp][take + lane + 32];
    __syncwarp();
    if (lane < rest) queue[warp][lane] = mv0;
    if (lane + 32 < rest) queue[warp][lane + 32] = mv1;
    __syncwarp();
    qn_count = rest;
  };
  int cur = next_needed(0);
  if (cur < ntiles && threadIdx.x == 0) issue(visit(cur), 0);
  for (int it = 0; cur < ntiles; it++) {
    const int nxt = next_needed(cur + 1);
    if (nxt < ntiles && threadIdx.x == 0) issue(visit(nxt), (it + 1) & 1);
    const int t = visit(cur);
    mbar_wait(&full[it & 1], (it >> 1) & 1);
    unsigned mask = __ballot_sync(0xffffffffu, my_need(t));  // the bound may have tightened since the block-level decision
    if (mask) {
      const float* tb = tile[it & 1];
      const float4* tn = tnorm[it & 1];
      const int cnt = min(NN_TILE, nb - t * NN_TILE);
      // this lane's two base records of the tile: filter coordinates and whether they are candidates (flag 1: not a duplicate)
      float4 bn0 = make_float4(0.f, 0.f, 0.f, 0.f), bn1 = bn0;
      bool ok0 = false, ok1 = false;
      if (lane < cnt) {
        bn0 = tn[lane];
        ok0 = tb[lane * FPAD + 34] == 1.f;
      }
      if (lane + 32 < cnt) {
        bn1 = tn[lane + 32];
        ok1 = tb[(lane + 32) * FPAD + 34] == 1.f;
      }
      while (mask) {
        const int ql = __ffs(mask) - 1;
        mask &= mask - 1;
        const float4 qv = sqn[warp][ql];  // broadcast
        const float bound = __int_as_float(sbound[warp][ql]);
        const bool p0 = ok0 && filt_lb(qv, bn0) <= bound;
        const bool p1 = ok1 && filt_lb(qv, bn1) <= bound;
        const unsigned m0 = __ballot_sync(0xffffffffu, p0), m1 = __ballot_sync(0xffffffffu, p1);
        const unsigned lt = (1u << lane) - 1u;
        if (p0) queue[warp][qn_count + __popc(m0 & lt)] = (unsigned short)((ql << 8) | lane);
        const int c0 = __popc(m0);
        if (p1) queue[warp][qn_count + c0 + __popc(m1 & lt)] = (unsigned short)((ql << 8) | (lane + 32));
        qn_count += c0 + __popc(m1);
        __syncwarp();
        while (qn_count >= 32) drain(tb, 32);
      }
      while (qn_count > 0) drain(tb, min(qn_count, 32));  // the queue refers to THIS tile: empty it before the tile is refilled
    }
    cur = nxt;
  }
  if (qi < nq && (mode == 0 || qok)) {
    const unsigned long long b = sbest[warp][lane];
    const int bo = (int)(b & 0xFFFFFFFFull);
    if (mode == 0) {
      if (qorig >= 0) {
        P.nn[qorig] = bo;  // 0xFFFFFFFF -> -1: nothing within the gate
        P.dis[qorig] = __uint_as_float((unsigned)(b >> 32));
      }
    } else {
      P.rnn[qorig] = bo;
    }
  }
}

__global__ void __launch_bounds__(256) k_match_init(const MatchDev* pairs) {
  const MatchDev& P = pairs[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.fi.n) {
    P.first_j[i] = 0x7FFFFFFF;
    P.rnn[i] = -1;
  }
  if (i < P.fj.n) P.tkey[i] = 0xFFFFFFFFu;
  if (i < 8) P.counters[i] = 0;
  if (i < 8) P.stats[i] = 0.0;
}

// gate on the FEATURE-space distance, remember the first (lowest) j that reaches each i (matcher.cc:441-447)
__global__ void __launch_bounds__(256) k_first_hit(const MatchDev* pairs, float thr2) {
  const MatchDev& P = pairs[blockIdx.y];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P.fj.n) return;
  const int i = P.nn[j];
  if (i < 0 || P.dis[j] > thr2) return;
  atomicMin(&P.first_j[i], j);
}

// ordered compaction over ascending original j: keep (i, j) iff j was the first hit of i AND nn_j(i) == j.
// advanced != 0 (Matcher::advancedMatching, TBB branch, matcher.cc:160-188): no gate, keep (nn(j), j) iff nn_j(nn(j)) == j.
__global__ void __launch_bounds__(1024) k_mutual(const MatchDev* pairs, float thr2, int advanced) {
  const MatchDev& P = pairs[blockIdx.x];
  __shared__ int wsum[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int nj = P.fj.n;
  for (int base = 0; base < nj; base += 1024) {
    const int j = base + threadIdx.x;
    int keep = 0, i = -1;
    if (j < nj) {
      i = P.nn[j];
      keep = (i >= 0 && !(P.dis[j] > thr2) && (advanced || P.first_j[i] == j) && P.rnn[i] == j) ? 1 : 0;
    }
    int incl = keep;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((threadIdx.x & 31) >= o) incl += t;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = incl;
    __syncthreads();
    if (threadIdx.x < 32) {
      const int w = wsum[threadIdx.x];
      int wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, wi, o);
        if (threadIdx.x >= o) wi += t;
      }
      wsum[threadIdx.x] = wi - w;
    }
    __syncthreads();
    const int pos = carry + wsum[threadIdx.x >> 5] + incl - keep;
    if (keep) {
      P.corres[2 * pos] = i;
      P.corres[2 * pos + 1] = j;
    }
    __syncthreads();
    if (threadIdx.x == 1023) carry = pos + keep;
    __syncthreads();
  }
  if (threadIdx.x == 0) P.counters[1] = carry;
}

// Matcher::normalizePoints: per-cloud mean (fp64 fixed-shape tree sum, cast to fp32) and the larger max radius.
// A deliberate deviation: the reference sums in fp32 in original point order (matcher.cc:70-76).  Kilometres from the
// map origin the two means differ by centimetres, which rescales every normalised length by ~1e-4 through the max radius
// but moves a length RATIO only by fp32 rounding (p - mean is exact there, Sterbenz).  The tuple test compares ratios
// only; tests/test_tuple_reference.py measures that no trial of it flips (20 pairs shifted by (3000, -2000, 50) m: mean
// gaps up to 19 mm, no verdict changed).
__global__ void __launch_bounds__(1024) k_cloud_sum(const MatchDev* pairs) {
  const MatchDev& P = pairs[blockIdx.y];
  const int which = blockIdx.z;
  const CloudDev& c = which == 0 ? P.fi : P.fj;
  double s[3] = {0, 0, 0};
  for (int i = threadIdx.x; i < c.n; i += 1024) {
    const float4 p = c.pts[i];
    s[0] += p.x; s[1] += p.y; s[2] += p.z;
  }
  __shared__ double red[32][3];
#pragma unroll
  for (int d = 0; d < 3; d++)
    for (int o = 16; o > 0; o >>= 1) s[d] += __shfl_down_sync(0xffffffffu, s[d], o);
  if ((threadIdx.x & 31) == 0)
    for (int d = 0; d < 3; d++) red[threadIdx.x >> 5][d] = s[d];
  __syncthreads();
  if (threadIdx.x < 3) {
    double t = 0;
    for (int w = 0; w < 32; w++) t += red[w][threadIdx.x];
    P.stats[3 * which + threadIdx.x] = t;
  }
}

__global__ void __launch_bounds__(256) k_cloud_scale(const MatchDev* pairs) {
  const MatchDev& P = pairs[blockIdx.y];
  const int which = blockIdx.z;
  const CloudDev& c = which == 0 ? P.fi : P.fj;
  const float mx = (float)(P.stats[3 * which + 0] / c.n), my = (float)(P.stats[3 * which + 1] / c.n), mz = (float)(P.stats[3 * which + 2] / c.n);
  float r = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < c.n; i += gridDim.x * blockDim.x) {
    const float4 p = c.pts[i];
    const float x = p.x - mx, y = p.y - my, z = p.z - mz;
    r = fmaxf(r, sqrtf((x * x + y * y) + z * z));
  }
  for (int o = 16; o > 0; o >>= 1) r = fmaxf(r, __shfl_xor_sync(0xffffffffu, r, o));
  if ((threadIdx.x & 31) == 0) atomicMax((int*)&P.stats[6], __float_as_int(r));  // r >= 0: int order == float order
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ int draw(unsigned long long seed, unsigned long long trial, int k, int n) {
  return (int)(splitmix64(seed ^ splitmix64(trial * 4 + k)) % (unsigned long long)n);
}

__device__ __forceinline__ void norm_point(const CloudDev& c, int orig, float mx, float my, float mz, float scale, float o[3]) {
  const float4 p = c.pts[c.rank[orig]];
  o[0] = p.x - mx; o[1] = p.y - my; o[2] = p.z - mz;
  if (scale != 1.0f) {
    o[0] /= scale; o[1] /= scale; o[2] /= scale;
  }
}
__device__ __forceinline__ float len3(const float a[3], const float b[3]) {
  const float d0 = a[0] - b[0], d1 = a[1] - b[1], d2 = a[2] - b[2];
  return sqrtf((d0 * d0 + d1 * d1) + d2 * d2);
}

// every trial evaluated independently (counter-based draws); a passing trial records, per correspondence,
// the earliest (trial, slot) at which the serial loop would have added it (matcher.cc:484-536)
__global__ void __launch_bounds__(256) k_tuple_trials(const MatchDev* pairs, QuatroParamsDev prm) {
  const MatchDev& P = pairs[blockIdx.y];
  const int ncorr = P.counters[1];
  // tuple_scale == 0: no trial runs.  optimizedMatching then keeps nothing (its tuple block is the only writer of corres_,
  // matcher.cc:461), so k_tuple_select finds no key; advancedMatching keeps every pair (k_adv_select's keepall).
  if (ncorr == 0 || prm.tuple_scale == 0.f) return;
  const long long trials = (long long)ncorr * 100;
  const float mxi = (float)(P.stats[0] / P.fi.n), myi = (float)(P.stats[1] / P.fi.n), mzi = (float)(P.stats[2] / P.fi.n);
  const float mxj = (float)(P.stats[3] / P.fj.n), myj = (float)(P.stats[4] / P.fj.n), mzj = (float)(P.stats[5] / P.fj.n);
  const float scale = __int_as_float(*(const int*)&P.stats[6]);
  const float ts = prm.tuple_scale;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < trials; t += (long long)gridDim.x * blockDim.x) {
    const int r0 = draw(prm.seed, t, 0, ncorr), r1 = draw(prm.seed, t, 1, ncorr);
    float pi0[3], pi1[3], pj0[3], pj1[3];
    norm_point(P.fi, P.corres[2 * r0], mxi, myi, mzi, scale, pi0);
    norm_point(P.fi, P.corres[2 * r1], mxi, myi, mzi, scale, pi1);
    norm_point(P.fj, P.corres[2 * r0 + 1], mxj, myj, mzj, scale, pj0);
    norm_point(P.fj, P.corres[2 * r1 + 1], mxj, myj, mzj, scale, pj1);
    const float li0 = len3(pi0, pi1), lj0 = len3(pj0, pj1);
    if (prm.advanced ? !((li0 * ts < lj0) && (lj0 < li0 / ts)) : ((li0 * ts > lj0) || (lj0 > li0 / ts))) continue;  // matcher.cc:314 / :509
    const int r2 = draw(prm.seed, t, 2, ncorr);
    float pi2[3], pj2[3];
    norm_point(P.fi, P.corres[2 * r2], mxi, myi, mzi, scale, pi2);
    norm_point(P.fj, P.corres[2 * r2 + 1], mxj, myj, mzj, scale, pj2);
    const float li1 = len3(pi1, pi2), li2 = len3(pi2, pi0), lj1 = len3(pj1, pj2), lj2 = len3(pj2, pj0);
    if ((li1 * ts < lj1) && (lj1 < li1 / ts) && (li2 * ts < lj2) && (lj2 < li2 / ts)) {
      const unsigned k = (unsigned)(t * 4);
      atomicMin(&P.tkey[r0], k);
      atomicMin(&P.tkey[r1], k + 1);
      atomicMin(&P.tkey[r2], k + 2);
    }
  }
}

// serial semantics recovered: the loop stops after the first trial that leaves more than max_corres unique
// correspondences; the survivors are emitted in insertion order.  One block per pair.
__global__ void __launch_bounds__(1024) k_tuple_select(const MatchDev* pairs, QuatroParamsDev prm) {
  const MatchDev& P = pairs[blockIdx.x];
  const int ncorr = P.counters[1];
  __shared__ unsigned hist[256];
  __shared__ unsigned prefix, remaining, tstar;
  __shared__ unsigned long long keys[1024];
  __shared__ int nsel;
  if (ncorr == 0) {
    if (threadIdx.x == 0) P.counters[2] = 0;
    return;
  }
  // (max_corres+1)-th smallest key by 4-pass radix select; none => keep everything
  if (threadIdx.x == 0) {
    prefix = 0;
    remaining = (unsigned)prm.max_corres + 1;
    tstar = 0xFFFFFFFFu;
  }
  __syncthreads();
  bool found = true;
  for (int pass = 3; pass >= 0 && found; pass--) {
    if (threadIdx.x < 256) hist[threadIdx.x] = 0;
    __syncthreads();
    const unsigned pfx = prefix;
    const int shift = pass * 8;
    for (int r = threadIdx.x; r < ncorr; r += 1024) {
      const unsigned k = P.tkey[r];
      if (k == 0xFFFFFFFFu) continue;
      if (pass == 3 || (k >> (shift + 8)) == (pfx >> (shift + 8))) atomicAdd(&hist[(k >> shift) & 255], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned rem = remaining, acc = 0;
      int b = 0;
      for (; b < 256; b++) {
        if (acc + hist[b] >= rem) break;
        acc += hist[b];
      }
      if (b == 256) {
        tstar = 0xFFFFFFFFu;  // fewer than max+1 unique additions in total
        remaining = 0;
      } else {
        prefix = pfx | ((unsigned)b << shift);
        remaining = rem - acc;
        if (pass == 0) tstar = prefix >> 2;  // trial index of the (max+1)-th addition
      }
    }
    __syncthreads();
    found = remaining != 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) nsel = 0;
  __syncthreads();
  const unsigned ts = tstar;
  for (int r = threadIdx.x; r < ncorr; r += 1024) {
    const unsigned k = P.tkey[r];
    if (k == 0xFFFFFFFFu) continue;
    if (ts == 0xFFFFFFFFu || (k >> 2) <= ts) {
      const int s = atomicAdd(&nsel, 1);
      if (s < 1024) keys[s] = ((unsigned long long)k << 32) | (unsigned)r;
    }
  }
  __syncthreads();
  const int n = min(nsel, MAXC);
  for (int s = threadIdx.x; s < 1024; s += 1024)
    if (s >= nsel) keys[s] = 0xFFFFFFFFFFFFFFFFull;
  __syncthreads();
  for (int k = 2; k <= 1024; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      const int i = threadIdx.x, l = i ^ j;
      if (l > i) {
        const unsigned long long a = keys[i], b = keys[l];
        const bool up = (i & k) == 0;
        if ((a > b) == up) {
          keys[i] = b;
          keys[l] = a;
        }
      }
      __syncthreads();
    }
  if ((int)threadIdx.x < n) {
    const int r = (int)(keys[threadIdx.x] & 0xFFFFFFFFu);
    const int i = P.corres[2 * r], j = P.corres[2 * r + 1];
    P.out_corr[2 * threadIdx.x] = P.swapped ? j : i;      // always (src, dst) (matcher.cc:527-535)
    P.out_corr[2 * threadIdx.x + 1] = P.swapped ? i : j;
  }
  if (threadIdx.x == 0) P.counters[2] = n;
}

// ------------------------------------------------------------------------------------------------
// Q5 TEASER++ solve (QUATRO rotation, PMC_HEU-style clique), one block per pair
// ------------------------------------------------------------------------------------------------
constexpr int SV_THREADS = 256;
constexpr int SV_WORDS = MAXC / 32;

struct SolveSmem {
  double S[MAXC][3], D[MAXC][3];
  unsigned adj[MAXC][SV_WORDS];
  unsigned radj[MAXC][SV_WORDS];
  int deg[MAXC], core[MAXC], rank[MAXC], order[MAXC], csize[MAXC];
  unsigned long long skey[MAXC];
  int clique[MAXC];
  double red[SV_THREADS];
  double w[MAXC], res[MAXC];
  double hval[2 * MAXC];
  int hidx[2 * MAXC];
  int m, best_r;
  double R2[4], mu, prev_cost, t[3];
  int stop;
};

// block reductions in a fixed order: butterfly inside each warp, then over the SV_THREADS / 32 warp results (two
// barriers per reduction; a shared-memory tree cost nine, and the GNC loop does six reductions per iteration)
__device__ __forceinline__ double block_sum(SolveSmem& sm, double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // the previous reduction's readers are done with sm.red
  if ((threadIdx.x & 31) == 0) sm.red[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = (threadIdx.x & 31) < SV_THREADS / 32 ? sm.red[threadIdx.x & 31] : 0.0;
  for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  return r;
}
__device__ __forceinline__ double block_max(SolveSmem& sm, double v) {  // of non-negative values
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm.red[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = (threadIdx.x & 31) < SV_THREADS / 32 ? sm.red[threadIdx.x & 31] : 0.0;
  for (int o = 16; o > 0; o >>= 1) r = fmax(r, __shfl_xor_sync(0xffffffffu, r, o));
  return r;
}

__global__ void __launch_bounds__(SV_THREADS) k_teaser_solve(const MatchDev* pairs, QuatroParamsDev prm) {
  extern __shared__ __align__(16) unsigned char smraw[];
  SolveSmem& sm = *reinterpret_cast<SolveSmem*>(smraw);
  const MatchDev& P = pairs[blockIdx.x];
  const int n = P.counters[2];
  const int tid = threadIdx.x;
  if (tid < 16) P.T[tid] = (tid % 5 == 0) ? 1.0 : 0.0;
  if (tid == 0) {
    P.counters[3] = 0;
    P.counters[4] = 0;
    P.counters[5] = 0;
  }
  if (n == 0) return;
  const CloudDev& src = P.swapped ? P.fj : P.fi;
  const CloudDev& dst = P.swapped ? P.fi : P.fj;
  for (int i = tid; i < n; i += SV_THREADS) {
    const float4 a = src.pts[src.rank[P.out_corr[2 * i]]], b = dst.pts[dst.rank[P.out_corr[2 * i + 1]]];
    sm.S[i][0] = a.x; sm.S[i][1] = a.y; sm.S[i][2] = a.z;
    sm.D[i][0] = b.x; sm.D[i][1] = b.y; sm.D[i][2] = b.z;
    for (int w = 0; w < SV_WORDS; w++) {
      sm.adj[i][w] = 0;
      sm.radj[i][w] = 0;
    }
  }
  __syncthreads();
  // TIM scale-consistency graph: | ||b_ij|| - ||a_ij|| | <= 2 * noise_bound (cbar2 = 1, quatro_module.cc:40)
  const double beta = 2.0 * prm.noise_bound;
  for (int e = tid; e < n * n; e += SV_THREADS) {
    const int i = e / n, j = e % n;
    if (j <= i) continue;
    double a = 0, b = 0;
#pragma unroll
    for (int d = 0; d < 3; d++) {
      const double da = sm.S[j][d] - sm.S[i][d], db = sm.D[j][d] - sm.D[i][d];
      a += da * da;
      b += db * db;
    }
    if (fabs(sqrt(a) - sqrt(b)) <= beta) {
      atomicOr(&sm.adj[i][j >> 5], 1u << (j & 31));
      atomicOr(&sm.adj[j][i >> 5], 1u << (i & 31));
    }
  }
  __syncthreads();
  for (int i = tid; i < n; i += SV_THREADS) {
    int d = 0;
    for (int w = 0; w < SV_WORDS; w++) d += __popc(sm.adj[i][w]);
    sm.deg[i] = d;
    sm.csize[i] = d;  // csize doubles as the peeling degree
    sm.rank[i] = 1;   // alive flag during peeling
  }
  __syncthreads();
  // core numbers: peel the minimum-degree vertex (lowest index on ties); one warp, lanes own strided vertices
  if (tid < 32) {
    int k = 0;
    for (int it = 0; it < n; it++) {
      int bv = 0x7FFFFFFF, bi = -1;
      for (int v = tid; v < n; v += 32)
        if (sm.rank[v] && (sm.csize[v] < bv)) {
          bv = sm.csize[v];
          bi = v;
        }
      for (int o = 16; o > 0; o >>= 1) {
        const int ov = __shfl_xor_sync(0xffffffffu, bv, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov < bv || (ov == bv && oi >= 0 && (bi < 0 || oi < bi))) {
          bv = ov;
          bi = oi;
        }
      }
      k = max(k, bv);
      __syncwarp();  // every lane has finished reading the alive flags of this round before lane 0 clears one
      if (tid == 0) {
        sm.core[bi] = k;
        sm.rank[bi] = 0;
      }
      __syncwarp();
      for (int v = tid; v < n; v += 32)
        if (sm.rank[v] && ((sm.adj[bi][v >> 5] >> (v & 31)) & 1u)) sm.csize[v]--;
      __syncwarp();
    }
  }
  __syncthreads();
  // order by (core desc, degree desc, index asc): bitonic sort of packed keys
  for (int i = tid; i < MAXC; i += SV_THREADS)
    sm.skey[i] = i < n ? (((unsigned long long)(MAXC - sm.core[i]) << 40) | ((unsigned long long)(MAXC - sm.deg[i]) << 20) | (unsigned)i)
                       : 0xFFFFFFFFFFFFFFFFull;
  __syncthreads();
  for (int k = 2; k <= MAXC; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < MAXC; i += SV_THREADS) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = sm.skey[i], b = sm.skey[l];
          const bool up = (i & k) == 0;
          if ((a > b) == up) {
            sm.skey[i] = b;
            sm.skey[l] = a;
          }
        }
      }
      __syncthreads();
    }
  for (int r = tid; r < n; r += SV_THREADS) {
    const int v = (int)(sm.skey[r] & 0xFFFFF);
    sm.order[r] = v;
    sm.rank[v] = r;
  }
  __syncthreads();
  // adjacency in rank space: "first vertex of P in the global order" becomes "lowest set bit"
  for (int v = tid; v < n; v += SV_THREADS) {
    const int rv = sm.rank[v];
    for (int u = 0; u < n; u++)
      if ((sm.adj[v][u >> 5] >> (u & 31)) & 1u) {
        const int ru = sm.rank[u];
        sm.radj[rv][ru >> 5] |= 1u << (ru & 31);  // row rv is written by this thread only
      }
  }
  __syncthreads();
  // greedy clique from every start vertex (independent => one thread each)
  for (int r = tid; r < n; r += SV_THREADS) {
    unsigned Pm[SV_WORDS];
    for (int w = 0; w < SV_WORDS; w++) Pm[w] = sm.radj[r][w];
    int size = 1;
    for (;;) {
      int u = -1;
      for (int w = 0; w < SV_WORDS; w++)
        if (Pm[w]) {
          u = w * 32 + __ffs(Pm[w]) - 1;
          break;
        }
      if (u < 0) break;
      size++;
      for (int w = 0; w < SV_WORDS; w++) Pm[w] &= sm.radj[u][w];
    }
    sm.csize[r] = size;
  }
  __syncthreads();
  if (tid == 0) {
    int best = 0, br = 0;
    for (int r = 0; r < n; r++)
      if (sm.csize[r] > best) {
        best = sm.csize[r];
        br = r;
      }
    // replay the winner and list its members (ascending ORIGINAL correspondence index)
    unsigned Pm[SV_WORDS], Cm[SV_WORDS];
    for (int w = 0; w < SV_WORDS; w++) {
      Pm[w] = sm.radj[br][w];
      Cm[w] = 0;
    }
    {
      const int v = sm.order[br];
      Cm[v >> 5] |= 1u << (v & 31);
    }
    for (;;) {
      int u = -1;
      for (int w = 0; w < SV_WORDS; w++)
        if (Pm[w]) {
          u = w * 32 + __ffs(Pm[w]) - 1;
          break;
        }
      if (u < 0) break;
      const int v = sm.order[u];
      Cm[v >> 5] |= 1u << (v & 31);
      for (int w = 0; w < SV_WORDS; w++) Pm[w] &= sm.radj[u][w];
    }
    int m = 0;
    for (int v = 0; v < n; v++)
      if ((Cm[v >> 5] >> (v & 31)) & 1u) sm.clique[m++] = v;
    sm.m = m;
    P.counters[4] = m;
    if (P.clique)
      for (int k = 0; k < m; k++) P.clique[k] = sm.clique[k];
  }
  __syncthreads();
  const int m = sm.m;
  if (m <= 1) return;  // solution_.valid stays false
  const int nt = m - 1;
  // GNC-TLS with a weighted 2-D (yaw-only) Kabsch step on the chain TIMs
  double nb2 = prm.noise_bound * prm.noise_bound;
  if (nb2 < 1e-16) nb2 = 1e-2;
  for (int k = tid; k < nt; k += SV_THREADS) sm.w[k] = 1.0;
  if (tid == 0) {
    sm.mu = 1.0;
    sm.prev_cost = INFINITY;
    sm.stop = 0;
    sm.R2[0] = 1; sm.R2[1] = 0; sm.R2[2] = 0; sm.R2[3] = 1;
  }
  __syncthreads();
  int iters = 0;
  for (int it = 0; it < prm.max_iter; it++) {
    iters = it + 1;
    double h0 = 0, h1 = 0, h2 = 0, h3 = 0;
    for (int k = tid; k < nt; k += SV_THREADS) {
      const int c0 = sm.clique[k], c1 = sm.clique[k + 1];
      const double ax = sm.S[c1][0] - sm.S[c0][0], ay = sm.S[c1][1] - sm.S[c0][1];
      const double bx = sm.D[c1][0] - sm.D[c0][0], by = sm.D[c1][1] - sm.D[c0][1];
      const double w = sm.w[k];
      h0 += ax * w * bx; h1 += ax * w * by; h2 += ay * w * bx; h3 += ay * w * by;
    }
    h0 = block_sum(sm, h0); h1 = block_sum(sm, h1); h2 = block_sum(sm, h2); h3 = block_sum(sm, h3);
    const double th = atan2(h1 - h2, h0 + h3);
    const double cs = cos(th), sn = sin(th);
    double mx = 0;
    for (int k = tid; k < nt; k += SV_THREADS) {
      const int c0 = sm.clique[k], c1 = sm.clique[k + 1];
      const double ax = sm.S[c1][0] - sm.S[c0][0], ay = sm.S[c1][1] - sm.S[c0][1], az = sm.S[c1][2] - sm.S[c0][2];
      const double bx = sm.D[c1][0] - sm.D[c0][0], by = sm.D[c1][1] - sm.D[c0][1], bz = sm.D[c1][2] - sm.D[c0][2];
      const double rx = bx - (cs * ax - sn * ay), ry = by - (sn * ax + cs * ay), rz = bz - az;
      sm.res[k] = rx * rx + ry * ry + rz * rz;
      mx = fmax(mx, sm.res[k]);
    }
    mx = block_max(sm, mx);
    if (tid == 0) {
      sm.R2[0] = cs; sm.R2[1] = -sn; sm.R2[2] = sn; sm.R2[3] = cs;
      if (it == 0) {
        sm.mu = 1.0 / (2.0 * mx / nb2 - 1.0);
        if (sm.mu <= 0) sm.stop = 1;
      }
    }
    __syncthreads();
    if (sm.stop) break;
    const double mu = sm.mu;
    const double th1 = (mu + 1) / mu * nb2, th2 = mu / (mu + 1) * nb2;
    double cost = 0;
    for (int k = tid; k < nt; k += SV_THREADS) {
      const double r = sm.res[k];
      cost += sm.w[k] * r;
      sm.w[k] = r >= th1 ? 0.0 : (r <= th2 ? 1.0 : sqrt(nb2 * mu * (mu + 1) / r) - mu);
    }
    cost = block_sum(sm, cost);
    if (tid == 0) {
      const double diff = fabs(cost - sm.prev_cost);
      sm.mu = mu * prm.gnc_factor;
      sm.prev_cost = cost;
      if (diff < prm.cost_thr) sm.stop = 1;
    }
    __syncthreads();
    if (sm.stop) break;
  }
  __syncthreads();
  // translation: per-axis TLS adaptive voting over dst_i - R src_i on the clique members
  const double range = prm.noise_bound;
  int sn = 2;  // sort size: the power of two that holds the 2m interval ends (not always 2 * MAXC)
  while (sn < 2 * m) sn <<= 1;
  for (int d = 0; d < 3; d++) {
    for (int k = tid; k < sn; k += SV_THREADS) {
      sm.hval[k] = INFINITY;
      sm.hidx[k] = 0;
    }
    __syncthreads();
    for (int k = tid; k < m; k += SV_THREADS) {
      const int c = sm.clique[k];
      const double rs = d == 0 ? sm.R2[0] * sm.S[c][0] + sm.R2[1] * sm.S[c][1] : (d == 1 ? sm.R2[2] * sm.S[c][0] + sm.R2[3] * sm.S[c][1] : sm.S[c][2]);
      const double x = sm.D[c][d] - rs;
      sm.res[k] = x;
      sm.hval[2 * k] = x - range; sm.hidx[2 * k] = k + 1;
      sm.hval[2 * k + 1] = x + range; sm.hidx[2 * k + 1] = -k - 1;
    }
    __syncthreads();
    // bitonic sort by (value, original slot) == std::stable_sort by value
    for (int k = 2; k <= sn; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < sn; i += SV_THREADS) {
          const int l = i ^ j;
          if (l > i) {
            const double a = sm.hval[i], b = sm.hval[l];
            const int ia = sm.hidx[i], ib = sm.hidx[l];
            // slot order of the unsorted array: 2k for +, 2k+1 for -
            const int sa = ia > 0 ? 2 * (ia - 1) : 2 * (-ia - 1) + 1, sb = ib > 0 ? 2 * (ib - 1) : 2 * (-ib - 1) + 1;
            const bool gt = a > b || (a == b && (ia == 0 ? 1 << 30 : sa) > (ib == 0 ? 1 << 30 : sb));
            const bool up = (i & k) == 0;
            if (gt == up) {
              sm.hval[i] = b; sm.hval[l] = a;
              sm.hidx[i] = ib; sm.hidx[l] = ia;
            }
          }
        }
        __syncthreads();
      }
    if (tid == 0) {
      const double w = 1.0 / (range * range);
      double ris = range * m, dxw = 0, dwc = 0, sxi = 0, sxq = 0, best_cost = INFINITY, best = 0;
      int card = 0;
      for (int i = 0; i < 2 * m; i++) {
        const int idx = abs(sm.hidx[i]) - 1;
        const int eps = sm.hidx[i] > 0 ? 1 : -1;
        const double X = sm.res[idx];
        card += eps;
        dwc += eps * w;
        dxw += eps * w * X;
        ris -= eps * range;
        sxi += eps * X;
        sxq += eps * X * X;
        const double xh = dxw / dwc;
        const double cost = (card * xh * xh + sxq - 2 * sxi * xh) + ris;
        if (cost < best_cost) {
          best_cost = cost;
          best = xh;
        }
      }
      sm.t[d] = best;
    }
    __syncthreads();
  }
  if (tid == 0) {
    P.T[0] = sm.R2[0]; P.T[1] = sm.R2[1]; P.T[2] = 0; P.T[3] = sm.t[0];
    P.T[4] = sm.R2[2]; P.T[5] = sm.R2[3]; P.T[6] = 0; P.T[7] = sm.t[1];
    P.T[8] = 0; P.T[9] = 0; P.T[10] = 1; P.T[11] = sm.t[2];
    P.T[12] = 0; P.T[13] = 0; P.T[14] = 0; P.T[15] = 1;
    P.counters[3] = 1;
    P.counters[5] = iters;
  }
}

// ------------------------------------------------------------------------------------------------
// Matcher::advancedMatching tail + the TEASER++ solve for correspondence sets beyond MAXC: the same algorithm as
// k_teaser_solve, restated as a short chain of kernels over a global-memory workspace (BigSolveWs) so that a set of
// several thousand correspondences (8 MB of adjacency bits) is spread over the whole GPU.
// ------------------------------------------------------------------------------------------------
// every member of a passing triplet survives (matcher.cc:314-320); (src, dst) ordering, sort, unique (:338-355).
// The cross-checked pairs are unique already, so "unique" is a no-op; the sort is a bitonic sort of packed keys.
__global__ void __launch_bounds__(1024) k_adv_select(const MatchDev* pairs, QuatroParamsDev prm) {
  extern __shared__ __align__(16) unsigned long long akeys[];  // [BIGC]
  const MatchDev& P = pairs[blockIdx.x];
  const int ncorr = P.counters[1];
  const int cap = P.big->cap;
  __shared__ int nsel;
  if (threadIdx.x == 0) nsel = 0;
  __syncthreads();
  const bool keepall = prm.tuple_scale == 0.f;  // "use_tuple_test && tuple_scale != 0" (matcher.cc:272)
  for (int r = threadIdx.x; r < ncorr; r += 1024) {
    if (!keepall && P.tkey[r] == 0xFFFFFFFFu) continue;
    const int s = atomicAdd(&nsel, 1);
    if (s < cap) {
      const int i = P.corres[2 * r], j = P.corres[2 * r + 1];
      akeys[s] = ((unsigned long long)(unsigned)(P.swapped ? j : i) << 32) | (unsigned)(P.swapped ? i : j);
    }
  }
  __syncthreads();
  const int total = nsel;
  if (total > cap) {  // reported as B200REG_ESTATE by the host; nothing is solved
    if (threadIdx.x == 0) {
      P.counters[2] = 0;
      P.counters[6] = total;
    }
    return;
  }
  int n2 = 2;
  while (n2 < total) n2 <<= 1;
  for (int i = total + threadIdx.x; i < n2; i += 1024) akeys[i] = 0xFFFFFFFFFFFFFFFFull;
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n2; i += 1024) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = akeys[i], b = akeys[l];
          if ((a > b) == ((i & k) == 0)) {
            akeys[i] = b;
            akeys[l] = a;
          }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < total; i += 1024) {
    P.out_corr[2 * i] = (int)(akeys[i] >> 32);
    P.out_corr[2 * i + 1] = (int)(akeys[i] & 0xFFFFFFFFull);
  }
  if (threadIdx.x == 0) P.counters[2] = total;
}

// ordered compaction by one block of 1024 threads: emit(pos, v) for every v < n with keep(v), pos ascending with v.
// Returns the number kept (to every thread).
template <class Keep, class Emit>
__device__ int block_compact(int n, Keep keep, Emit emit) {
  __shared__ int wsum[32];
  __shared__ int carry;
  const int tid = threadIdx.x;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int v = base + tid;
    const int k = (v < n && keep(v)) ? 1 : 0;
    int incl = k;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((tid & 31) >= o) incl += t;
    }
    if ((tid & 31) == 31) wsum[tid >> 5] = incl;
    __syncthreads();
    if (tid < 32) {
      const int w = wsum[tid];
      int wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, wi, o);
        if (tid >= o) wi += t;
      }
      wsum[tid] = wi - w;
    }
    __syncthreads();
    const int pos = carry + wsum[tid >> 5] + incl - k;
    if (k) emit(pos, v);
    __syncthreads();
    if (tid == 1023) carry = pos + k;
    __syncthreads();
  }
  return carry;
}

// k_adv_select for a set larger than BIGC (one pair, one block; W.slot holds a source cloud's worth of ints).  The
// cross-checked pairs are one-to-one: (i, j) is kept only if j = rnn[i], so no fi point appears twice, and no fj point
// either (k_mutual lists each j once).  Hence the (src, dst) order is the order of src alone: scatter dst by src and
// compact in source-index order.  Same list as k_adv_select's sort, for any size.
__global__ void __launch_bounds__(1024) k_adv_select_wide(const MatchDev* pairs, QuatroParamsDev prm) {
  const MatchDev& P = pairs[blockIdx.x];
  const BigSolveWs& W = *P.big;
  const int ncorr = P.counters[1];
  const int nsrc = P.swapped ? P.fj.n : P.fi.n;
  const bool keepall = prm.tuple_scale == 0.f;
  for (int v = threadIdx.x; v < nsrc; v += 1024) W.slot[v] = -1;
  __syncthreads();
  for (int r = threadIdx.x; r < ncorr; r += 1024) {
    if (!keepall && P.tkey[r] == 0xFFFFFFFFu) continue;
    const int i = P.corres[2 * r], j = P.corres[2 * r + 1];
    W.slot[P.swapped ? j : i] = P.swapped ? i : j;
  }
  __syncthreads();
  const int total = block_compact(
      nsrc, [&](int v) { return W.slot[v] >= 0; },
      [&](int pos, int v) {
        P.out_corr[2 * pos] = v;
        P.out_corr[2 * pos + 1] = W.slot[v];
      });
  if (threadIdx.x == 0) P.counters[2] = total;
}

__global__ void __launch_bounds__(256) k_big_gather(const MatchDev* pairs) {
  const MatchDev& P = pairs[blockIdx.y];
  const BigSolveWs& W = *P.big;
  const int n = P.counters[2];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 16) P.T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  if (i == 0) {
    P.counters[3] = 0;
    P.counters[4] = 0;
    P.counters[5] = 0;
  }
  if (i >= n) return;
  const CloudDev& src = P.swapped ? P.fj : P.fi;
  const CloudDev& dst = P.swapped ? P.fi : P.fj;
  const float4 a = src.pts[src.rank[P.out_corr[2 * i]]], b = dst.pts[dst.rank[P.out_corr[2 * i + 1]]];
  W.S[3 * i] = a.x; W.S[3 * i + 1] = a.y; W.S[3 * i + 2] = a.z;
  W.D[3 * i] = b.x; W.D[3 * i + 1] = b.y; W.D[3 * i + 2] = b.z;
  W.deg[i] = 0;
}

// one thread per (vertex i, 32-vertex word w) of the TIM consistency graph: no atomics on the bit matrix; the test is
// symmetric bit for bit ((x - y)^2 == (y - x)^2), so row i and row j agree without communicating
__global__ void __launch_bounds__(256) k_big_tim(const MatchDev* pairs, QuatroParamsDev prm) {
  const MatchDev& P = pairs[blockIdx.y];
  const BigSolveWs& W = *P.big;
  const int n = P.counters[2];
  const int wn = (n + 31) >> 5;
  const double beta = 2.0 * prm.noise_bound;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < (long long)n * wn; idx += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(idx / wn), w = (int)(idx % wn);
    const double sx = W.S[3 * i], sy = W.S[3 * i + 1], sz = W.S[3 * i + 2];
    const double dx = W.D[3 * i], dy = W.D[3 * i + 1], dz = W.D[3 * i + 2];
    unsigned bits = 0;
    const int jend = min(32, n - w * 32);
    for (int b = 0; b < jend; b++) {
      const int j = w * 32 + b;
      if (j == i) continue;
      double a = 0, c = 0, t;
      t = W.S[3 * j] - sx; a += t * t;
      t = W.S[3 * j + 1] - sy; a += t * t;
      t = W.S[3 * j + 2] - sz; a += t * t;
      t = W.D[3 * j] - dx; c += t * t;
      t = W.D[3 * j + 1] - dy; c += t * t;
      t = W.D[3 * j + 2] - dz; c += t * t;
      if (fabs(sqrt(a) - sqrt(c)) <= beta) bits |= 1u << b;
    }
    W.adj[(size_t)i * W.words + w] = bits;
    if (bits) atomicAdd(&W.deg[i], __popc(bits));
  }
}

__device__ __forceinline__ int block_min_i(int v, int* red) {
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();  // red may still be read from the previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int r = red[threadIdx.x & 31];
  for (int o = 16; o > 0; o >>= 1) r = min(r, __shfl_xor_sync(0xffffffffu, r, o));
  return r;
}

// core numbers by level-synchronous peeling (every vertex whose remaining degree is <= the current level leaves in
// the same round); core numbers do not depend on the peeling order, so this equals the one-at-a-time peel of
// k_teaser_solve / the oracle.  Then the clique order (core desc, degree desc, index asc).  One block per pair.
__global__ void __launch_bounds__(1024) k_big_core(const MatchDev* pairs) {
  const MatchDev& P = pairs[blockIdx.x];
  const BigSolveWs& W = *P.big;
  const int n = P.counters[2];
  if (n == 0) return;
  const int wn = (n + 31) >> 5;
  const int tid = threadIdx.x;
  __shared__ int red[32];
  __shared__ int nf;
  for (int v = tid; v < n; v += 1024) {
    W.pdeg[v] = W.deg[v];
    W.alive[v] = 1;
  }
  __syncthreads();
  int remaining = n, k = 0;
  while (remaining > 0) {
    int mn = 0x7FFFFFFF;
    for (int v = tid; v < n; v += 1024)
      if (W.alive[v]) mn = min(mn, W.pdeg[v]);
    mn = block_min_i(mn, red);
    k = max(k, mn);
    if (tid == 0) nf = 0;
    __syncthreads();
    for (int v = tid; v < n; v += 1024)
      if (W.alive[v] && W.pdeg[v] <= k) {
        W.alive[v] = 0;
        W.core[v] = k;
        W.list[atomicAdd(&nf, 1)] = v;
      }
    __syncthreads();
    const int f = nf;
    for (long long idx = tid; idx < (long long)f * wn; idx += 1024) {
      const int fv = W.list[idx / wn], w = (int)(idx % wn);
      unsigned bits = W.adj[(size_t)fv * W.words + w];
      while (bits) {
        const int u = w * 32 + __ffs(bits) - 1;
        bits &= bits - 1;
        if (W.alive[u]) atomicSub(&W.pdeg[u], 1);
      }
    }
    __syncthreads();
    remaining -= f;
  }
  // core and degree are at most n - 1 and i < n < 2^20 (BIG_NMAX), so each field fits its bits
  int n2 = 2;
  while (n2 < n) n2 <<= 1;
  for (int i = tid; i < n2; i += 1024)
    W.skey[i] = i < n ? (((unsigned long long)(n - W.core[i]) << 40) | ((unsigned long long)(n - W.deg[i]) << 20) | (unsigned)i)
                      : 0xFFFFFFFFFFFFFFFFull;
  if (tid == 0) *W.best = 0;
  __syncthreads();
  for (int kk = 2; kk <= n2; kk <<= 1)
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < n2; i += 1024) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = W.skey[i], b = W.skey[l];
          if ((a > b) == ((i & kk) == 0)) {
            W.skey[i] = b;
            W.skey[l] = a;
          }
        }
      }
      __syncthreads();
    }
  for (int r = tid; r < n; r += 1024) {
    const int v = (int)(W.skey[r] & 0xFFFFF);
    W.order[r] = v;
    W.rank[v] = r;
  }
}

// adjacency in rank space, one thread per (rank row, word)
__global__ void __launch_bounds__(256) k_big_radj(const MatchDev* pairs) {
  const MatchDev& P = pairs[blockIdx.y];
  const BigSolveWs& W = *P.big;
  const int n = P.counters[2];
  const int wn = (n + 31) >> 5;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < (long long)n * wn; idx += (long long)gridDim.x * blockDim.x) {
    const int rv = (int)(idx / wn), w = (int)(idx % wn);
    const unsigned* row = W.adj + (size_t)W.order[rv] * W.words;
    unsigned bits = 0;
    const int end = min(32, n - w * 32);
    for (int b = 0; b < end; b++) {
      const int u = W.order[w * 32 + b];
      bits |= ((row[u >> 5] >> (u & 31)) & 1u) << b;
    }
    W.radj[(size_t)rv * W.words + w] = bits;
  }
}

constexpr int BIG_WPL = BIGC / 32 / 32;  // candidate-set words per lane

// the order in which greedy cliques compete: larger clique first, then lower start rank
__device__ __forceinline__ unsigned long long clique_key(int size, int r) {
  return ((unsigned long long)size << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)r);
}

// the greedy clique grown from start vertex `r` by one warp: the candidate set lives in registers, word w in lane
// w % 32; "first candidate in the global order" is a warp-wide minimum over bit positions.  mark != nullptr lists
// the members (by original correspondence index) as flags.
__device__ __forceinline__ int warp_greedy_clique(const BigSolveWs& W, int wn, int r, int* mark) {
  const int lane = threadIdx.x & 31;
  unsigned Pm[BIG_WPL];
#pragma unroll
  for (int s = 0; s < BIG_WPL; s++) {
    const int w = s * 32 + lane;
    Pm[s] = w < wn ? W.radj[(size_t)r * W.words + w] : 0u;
  }
  if (mark && lane == 0) mark[W.order[r]] = 1;
  int size = 1;
  for (;;) {
    unsigned pos = 0xFFFFFFFFu;
#pragma unroll
    for (int s = 0; s < BIG_WPL; s++)
      if (pos == 0xFFFFFFFFu && Pm[s]) pos = (unsigned)((s * 32 + lane) * 32 + __ffs(Pm[s]) - 1);
    pos = __reduce_min_sync(0xffffffffu, pos);
    if (pos == 0xFFFFFFFFu) break;
    size++;
    if (mark && lane == 0) mark[W.order[pos]] = 1;
#pragma unroll
    for (int s = 0; s < BIG_WPL; s++) {
      const int w = s * 32 + lane;
      if (w < wn) Pm[s] &= W.radj[(size_t)pos * W.words + w];
    }
  }
  return size;
}

__global__ void __launch_bounds__(256) k_big_greedy(const MatchDev* pairs) {
  const MatchDev& P = pairs[blockIdx.y];
  const BigSolveWs& W = *P.big;
  const int n = P.counters[2];
  const int wn = (n + 31) >> 5;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  for (int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nwarps) {
    const int size = warp_greedy_clique(W, wn, r, nullptr);
    if ((threadIdx.x & 31) == 0) W.csize[r] = size;
  }
}

// warp_greedy_clique for any n: the candidate set lives in Pm[wn] (shared or global memory), word w always handled by
// lane w % 32, so no lane reads a word another lane wrote.  The chosen vertex is the lowest candidate and its own row has
// no bit at itself, so after each step every candidate lies above it: the pass starts at its 32-word block.
__device__ __forceinline__ int warp_greedy_clique_buf(const BigSolveWs& W, int wn, int r, unsigned* Pm, int* mark) {
  const int lane = threadIdx.x & 31;
  const unsigned* row = W.radj + (size_t)r * W.words;
  unsigned pos = 0xFFFFFFFFu;
  for (int w = lane; w < wn; w += 32) {
    const unsigned b = row[w];
    Pm[w] = b;
    if (pos == 0xFFFFFFFFu && b) pos = (unsigned)(w * 32 + __ffs(b) - 1);
  }
  pos = __reduce_min_sync(0xffffffffu, pos);
  if (mark && lane == 0) mark[W.order[r]] = 1;
  int size = 1;
  while (pos != 0xFFFFFFFFu) {
    size++;
    if (mark && lane == 0) mark[W.order[pos]] = 1;
    const unsigned* urow = W.radj + (size_t)pos * W.words;
    unsigned next = 0xFFFFFFFFu;
    for (int w = (int)((pos >> 5) & ~31u) + lane; w < wn; w += 32) {
      const unsigned b = Pm[w] & urow[w];
      Pm[w] = b;
      if (next == 0xFFFFFFFFu && b) next = (unsigned)(w * 32 + __ffs(b) - 1);
    }
    pos = __reduce_min_sync(0xffffffffu, next);
  }
  return size;
}

// The greedy cliques of a set of any size (one pair): one warp per start rank, its candidate set in shared memory.
// Pruning keeps the winner.  The winner is the start with the largest clique_key(size, r) (largest clique, lowest rank on
// ties).  A clique grown from r lies in r's neighbourhood and every member has at least size - 1 neighbours inside it,
// so size <= core(r) + 1 and clique_key(core(r) + 1, r) bounds r's key.  W.best only ever holds keys that some start
// reached, so it never exceeds the winner's key: a start whose bound is below W.best cannot be the winner and is skipped
// (csize 0), and the winner is never skipped.  Ranks are ordered by core number descending and blocks start roughly in
// rank order, so the large cores run first and set W.best early.
__global__ void __launch_bounds__(256) k_big_greedy_wide(const MatchDev* pairs) {
  extern __shared__ unsigned cand[];  // [warps per block][wn]
  const MatchDev& P = pairs[blockIdx.y];
  const BigSolveWs& W = *P.big;
  const int n = P.counters[2];
  const int wn = (n + 31) >> 5;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= n) return;
  const unsigned long long seen = *(volatile unsigned long long*)W.best;
  int size = 0;
  if (clique_key(W.core[W.order[r]] + 1, r) >= seen) size = warp_greedy_clique_buf(W, wn, r, cand + (threadIdx.x >> 5) * wn, nullptr);
  if ((threadIdx.x & 31) == 0) {
    W.csize[r] = size;
    if (size) atomicMax(W.best, clique_key(size, r));
  }
}

__device__ __forceinline__ double block_sum_d(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = red[threadIdx.x & 31];
  for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  return r;
}
__device__ __forceinline__ double block_max_d(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = red[threadIdx.x & 31];
  for (int o = 16; o > 0; o >>= 1) r = fmax(r, __shfl_xor_sync(0xffffffffu, r, o));
  return r;
}

// pick the largest clique (lowest rank on ties), list it, GNC-TLS yaw rotation, TLS translation.  One block per pair.
__global__ void __launch_bounds__(1024) k_big_finish(const MatchDev* pairs, QuatroParamsDev prm, int wide) {
  const MatchDev& P = pairs[blockIdx.x];
  const BigSolveWs& W = *P.big;
  const int n = P.counters[2];
  if (n == 0) return;
  const int wn = (n + 31) >> 5;
  const int tid = threadIdx.x;
  __shared__ double red[32];
  __shared__ unsigned long long kred[32];
  __shared__ int stop;
  __shared__ double s_mu, s_prev, s_R2[4], s_t[3];
  constexpr int SWEEP = 2048;
  __shared__ double cX[SWEEP];
  __shared__ int cE[SWEEP];
  {
    unsigned long long key = 0;
    for (int r = tid; r < n; r += 1024) key = max(key, clique_key(W.csize[r], r));
    for (int o = 16; o > 0; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
    if ((tid & 31) == 0) kred[tid >> 5] = key;
    __syncthreads();
    key = kred[tid & 31];
    for (int o = 16; o > 0; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
    const int br = (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull));
    for (int v = tid; v < n; v += 1024) W.alive[v] = 0;  // member flags
    __syncthreads();
    if (tid < 32) {
      if (wide) warp_greedy_clique_buf(W, wn, br, (unsigned*)W.list, W.alive);  // list is free once k_big_core is done
      else warp_greedy_clique(W, wn, br, W.alive);
    }
    __syncthreads();
  }
  // members in ascending ORIGINAL correspondence index
  const int m = block_compact(
      n, [&](int v) { return W.alive[v] != 0; }, [&](int pos, int v) { W.clique[pos] = v; });
  if (tid == 0) P.counters[4] = m;
  if (m <= 1) return;  // solution_.valid stays false
  const int nt = m - 1;
  double nb2 = prm.noise_bound * prm.noise_bound;
  if (nb2 < 1e-16) nb2 = 1e-2;
  for (int k = tid; k < nt; k += 1024) W.w[k] = 1.0;
  if (tid == 0) {
    s_mu = 1.0;
    s_prev = INFINITY;
    stop = 0;
    s_R2[0] = 1; s_R2[1] = 0; s_R2[2] = 0; s_R2[3] = 1;
  }
  __syncthreads();
  int iters = 0;
  for (int it = 0; it < prm.max_iter; it++) {
    iters = it + 1;
    double h0 = 0, h1 = 0, h2 = 0, h3 = 0;
    for (int k = tid; k < nt; k += 1024) {
      const int c0 = W.clique[k], c1 = W.clique[k + 1];
      const double ax = W.S[3 * c1] - W.S[3 * c0], ay = W.S[3 * c1 + 1] - W.S[3 * c0 + 1];
      const double bx = W.D[3 * c1] - W.D[3 * c0], by = W.D[3 * c1 + 1] - W.D[3 * c0 + 1];
      const double w = W.w[k];
      h0 += ax * w * bx; h1 += ax * w * by; h2 += ay * w * bx; h3 += ay * w * by;
    }
    h0 = block_sum_d(h0, red); h1 = block_sum_d(h1, red); h2 = block_sum_d(h2, red); h3 = block_sum_d(h3, red);
    const double th = atan2(h1 - h2, h0 + h3);
    const double cs = cos(th), sn = sin(th);
    double mx = 0;
    for (int k = tid; k < nt; k += 1024) {
      const int c0 = W.clique[k], c1 = W.clique[k + 1];
      const double ax = W.S[3 * c1] - W.S[3 * c0], ay = W.S[3 * c1 + 1] - W.S[3 * c0 + 1], az = W.S[3 * c1 + 2] - W.S[3 * c0 + 2];
      const double bx = W.D[3 * c1] - W.D[3 * c0], by = W.D[3 * c1 + 1] - W.D[3 * c0 + 1], bz = W.D[3 * c1 + 2] - W.D[3 * c0 + 2];
      const double rx = bx - (cs * ax - sn * ay), ry = by - (sn * ax + cs * ay), rz = bz - az;
      const double r = rx * rx + ry * ry + rz * rz;
      W.res[k] = r;
      mx = fmax(mx, r);
    }
    mx = block_max_d(mx, red);
    if (tid == 0) {
      s_R2[0] = cs; s_R2[1] = -sn; s_R2[2] = sn; s_R2[3] = cs;
      if (it == 0) {
        s_mu = 1.0 / (2.0 * mx / nb2 - 1.0);
        if (s_mu <= 0) stop = 1;
      }
    }
    __syncthreads();
    if (stop) break;
    const double mu = s_mu;
    const double th1 = (mu + 1) / mu * nb2, th2 = mu / (mu + 1) * nb2;
    double cost = 0;
    for (int k = tid; k < nt; k += 1024) {
      const double r = W.res[k];
      cost += W.w[k] * r;
      W.w[k] = r >= th1 ? 0.0 : (r <= th2 ? 1.0 : sqrt(nb2 * mu * (mu + 1) / r) - mu);
    }
    cost = block_sum_d(cost, red);
    if (tid == 0) {
      const double diff = fabs(cost - s_prev);
      s_mu = mu * prm.gnc_factor;
      s_prev = cost;
      if (diff < prm.cost_thr) stop = 1;
    }
    __syncthreads();
    if (stop) break;
  }
  __syncthreads();
  const double range = prm.noise_bound;
  int n2 = 2;
  while (n2 < 2 * m) n2 <<= 1;
  for (int d = 0; d < 3; d++) {
    for (int k = tid; k < n2; k += 1024) {
      W.hval[k] = INFINITY;
      W.hidx[k] = 0;
    }
    __syncthreads();
    for (int k = tid; k < m; k += 1024) {
      const int c = W.clique[k];
      const double rs = d == 0 ? s_R2[0] * W.S[3 * c] + s_R2[1] * W.S[3 * c + 1] : (d == 1 ? s_R2[2] * W.S[3 * c] + s_R2[3] * W.S[3 * c + 1] : W.S[3 * c + 2]);
      const double x = W.D[3 * c + d] - rs;
      W.res[k] = x;
      W.hval[2 * k] = x - range; W.hidx[2 * k] = k + 1;
      W.hval[2 * k + 1] = x + range; W.hidx[2 * k + 1] = -k - 1;
    }
    __syncthreads();
    for (int k = 2; k <= n2; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < n2; i += 1024) {
          const int l = i ^ j;
          if (l > i) {
            const double a = W.hval[i], b = W.hval[l];
            const int ia = W.hidx[i], ib = W.hidx[l];
            const int sa = ia > 0 ? 2 * (ia - 1) : 2 * (-ia - 1) + 1, sb = ib > 0 ? 2 * (ib - 1) : 2 * (-ib - 1) + 1;
            const bool gt = a > b || (a == b && (ia == 0 ? 1 << 30 : sa) > (ib == 0 ? 1 << 30 : sb));
            if (gt == ((i & k) == 0)) {
              W.hval[i] = b; W.hval[l] = a;
              W.hidx[i] = ib; W.hidx[l] = ia;
            }
          }
        }
        __syncthreads();
      }
    // serial consensus sweep by one thread, fed from shared memory in chunks
    const double w = 1.0 / (range * range);
    double ris = range * m, dxw = 0, dwc = 0, sxi = 0, sxq = 0, best_cost = INFINITY, best = 0;
    int card = 0;
    for (int base = 0; base < 2 * m; base += SWEEP) {
      const int cnt = min(SWEEP, 2 * m - base);
      for (int i = tid; i < cnt; i += 1024) {
        const int h = W.hidx[base + i];
        cE[i] = h > 0 ? 1 : -1;
        cX[i] = W.res[abs(h) - 1];
      }
      __syncthreads();
      if (tid == 0)
        for (int i = 0; i < cnt; i++) {
          const int eps = cE[i];
          const double X = cX[i];
          card += eps;
          dwc += eps * w;
          dxw += eps * w * X;
          ris -= eps * range;
          sxi += eps * X;
          sxq += eps * X * X;
          const double xh = dxw / dwc;
          const double cost = (card * xh * xh + sxq - 2 * sxi * xh) + ris;
          if (cost < best_cost) {
            best_cost = cost;
            best = xh;
          }
        }
      __syncthreads();
    }
    if (tid == 0) s_t[d] = best;
    __syncthreads();
  }
  if (tid == 0) {
    P.T[0] = s_R2[0]; P.T[1] = s_R2[1]; P.T[2] = 0; P.T[3] = s_t[0];
    P.T[4] = s_R2[2]; P.T[5] = s_R2[3]; P.T[6] = 0; P.T[7] = s_t[1];
    P.T[8] = 0; P.T[9] = 0; P.T[10] = 1; P.T[11] = s_t[2];
    P.T[12] = 0; P.T[13] = 0; P.T[14] = 0; P.T[15] = 1;
    P.counters[3] = 1;
    P.counters[5] = iters;
  }
}

// coarse_aligned_ = transformPcd(src, T_quatro): double math, cast to float (utilities.hpp:164-175), ORIGINAL order,
// emitted as (x, y, z, 1) records so that it can be fed straight back into the index build
__global__ void __launch_bounds__(256) k_transform_raw(const CloudDev* clouds, const double* T16s, float4* const* outs) {
  const CloudDev& src = clouds[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= src.n) return;
  const float4 p = src.pts[i];
  const double* T = T16s + 16 * blockIdx.y;
  const double x = p.x, y = p.y, z = p.z;
  float4 o;
  o.x = (float)(T[0] * x + T[1] * y + T[2] * z + T[3]);
  o.y = (float)(T[4] * x + T[5] * y + T[6] * z + T[7]);
  o.z = (float)(T[8] * x + T[9] * y + T[10] * z + T[11]);
  o.w = 1.f;
  outs[blockIdx.y][__float_as_int(p.w)] = o;
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
int launch_fpfh(const CloudDev* d_clouds, int count, int max_n, float normal_r2, float fpfh_r2, cudaStream_t s) {
  dim3 grid((max_n + STEP_THREADS - 1) / STEP_THREADS, count);
  k_normals<<<grid, STEP_THREADS, 0, s>>>(d_clouds, normal_r2);
  k_spfh<<<grid, STEP_THREADS, 0, s>>>(d_clouds, fpfh_r2);
  k_fpfh<<<grid, STEP_THREADS, 0, s>>>(d_clouds, fpfh_r2);
  // the matcher's view: records in the order of their filter-space Morton code, duplicates collapsed, boxed per tile
  k_fcode<<<dim3((max_n + 255) / 256, count), 256, 0, s>>>(d_clouds);
  const int ls = launch_radix_sort(d_clouds, count, max_n, 32, s);  // 32-bit keys, 3 passes of 11 bits: result in keys[1] / vals[1]
  k_fgather<<<dim3((max_n + NN_TILE - 1) / NN_TILE, count), NN_TILE, 0, s>>>(d_clouds);
  return 5 + ls;
}

size_t solve_smem_bytes() { return sizeof(SolveSmem); }

constexpr int WIDE_SMEM = 227 * 1024;  // opt-in shared memory per block on sm_90

// Opt-in shared-memory sizes are a PER-DEVICE function attribute: b200reg_ctx_create calls this after cudaSetDevice, so
// every context (one per GPU in a multi-GPU process) gets them on its own device.
cudaError_t quatro_init_device() {
  cudaError_t e = cudaFuncSetAttribute(k_teaser_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SolveSmem));
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(k_big_greedy_wide, cudaFuncAttributeMaxDynamicSharedMemorySize, WIDE_SMEM);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(k_adv_select, cudaFuncAttributeMaxDynamicSharedMemorySize, BIGC * 8);
}

int launch_teaser_solve(const MatchDev* d_pairs, int count, const QuatroParamsDev& prm, cudaStream_t s) {
  k_teaser_solve<<<count, SV_THREADS, solve_smem_bytes(), s>>>(d_pairs, prm);
  return 1;
}

int launch_quatro_match_solve(const MatchDev* d_pairs, int count, int max_ni, int max_nj, const QuatroParamsDev& prm, cudaStream_t s) {
  int l = 0;
  k_match_init<<<dim3((max_ni + 255) / 256, count), 256, 0, s>>>(d_pairs); l++;
  k_cloud_sum<<<dim3(1, count, 2), 1024, 0, s>>>(d_pairs); l++;
  k_cloud_scale<<<dim3(64, count, 2), 256, 0, s>>>(d_pairs); l++;
  k_feat_nn<<<dim3((max_nj + NN_THREADS - 1) / NN_THREADS, count), NN_THREADS, 0, s>>>(d_pairs, 0, prm.thr2); l++;
  k_first_hit<<<dim3((max_nj + 255) / 256, count), 256, 0, s>>>(d_pairs, prm.thr2); l++;
  k_feat_nn<<<dim3((max_ni + NN_THREADS - 1) / NN_THREADS, count), NN_THREADS, 0, s>>>(d_pairs, 1, prm.thr2); l++;
  k_mutual<<<count, 1024, 0, s>>>(d_pairs, prm.thr2, prm.advanced); l++;
  k_tuple_trials<<<dim3(128, count), 256, 0, s>>>(d_pairs, prm); l++;
  if (!prm.advanced) {
    k_tuple_select<<<count, 1024, 0, s>>>(d_pairs, prm); l++;
    return l + launch_teaser_solve(d_pairs, count, prm, s);
  }
  k_adv_select<<<count, 1024, BIGC * 8, s>>>(d_pairs, prm); l++;
  k_big_gather<<<dim3(BIGC / 256, count), 256, 0, s>>>(d_pairs); l++;
  return l + launch_big_graph_solve(d_pairs, count, prm, 0, s);
}

// one pair whose advancedMatching set outgrew k_adv_select (n > BIGC correspondences, counters[6] = n): select into the
// pair's own workspace, gather, solve
int launch_adv_wide(const MatchDev* d_pair, int n, const QuatroParamsDev& prm, cudaStream_t s) {
  k_adv_select_wide<<<1, 1024, 0, s>>>(d_pair, prm);
  k_big_gather<<<(n + 255) / 256, 256, 0, s>>>(d_pair);
  return 2 + launch_big_graph_solve(d_pair, 1, prm, n, s);
}

// TEASER++ solve over the global-memory workspace (S / D gathered, counters[2] set): TIM graph, core order, greedy
// cliques, GNC-TLS.  n_wide == 0: sets of at most BIGC, candidate sets in registers, any batch; n_wide > 0: one pair of
// n_wide correspondences, candidate sets in shared memory and pruned starts (k_big_greedy_wide).
int launch_big_graph_solve(const MatchDev* d_pairs, int count, const QuatroParamsDev& prm, int n_wide, cudaStream_t s) {
  int l = 0;
  const int wide = 592 / count > 0 ? 592 / count : 1;  // ~4 CTAs per SM over the batch
  k_big_tim<<<dim3(wide, count), 256, 0, s>>>(d_pairs, prm); l++;
  k_big_core<<<count, 1024, 0, s>>>(d_pairs); l++;
  k_big_radj<<<dim3(wide, count), 256, 0, s>>>(d_pairs); l++;
  if (n_wide > 0) {
    const int wn = (n_wide + 31) / 32;
    const int wpb = std::min(8, WIDE_SMEM / (wn * 4));  // >= 1: n < 2^20 needs 128 KB per warp at most
    k_big_greedy_wide<<<dim3((n_wide + wpb - 1) / wpb, count), 32 * wpb, (size_t)wpb * wn * 4, s>>>(d_pairs); l++;
  } else {
    k_big_greedy<<<dim3(wide, count), 256, 0, s>>>(d_pairs); l++;
  }
  k_big_finish<<<count, 1024, 0, s>>>(d_pairs, prm, n_wide > 0); l++;
  return l;
}

void launch_transform_raw(const CloudDev* d_clouds, const double* d_T16s, int count, int max_n, float4* const* d_outs, cudaStream_t s) {
  k_transform_raw<<<dim3((max_n + 255) / 256, count), 256, 0, s>>>(d_clouds, d_T16s, d_outs);
}

}  // namespace b200
