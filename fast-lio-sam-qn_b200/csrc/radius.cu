// radius.cu -- batched fixed-radius search over one indexed cloud, CSR output (b200reg_radius_search).
//
// Replaces KdTreeFLANN::radiusSearch (third_party/nano_gicp/include/nano_gicp/nanoflann.hpp:154-175: RadiusResultSet
// through findNeighbors, .../impl/nanoflann_impl.hpp:229-262, 1354-1376) for a whole batch of queries:
//   k_rs_query_keys  Morton key of every query in the CLOUD's quantisation (its bounding box, 10 bits per axis), so that
//                    after a stable sort (launch_radix_sort) the 32 queries of a warp are spatial neighbours
//   k_rs_count       neighbour count per query: the warp-shared walk of knn.cuh (radius_visit_warp)
//   k_rs_tile_sums,  int64 exclusive scan of the counts in CALLER order -> the CSR offsets
//   k_rs_scan
//   k_rs_fill        the same walk again, every hit written at its query's offset (per chunk of queries)
//   k_rs_rekey +     segmented sort of a chunk's entries as stable LSD passes of launch_radix_sort: by original index,
//   launch_radix_sort  then (sorted mode) by d2, then by query -- ascending index, or ascending (d2, index), per query
//   k_rs_gather
// Exactness: d2 is dist2_rn (diff = query - point, ((dx*dx) + dy*dy) + dz*dz, no FMA), a point is kept iff d2 < r2
// (strict, RadiusResultSet::addPoint) and a subtree is skipped only when its box bound is >= r2 (radius_visit_warp).
// Every step is deterministic: the sort is stable, the walk visits a lane's exact set whatever its warp-mates are.
#include "knn.cuh"
#include "launchers.cuh"

namespace b200 {

constexpr int RS_THREADS = 128;
constexpr int RS_BUF = 16;  // per-lane hit buffer of the warp-shared walk (flushed when it could overflow within a leaf)
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__global__ void __launch_bounds__(256) k_rs_query_keys(CloudDev c, const float* q, int nq, int qstride, uint32_t* keys, uint32_t* vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  uint32_t key = 0;
  if (c.n > LEAF) {  // the root record holds both children's boxes: their union is the cloud's bounding box
    const NodeRec root = load_node(c.tnodes, 0);
    const float lo0 = fminf(root.lo0.x, root.lo1.x), lo1 = fminf(root.lo0.y, root.lo1.y), lo2 = fminf(root.lo0.z, root.lo1.z);
    const float ext = fmaxf(fmaxf(fmaxf(root.hi0.x, root.hi1.x) - lo0, fmaxf(root.hi0.y, root.hi1.y) - lo1), fmaxf(root.hi0.z, root.hi1.z) - lo2);
    const float scale = ext > 0.f ? 1023.0f / ext : 0.f;  // cubic cells, as k_morton_ghist quantises the cloud itself
    const float* p = q + (size_t)i * qstride;
    const uint32_t q0 = (uint32_t)min(max((int)((p[0] - lo0) * scale), 0), 1023);
    const uint32_t q1 = (uint32_t)min(max((int)((p[1] - lo1) * scale), 0), 1023);
    const uint32_t q2 = (uint32_t)min(max((int)((p[2] - lo2) * scale), 0), 1023);
    key = (expand10(q2) << 2) | (expand10(q1) << 1) | expand10(q0);
  }
  keys[i] = key;
  vals[i] = (uint32_t)i;
}

// one lane = one query, taken in Morton order (order[r] = caller index); counts in caller order
__global__ void __launch_bounds__(RS_THREADS) k_rs_count(CloudDev c, const float* q, int qstride, const uint32_t* order, int nq, float r2,
                                                         int* counts) {
  __shared__ int spos[RS_BUF * RS_THREADS];
  __shared__ int wstack[RS_THREADS / 32][MAX_STACK];
  const int r = blockIdx.x * RS_THREADS + threadIdx.x;
  const bool active = r < nq;
  const int qi = active ? (int)order[r] : 0;
  const float* p = q + (size_t)qi * qstride;
  const float qx = active ? p[0] : 0.f, qy = active ? p[1] : 0.f, qz = active ? p[2] : 0.f;
  int cnt = 0;
  radius_visit_warp<RS_BUF>(c, active, qx, qy, qz, r2, spos, nullptr, wstack[threadIdx.x >> 5], [&](int, float) { cnt++; });
  if (active) counts[qi] = cnt;
}

// per tile of SCAN_TILE counts: its sum
__global__ void __launch_bounds__(SCAN_THREADS) k_rs_tile_sums(const int* counts, int nq, long long* sums) {
  __shared__ long long red[SCAN_THREADS / 32];
  const int base = blockIdx.x * SCAN_TILE;
  long long s = 0;
  for (int j = threadIdx.x; j < SCAN_TILE; j += SCAN_THREADS)
    if (base + j < nq) s += counts[base + j];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int w = 0; w < SCAN_THREADS / 32; w++) t += red[w];
    sums[blockIdx.x] = t;
  }
}

// offsets[i] = sum of counts[0..i); the last tile also writes offsets[nq].  Every block re-adds the sums of the tiles
// before it (a few hundred values for 10^5..10^6 queries: cheaper than a third kernel).
__global__ void __launch_bounds__(SCAN_THREADS) k_rs_scan(const int* counts, int nq, const long long* sums, long long* offsets) {
  __shared__ long long red[SCAN_THREADS / 32];
  __shared__ long long s_prefix;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  long long pre = 0;
  for (int t = threadIdx.x; t < (int)blockIdx.x; t += SCAN_THREADS) pre += sums[t];
  for (int o = 16; o > 0; o >>= 1) pre += __shfl_xor_sync(0xffffffffu, pre, o);
  if (lane == 0) red[w] = pre;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int k = 0; k < SCAN_THREADS / 32; k++) t += red[k];
    s_prefix = t;
  }
  __syncthreads();
  // thread t owns SCAN_ITEMS consecutive counts
  const int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  int v[SCAN_ITEMS];
  long long run = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    v[k] = base + k < nq ? counts[base + k] : 0;
    run += v[k];
  }
  long long incl = run;
  for (int o = 1; o < 32; o <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  __syncthreads();
  if (lane == 31) red[w] = incl;
  __syncthreads();
  long long woff = s_prefix;
  for (int k = 0; k < w; k++) woff += red[k];
  long long e = woff + incl - run;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    if (base + k < nq) offsets[base + k] = e;
    e += v[k];
    if (base + k == nq - 1) offsets[nq] = e;
  }
}

// chunk id of every sorted query (starts: nchunks + 1 ascending caller indices): a stable sort by it groups the queries
// by chunk and keeps the Morton order inside each
__global__ void __launch_bounds__(256) k_rs_chunk_keys(const uint32_t* order, int nq, const int* starts, int nchunks, uint32_t* keys,
                                                       uint32_t* vals) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nq) return;
  const int qi = (int)order[r];
  int lo = 0, hi = nchunks - 1;  // last chunk whose start is <= qi
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (starts[mid] <= qi) lo = mid; else hi = mid - 1;
  }
  keys[r] = (uint32_t)lo;
  vals[r] = (uint32_t)qi;
}

__global__ void __launch_bounds__(RS_THREADS) k_rs_fill(CloudDev c, const float* q, int qstride, const uint32_t* order, float r2,
                                                        const long long* offsets, RadiusChunk ch) {
  __shared__ int spos[RS_BUF * RS_THREADS];
  __shared__ float sd2[RS_BUF * RS_THREADS];
  __shared__ int wstack[RS_THREADS / 32][MAX_STACK];
  const int r = blockIdx.x * RS_THREADS + threadIdx.x;
  const bool active = r < ch.nr;
  const int qi = active ? (int)order[ch.r0 + r] : 0;
  const float* p = q + (size_t)qi * qstride;
  const float qx = active ? p[0] : 0.f, qy = active ? p[1] : 0.f, qz = active ? p[2] : 0.f;
  int e = active ? (int)(offsets[qi] - ch.base) : 0;
  const uint32_t seg = (uint32_t)(qi - ch.q0);
  const float4* __restrict__ pts = c.pts;
  radius_visit_warp<RS_BUF>(c, active, qx, qy, qz, r2, spos, sd2, wstack[threadIdx.x >> 5], [&](int pos, float d2) {
    const int idx = __float_as_int(__ldg(&pts[pos].w));
    ch.e_idx[e] = idx;
    ch.e_d2[e] = d2;
    ch.e_seg[e] = seg;
    ch.keys[e] = (uint32_t)idx;
    ch.vals[e] = (uint32_t)e;
    e++;
  });
}

// keys[k] = src[perm[k]]: the next LSD key of the entries in their current order
__global__ void __launch_bounds__(256) k_rs_rekey(const uint32_t* perm, int m, const uint32_t* src, uint32_t* keys) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) keys[k] = src[perm[k]];
}

__global__ void __launch_bounds__(256) k_rs_gather(const uint32_t* perm, int m, const int* e_idx, const float* e_d2, int* idx_out,
                                                   float* d2_out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const uint32_t e = perm[k];
  idx_out[k] = e_idx[e];
  d2_out[k] = e_d2[e];
}

// ---------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------
static int blocks(int n, int t) { return (n + t - 1) / t; }

int launch_radius_query_keys(const CloudDev& c, const float* d_q, int nq, int qstride, uint32_t* keys, uint32_t* vals, cudaStream_t s) {
  k_rs_query_keys<<<blocks(nq, 256), 256, 0, s>>>(c, d_q, nq, qstride, keys, vals);
  return 1;
}

int launch_radius_count(const CloudDev& c, const float* d_q, int qstride, const uint32_t* order, int nq, float r2, int* counts,
                        cudaStream_t s) {
  k_rs_count<<<blocks(nq, RS_THREADS), RS_THREADS, 0, s>>>(c, d_q, qstride, order, nq, r2, counts);
  return 1;
}

size_t radius_scan_ws_bytes(int nq) { return (size_t)blocks(nq, SCAN_TILE) * sizeof(long long); }

int launch_radius_scan(const int* counts, int nq, int64_t* offsets, void* ws, cudaStream_t s) {
  const int tiles = blocks(nq, SCAN_TILE);
  k_rs_tile_sums<<<tiles, SCAN_THREADS, 0, s>>>(counts, nq, (long long*)ws);
  k_rs_scan<<<tiles, SCAN_THREADS, 0, s>>>(counts, nq, (const long long*)ws, (long long*)offsets);
  return 2;
}

int launch_radius_chunk_keys(const uint32_t* order, int nq, const int* starts, int nchunks, uint32_t* keys, uint32_t* vals,
                             cudaStream_t s) {
  k_rs_chunk_keys<<<blocks(nq, 256), 256, 0, s>>>(order, nq, starts, nchunks, keys, vals);
  return 1;
}

int launch_radius_fill(const CloudDev& c, const float* d_q, int qstride, const uint32_t* order, float r2, const int64_t* offsets,
                       const RadiusChunk& ch, cudaStream_t s) {
  k_rs_fill<<<blocks(ch.nr, RS_THREADS), RS_THREADS, 0, s>>>(c, d_q, qstride, order, r2, (const long long*)offsets, ch);
  return 1;
}

int launch_radius_rekey(const uint32_t* perm, int m, const uint32_t* src, uint32_t* keys, cudaStream_t s) {
  k_rs_rekey<<<blocks(m, 256), 256, 0, s>>>(perm, m, src, keys);
  return 1;
}

int launch_radius_gather(const uint32_t* perm, int m, const int* e_idx, const float* e_d2, int* idx_out, float* d2_out, cudaStream_t s) {
  k_rs_gather<<<blocks(m, 256), 256, 0, s>>>(perm, m, e_idx, e_d2, idx_out, d2_out);
  return 1;
}

}  // namespace b200
