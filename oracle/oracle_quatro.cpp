// oracle/oracle_quatro.cpp -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// CPU restatement of the Quatro half of the loop-closure path:
//   quatro<T>::align                      third_party/Quatro/src/quatro_module.cc:48-79
//   teaser::FPFHEstimation                third_party/Quatro/src/fpfh.cc:14-42  (PCL NormalEstimation + FPFHEstimationOMP)
//   teaser::Matcher::normalizePoints      third_party/Quatro/src/matcher.cc:58-116
//   teaser::Matcher::optimizedMatching    third_party/Quatro/src/matcher.cc:358-561
//   teaser::RobustRegistrationSolver      TEASER++ (not vendored), QUATRO rotation + PMC_HEU clique
// The PCL / FLANN / TEASER++ arithmetic is NOT in the reference tree; it is restated from their published
// algorithms as summarised in SURVEY.md App. B.  "Parity unpinned": no reference output exists for any
// of this (no tests, libraries not installable), and the reference stage is itself nondeterministic
// (srand(time(NULL)) matcher.cc:465; unsynchronised TBB writes :424-431).  Deliberate, documented
// definitions where the reference is order- or seed-dependent:
//   * normal covariance accumulated in fp64 (PCL 1.10 uses a single-pass fp32 accumulation whose
//     result depends on the neighbour order);
//   * pair features, histograms and feature distances in fp32 with a fixed sequential operation order;
//   * rand() replaced by a counter-based generator keyed by (seed, trial, draw);
//   * PMC's parallel heuristic replaced by a deterministic greedy k-core-ordered clique search.
#include <omp.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <numeric>
#include <vector>

#include "linalg.hpp"

namespace orq {

// ------------------------------------------------------------------------------------------
// uniform-grid fixed-radius search (independent of the product's LBVH)
struct Grid {
  float cell;
  float lo[3];
  int dim[3];
  std::vector<int> start;  // per cell
  std::vector<int> order;  // point indices sorted by cell
  const float* xyz;
  int n, stride;
  inline int cidx(const float* p, int d) const {
    int c = (int)std::floor((p[d] - lo[d]) / cell);
    return std::min(std::max(c, 0), dim[d] - 1);
  }
  void build(const float* xyz_, int n_, int stride_, float radius) {
    xyz = xyz_;
    n = n_;
    stride = stride_;
    cell = radius;
    float hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    lo[0] = lo[1] = lo[2] = INFINITY;
    for (int i = 0; i < n; i++)
      for (int d = 0; d < 3; d++) {
        lo[d] = std::min(lo[d], xyz[(size_t)i * stride + d]);
        hi[d] = std::max(hi[d], xyz[(size_t)i * stride + d]);
      }
    size_t cells = 1;
    for (int d = 0; d < 3; d++) {
      dim[d] = std::max(1, (int)std::floor((hi[d] - lo[d]) / cell) + 1);
      cells *= dim[d];
    }
    while (cells > (size_t)64 * 1024 * 1024) {  // keep the table bounded for huge extents
      cell *= 2;
      cells = 1;
      for (int d = 0; d < 3; d++) {
        dim[d] = std::max(1, (int)std::floor((hi[d] - lo[d]) / cell) + 1);
        cells *= dim[d];
      }
    }
    std::vector<int> cid(n);
    start.assign(cells + 1, 0);
    for (int i = 0; i < n; i++) {
      const float* p = &xyz[(size_t)i * stride];
      cid[i] = (cidx(p, 2) * dim[1] + cidx(p, 1)) * dim[0] + cidx(p, 0);
      start[cid[i] + 1]++;
    }
    for (size_t c = 0; c < cells; c++) start[c + 1] += start[c];
    order.resize(n);
    std::vector<int> cur(start.begin(), start.end() - 1);
    for (int i = 0; i < n; i++) order[cur[cid[i]]++] = i;  // ascending index inside a cell
  }
  // neighbours with fp32 d2 < r2 (FLANN RadiusResultSet: strict), ascending (d2, index) like
  // pcl::search::KdTree with sorted results
  void radius(const float* q, float r2, std::vector<std::pair<float, int>>& out) const {
    out.clear();
    int c0[3], c1[3];
    const float r = std::sqrt(r2);
    for (int d = 0; d < 3; d++) {
      float a[3] = {q[0], q[1], q[2]};
      a[d] = q[d] - r;
      c0[d] = cidx(a, d);
      a[d] = q[d] + r;
      c1[d] = cidx(a, d);
    }
    for (int z = c0[2]; z <= c1[2]; z++)
      for (int y = c0[1]; y <= c1[1]; y++)
        for (int x = c0[0]; x <= c1[0]; x++) {
          int c = (z * dim[1] + y) * dim[0] + x;
          for (int k = start[c]; k < start[c + 1]; k++) {
            int j = order[k];
            const float* p = &xyz[(size_t)j * stride];
            float d2 = 0.f;
            for (int d = 0; d < 3; d++) {
              float df = q[d] - p[d];
              d2 += df * df;
            }
            if (d2 < r2) out.emplace_back(d2, j);
          }
        }
    std::sort(out.begin(), out.end());
  }
};

// symmetric 3x3 eigenvector of the smallest eigenvalue (fp64 cyclic Jacobi on the SVD helper)
static void smallest_evec(const orc::M3& C, double n[3]) {
  orc::M3 U, V;
  double s[3];
  orc::m3_svd(C, U, s, V);
  n[0] = U(0, 2);
  n[1] = U(1, 2);
  n[2] = U(2, 2);
}

// pcl::NormalEstimation (fpfh.cc:27-32): radius neighbours incl. self, < 3 => NaN, normal = smallest
// eigenvector, flipped towards the viewpoint (0,0,0) of the MAP frame (SURVEY App. A.8 vi, B.4).
static void normals(const Grid& g, float radius, float* nrm /* n x 3 */) {
  const float r2 = (float)((double)radius * (double)radius);
#pragma omp parallel
  {
    std::vector<std::pair<float, int>> nb;
#pragma omp for schedule(dynamic, 64)
    for (int i = 0; i < g.n; i++) {
      const float* p = &g.xyz[(size_t)i * g.stride];
      g.radius(p, r2, nb);
      float* o = &nrm[(size_t)i * 3];
      if (nb.size() < 3) {
        o[0] = o[1] = o[2] = NAN;
        continue;
      }
      double m[3] = {0, 0, 0}, cc[6] = {0, 0, 0, 0, 0, 0};
      for (auto& e : nb) {
        const float* q = &g.xyz[(size_t)e.second * g.stride];
        const double x = (double)q[0] - (double)p[0], y = (double)q[1] - (double)p[1], z = (double)q[2] - (double)p[2];
        m[0] += x; m[1] += y; m[2] += z;
        cc[0] += x * x; cc[1] += x * y; cc[2] += x * z; cc[3] += y * y; cc[4] += y * z; cc[5] += z * z;
      }
      const double inv = 1.0 / (double)nb.size();
      for (int d = 0; d < 3; d++) m[d] *= inv;
      orc::M3 C;
      C(0, 0) = cc[0] * inv - m[0] * m[0];
      C(0, 1) = C(1, 0) = cc[1] * inv - m[0] * m[1];
      C(0, 2) = C(2, 0) = cc[2] * inv - m[0] * m[2];
      C(1, 1) = cc[3] * inv - m[1] * m[1];
      C(1, 2) = C(2, 1) = cc[4] * inv - m[1] * m[2];
      C(2, 2) = cc[5] * inv - m[2] * m[2];
      double nd[3];
      smallest_evec(C, nd);
      float nf[3] = {(float)nd[0], (float)nd[1], (float)nd[2]};
      // flipNormalTowardsViewpoint: (vp - p) . n < 0 => flip, vp = 0
      float cos_theta = (0.f - p[0]) * nf[0] + (0.f - p[1]) * nf[1] + (0.f - p[2]) * nf[2];
      if (cos_theta < 0.f) {
        nf[0] = -nf[0]; nf[1] = -nf[1]; nf[2] = -nf[2];
      }
      o[0] = nf[0]; o[1] = nf[1]; o[2] = nf[2];
    }
  }
}

// pcl::computePairFeatures (SURVEY App. B.5), fp32, fixed op order
static inline bool pair_features(const float* p1, const float* n1, const float* p2, const float* n2, float& f1, float& f2,
                                 float& f3, float& f4) {
  float dp[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  f4 = std::sqrt((dp[0] * dp[0] + dp[1] * dp[1]) + dp[2] * dp[2]);
  if (f4 == 0.f) return false;
  float a[3] = {n1[0], n1[1], n1[2]}, b[3] = {n2[0], n2[1], n2[2]};
  float angle1 = ((a[0] * dp[0] + a[1] * dp[1]) + a[2] * dp[2]) / f4;
  float angle2 = ((b[0] * dp[0] + b[1] * dp[1]) + b[2] * dp[2]) / f4;
  if (std::fabs(angle1) < std::fabs(angle2)) {  // acos(|angle1|) > acos(|angle2|): swap the roles
    for (int d = 0; d < 3; d++) {
      std::swap(a[d], b[d]);
      dp[d] = -dp[d];
    }
    f3 = -angle2;
  } else {
    f3 = angle1;
  }
  float v[3] = {dp[1] * a[2] - dp[2] * a[1], dp[2] * a[0] - dp[0] * a[2], dp[0] * a[1] - dp[1] * a[0]};
  float vn = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
  if (vn == 0.f) return false;
  v[0] /= vn; v[1] /= vn; v[2] /= vn;
  float w[3] = {a[1] * v[2] - a[2] * v[1], a[2] * v[0] - a[0] * v[2], a[0] * v[1] - a[1] * v[0]};
  f2 = (v[0] * b[0] + v[1] * b[1]) + v[2] * b[2];
  f1 = std::atan2((w[0] * b[0] + w[1] * b[1]) + w[2] * b[2], (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]);
  return true;
}

static inline int bin11(float v) {
  int h = (int)std::floor(v);
  return h < 0 ? 0 : (h > 10 ? 10 : h);
}

// FPFHEstimation::computePointSPFHSignature: 3 x 11 bins, increment 100/(|nbrs|-1)
static void spfh(const Grid& g, const float* nrm, float radius, float* out /* n x 33 */) {
  const float r2 = (float)((double)radius * (double)radius);
  const float d_pi = 1.0f / (2.0f * (float)M_PI);
#pragma omp parallel
  {
    std::vector<std::pair<float, int>> nb;
#pragma omp for schedule(dynamic, 64)
    for (int i = 0; i < g.n; i++) {
      float* h = &out[(size_t)i * 33];
      for (int k = 0; k < 33; k++) h[k] = 0.f;
      const float* p = &g.xyz[(size_t)i * g.stride];
      const float* np = &nrm[(size_t)i * 3];
      if (!std::isfinite(np[0])) continue;
      g.radius(p, r2, nb);
      if (nb.size() < 2) continue;
      const float incr = 100.0f / (float)(nb.size() - 1);
      for (auto& e : nb) {
        const int j = e.second;
        if (j == i) continue;
        const float* nq = &nrm[(size_t)j * 3];
        if (!std::isfinite(nq[0])) continue;
        float f1, f2, f3, f4;
        if (!pair_features(p, np, &g.xyz[(size_t)j * g.stride], nq, f1, f2, f3, f4)) continue;
        h[bin11(11.0f * ((f1 + (float)M_PI) * d_pi))] += incr;
        h[11 + bin11(11.0f * ((f2 + 1.0f) * 0.5f))] += incr;
        h[22 + bin11(11.0f * ((f3 + 1.0f) * 0.5f))] += incr;
      }
    }
  }
}

// FPFHEstimation::weightPointSPFHSignature: sum SPFH(q)/d2 over neighbours with d2 != 0, each
// 11-bin block rescaled to sum 100
static void fpfh(const Grid& g, const float* sp, const float* nrm, float radius, float* out /* n x 33 */) {
  const float r2 = (float)((double)radius * (double)radius);
#pragma omp parallel
  {
    std::vector<std::pair<float, int>> nb;
#pragma omp for schedule(dynamic, 64)
    for (int i = 0; i < g.n; i++) {
      float* h = &out[(size_t)i * 33];
      for (int k = 0; k < 33; k++) h[k] = 0.f;
      if (!std::isfinite(nrm[(size_t)i * 3])) continue;
      g.radius(&g.xyz[(size_t)i * g.stride], r2, nb);
      float sum[3] = {0.f, 0.f, 0.f};
      for (auto& e : nb) {
        if (e.first == 0.f) continue;
        const float w = 1.0f / e.first;
        const float* s = &sp[(size_t)e.second * 33];
        for (int b = 0; b < 3; b++)
          for (int k = 0; k < 11; k++) {
            const float v = s[11 * b + k] * w;
            sum[b] += v;
            h[11 * b + k] += v;
          }
      }
      for (int b = 0; b < 3; b++) {
        const float sc = sum[b] != 0.f ? 100.0f / sum[b] : 0.f;
        for (int k = 0; k < 11; k++) h[11 * b + k] *= sc;
      }
    }
  }
}

// FLANN L2 over 33 floats, fixed sequential fp32 order (SURVEY App. B.6)
static inline float feat_d2(const float* a, const float* b) {
  float r = 0.f;
  for (int k = 0; k < 33; k++) {
    const float d = a[k] - b[k];
    r += d * d;
  }
  return r;
}

// exact 1-NN of every query feature in `base` (ties: lower index); descriptors that are all zero
// (invalid normal) never match and are never matched
static void feature_nn(const float* q, int nq, const float* base, int nb, const unsigned char* base_ok, int* idx, float* d2) {
#pragma omp parallel for schedule(dynamic, 16)
  for (int i = 0; i < nq; i++) {
    float best = std::numeric_limits<float>::max();
    int bi = -1;
    for (int j = 0; j < nb; j++) {
      if (!base_ok[j]) continue;
      const float d = feat_d2(&q[(size_t)i * 33], &base[(size_t)j * 33]);
      if (d < best) {
        best = d;
        bi = j;
      }
    }
    idx[i] = bi;
    d2[i] = best;
  }
}

static inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
static inline int draw(uint64_t seed, uint64_t trial, int k, int n) {
  return (int)(splitmix64(seed ^ splitmix64(trial * 4 + k)) % (uint64_t)n);
}

struct Corr {
  int s, d;  // (source index, destination index)
};

// Matcher::optimizedMatching (matcher.cc:358-561).  Returns corres_ (always (src,dst) pairs).
// `mutual` receives the pre-tuple-test list in ascending-j order as (i, j) in fi/fj numbering.
static std::vector<Corr> optimized_matching(const float* src, int N, int sstride, const float* dst, int M, int dstride,
                                            const float* fsrc, const float* fdst, float thr_dist, int max_corr,
                                            float tuple_scale, uint64_t seed, std::vector<Corr>* mutual) {
  // fi = larger cloud, fj = smaller (matcher.cc:364-369)
  const bool swapped = M > N;
  const float* P[2] = {src, dst};
  const int np[2] = {N, M}, st[2] = {sstride, dstride};
  const float* F[2] = {fsrc, fdst};
  const int fi = swapped ? 1 : 0, fj = swapped ? 0 : 1;
  const int nPti = np[fi], nPtj = np[fj];
  // normalizePoints (matcher.cc:58-116): centre each cloud (fp32 running sum), divide by the larger max radius
  std::vector<float> pc[2];
  float scale = 0.f;
  for (int c = 0; c < 2; c++) {
    pc[c].resize((size_t)np[c] * 3);
    float mean[3] = {0.f, 0.f, 0.f};
    for (int i = 0; i < np[c]; i++)
      for (int d = 0; d < 3; d++) mean[d] = mean[d] + P[c][(size_t)i * st[c] + d];
    for (int d = 0; d < 3; d++) mean[d] = mean[d] / np[c];
    float mx = 0.f;
    for (int i = 0; i < np[c]; i++) {
      float v[3];
      for (int d = 0; d < 3; d++) v[d] = pc[c][(size_t)i * 3 + d] = P[c][(size_t)i * st[c] + d] - mean[d];
      float nrm = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
      if (nrm > mx) mx = nrm;
    }
    if (mx > scale) scale = mx;
  }
  if (scale != 1.0f)
    for (int c = 0; c < 2; c++)
      for (auto& v : pc[c]) v /= scale;

  std::vector<unsigned char> ok[2];
  for (int c = 0; c < 2; c++) {
    ok[c].assign(np[c], 0);
    for (int i = 0; i < np[c]; i++)
      for (int k = 0; k < 33; k++)
        if (F[c][(size_t)i * 33 + k] != 0.f) {
          ok[c][i] = 1;
          break;
        }
  }
  // every fj feature -> exact 1-NN in fi (matcher.cc:399)
  std::vector<int> nn(nPtj);
  std::vector<float> dis(nPtj);
  feature_nn(F[fj], nPtj, F[fi], nPti, ok[fi].data(), nn.data(), dis.data());
  // gate + first-hit reverse search + mutual check (matcher.cc:441-455; deterministic serial order)
  std::vector<int> i_to_j(nPti, -1);
  std::vector<int> need;  // the i's whose reverse NN is needed, in first-hit order
  std::vector<int> first_j(nPti, -1);
  const float thr2 = thr_dist * thr_dist;
  for (int j = 0; j < nPtj; j++) {
    if (!ok[fj][j] || nn[j] < 0) continue;
    if (dis[j] > thr2) continue;
    const int i = nn[j];
    if (first_j[i] == -1) {
      first_j[i] = j;
      need.push_back(i);
    }
  }
  std::vector<float> qf((size_t)need.size() * 33);
  for (size_t k = 0; k < need.size(); k++) std::memcpy(&qf[k * 33], &F[fi][(size_t)need[k] * 33], 33 * sizeof(float));
  std::vector<int> rnn(need.size());
  std::vector<float> rd(need.size());
  feature_nn(qf.data(), (int)need.size(), F[fj], nPtj, ok[fj].data(), rnn.data(), rd.data());
  std::vector<std::pair<int, int>> corres;  // (i, j), ascending j
  for (size_t k = 0; k < need.size(); k++)
    if (rnn[k] == first_j[need[k]]) corres.emplace_back(need[k], first_j[need[k]]);
  std::sort(corres.begin(), corres.end(), [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.second < b.second; });
  if (mutual) {
    mutual->clear();
    for (auto& c : corres) mutual->push_back({c.first, c.second});
  }
  // tuple test (matcher.cc:461-538) with the counter-based generator
  std::vector<Corr> out;
  const int ncorr = (int)corres.size();
  // tuple_scale == 0 skips the tuple block, the only writer of corres_ (matcher.cc:461-543): nothing is kept, and
  // quatro::align returns invalid with the identity (quatro_module.cc:63-66)
  if (ncorr == 0 || tuple_scale == 0.f) return out;
  std::vector<unsigned char> included(ncorr, 0);
  const long trials = (long)ncorr * 100;
  auto len = [&](int c, int a, int b) {
    const float* pa = &pc[c][(size_t)a * 3];
    const float* pb = &pc[c][(size_t)b * 3];
    const float d0 = pa[0] - pb[0], d1 = pa[1] - pb[1], d2 = pa[2] - pb[2];
    return std::sqrt((d0 * d0 + d1 * d1) + d2 * d2);
  };
  auto add = [&](int r) {
    if (!included[r]) {
      included[r] = 1;
      out.push_back(swapped ? Corr{corres[r].second, corres[r].first} : Corr{corres[r].first, corres[r].second});
    }
  };
  for (long t = 0; t < trials; t++) {
    const int r0 = draw(seed, t, 0, ncorr), r1 = draw(seed, t, 1, ncorr);
    const int idi0 = corres[r0].first, idj0 = corres[r0].second, idi1 = corres[r1].first, idj1 = corres[r1].second;
    const float li0 = len(fi, idi0, idi1), lj0 = len(fj, idj0, idj1);
    if ((li0 * tuple_scale > lj0) || (lj0 > li0 / tuple_scale)) continue;
    const int r2 = draw(seed, t, 2, ncorr);
    const int idi2 = corres[r2].first, idj2 = corres[r2].second;
    const float li1 = len(fi, idi1, idi2), li2 = len(fi, idi2, idi0);
    const float lj1 = len(fj, idj1, idj2), lj2 = len(fj, idj2, idj0);
    if ((li1 * tuple_scale < lj1) && (lj1 < li1 / tuple_scale) && (li2 * tuple_scale < lj2) && (lj2 < li2 / tuple_scale)) {
      add(r0);
      add(r1);
      add(r2);
    }
    if ((int)out.size() > max_corr) break;  // strictly greater: up to max+3 pairs (SURVEY A.8 iv)
  }
  return out;
}

// Matcher::advancedMatching (matcher.cc:118-356): forward 1-NN of every fj feature in fi (no distance gate), reverse
// 1-NN for every i that was hit, cross check (keep (i, j) iff j = nn_j(i) and nn_i(j) = i; the TBB branch :160-188
// lists them by ascending j, which fixes the index space of the random triplets), tuple test with ALL three edge
// ratios on 100*ncorr random triplets (every member of a passing triplet is kept, no cap), (src, dst) ordering,
// sort + unique.  use_crosscheck = false exists only in the non-TBB branch (:215-218).
static std::vector<Corr> advanced_matching(const float* src, int N, int sstride, const float* dst, int M, int dstride, const float* fsrc,
                                           const float* fdst, bool use_crosscheck, bool use_tuple_test, float tuple_scale,
                                           uint64_t seed) {
  const bool swapped = M > N;
  const float* P[2] = {src, dst};
  const int np[2] = {N, M}, st[2] = {sstride, dstride};
  const float* F[2] = {fsrc, fdst};
  const int fi = swapped ? 1 : 0, fj = swapped ? 0 : 1;
  const int nPti = np[fi], nPtj = np[fj];
  // normalizePoints, as in optimized_matching
  std::vector<float> pc[2];
  float scale = 0.f;
  for (int c = 0; c < 2; c++) {
    pc[c].resize((size_t)np[c] * 3);
    float mean[3] = {0.f, 0.f, 0.f};
    for (int i = 0; i < np[c]; i++)
      for (int d = 0; d < 3; d++) mean[d] = mean[d] + P[c][(size_t)i * st[c] + d];
    for (int d = 0; d < 3; d++) mean[d] = mean[d] / np[c];
    float mx = 0.f;
    for (int i = 0; i < np[c]; i++) {
      float v[3];
      for (int d = 0; d < 3; d++) v[d] = pc[c][(size_t)i * 3 + d] = P[c][(size_t)i * st[c] + d] - mean[d];
      float nrm = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
      if (nrm > mx) mx = nrm;
    }
    if (mx > scale) scale = mx;
  }
  if (scale != 1.0f)
    for (int c = 0; c < 2; c++)
      for (auto& v : pc[c]) v /= scale;
  std::vector<unsigned char> ok[2];
  for (int c = 0; c < 2; c++) {
    ok[c].assign(np[c], 0);
    for (int i = 0; i < np[c]; i++)
      for (int k = 0; k < 33; k++)
        if (F[c][(size_t)i * 33 + k] != 0.f) {
          ok[c][i] = 1;
          break;
        }
  }
  std::vector<int> nn(nPtj);
  std::vector<float> dis(nPtj);
  feature_nn(F[fj], nPtj, F[fi], nPti, ok[fi].data(), nn.data(), dis.data());
  std::vector<int> need;
  std::vector<unsigned char> hit(nPti, 0);
  for (int j = 0; j < nPtj; j++) {
    if (!ok[fj][j] || nn[j] < 0) continue;
    if (!hit[nn[j]]) {
      hit[nn[j]] = 1;
      need.push_back(nn[j]);
    }
  }
  std::vector<float> qf((size_t)need.size() * 33);
  for (size_t k = 0; k < need.size(); k++) std::memcpy(&qf[k * 33], &F[fi][(size_t)need[k] * 33], 33 * sizeof(float));
  std::vector<int> rnn(need.size());
  std::vector<float> rd(need.size());
  feature_nn(qf.data(), (int)need.size(), F[fj], nPtj, ok[fj].data(), rnn.data(), rd.data());
  std::vector<int> i_to_j(nPti, -1);
  for (size_t k = 0; k < need.size(); k++) i_to_j[need[k]] = rnn[k];
  std::vector<std::pair<int, int>> corres;  // (i, j)
  if (use_crosscheck) {
    for (int j = 0; j < nPtj; j++)  // ascending j (matcher.cc:181-186)
      if (ok[fj][j] && nn[j] >= 0 && i_to_j[nn[j]] == j) corres.emplace_back(nn[j], j);
  } else {  // corres_ij followed by corres_ji (matcher.cc:215-218)
    for (int i = 0; i < nPti; i++)
      if (i_to_j[i] != -1) corres.emplace_back(i, i_to_j[i]);
    for (int j = 0; j < nPtj; j++)
      if (ok[fj][j] && nn[j] >= 0) corres.emplace_back(nn[j], j);
  }
  const int ncorr = (int)corres.size();
  std::vector<std::pair<int, int>> kept;
  if (use_tuple_test && tuple_scale != 0.f && ncorr > 0) {
    std::vector<unsigned char> inc(ncorr, 0);
    auto len = [&](int c, int a, int b) {
      const float* pa = &pc[c][(size_t)a * 3];
      const float* pb = &pc[c][(size_t)b * 3];
      const float d0 = pa[0] - pb[0], d1 = pa[1] - pb[1], d2 = pa[2] - pb[2];
      return std::sqrt((d0 * d0 + d1 * d1) + d2 * d2);
    };
    const long trials = (long)ncorr * 100;
    for (long t = 0; t < trials; t++) {
      const int r0 = draw(seed, t, 0, ncorr), r1 = draw(seed, t, 1, ncorr), r2 = draw(seed, t, 2, ncorr);
      const float li0 = len(fi, corres[r0].first, corres[r1].first), li1 = len(fi, corres[r1].first, corres[r2].first),
                  li2 = len(fi, corres[r2].first, corres[r0].first);
      const float lj0 = len(fj, corres[r0].second, corres[r1].second), lj1 = len(fj, corres[r1].second, corres[r2].second),
                  lj2 = len(fj, corres[r2].second, corres[r0].second);
      if ((li0 * tuple_scale < lj0) && (lj0 < li0 / tuple_scale) && (li1 * tuple_scale < lj1) && (lj1 < li1 / tuple_scale) &&
          (li2 * tuple_scale < lj2) && (lj2 < li2 / tuple_scale)) {
        inc[r0] = inc[r1] = inc[r2] = 1;
      }
    }
    for (int r = 0; r < ncorr; r++)
      if (inc[r]) kept.push_back(corres[r]);
  } else {
    kept = corres;
  }
  std::vector<std::pair<int, int>> outp;
  for (auto& c : kept) outp.emplace_back(swapped ? c.second : c.first, swapped ? c.first : c.second);
  std::sort(outp.begin(), outp.end());
  outp.erase(std::unique(outp.begin(), outp.end()), outp.end());
  std::vector<Corr> out;
  for (auto& c : outp) out.push_back({c.first, c.second});
  return out;
}

// ---- TEASER++ solve in QUATRO / PMC_HEU mode (SURVEY App. B.7) ---------------------------------
struct SolveOut {
  double R[9], t[3];
  int valid;
  std::vector<int> clique;
  int gnc_iters;
};

static std::vector<int> greedy_max_clique(int n, const std::vector<std::vector<unsigned char>>& adj) {
  std::vector<int> deg(n, 0), core(n, 0), alive(n, 1);
  for (int i = 0; i < n; i++)
    for (int j = 0; j < n; j++) deg[i] += adj[i][j];
  std::vector<int> d(deg);
  int k = 0;
  for (int it = 0; it < n; it++) {  // peel the minimum-degree vertex (lowest index on ties)
    int v = -1;
    for (int i = 0; i < n; i++)
      if (alive[i] && (v < 0 || d[i] < d[v])) v = i;
    k = std::max(k, d[v]);
    core[v] = k;
    alive[v] = 0;
    for (int j = 0; j < n; j++)
      if (alive[j] && adj[v][j]) d[j]--;
  }
  std::vector<int> order(n);
  std::iota(order.begin(), order.end(), 0);
  std::sort(order.begin(), order.end(), [&](int a, int b) {
    if (core[a] != core[b]) return core[a] > core[b];
    if (deg[a] != deg[b]) return deg[a] > deg[b];
    return a < b;
  });
  std::vector<int> best;
  for (int oi = 0; oi < n; oi++) {
    const int v = order[oi];
    std::vector<unsigned char> P(adj[v]);
    std::vector<int> C{v};
    for (;;) {
      int u = -1;
      for (int oj = 0; oj < n; oj++)
        if (P[order[oj]]) {
          u = order[oj];
          break;
        }
      if (u < 0) break;
      C.push_back(u);
      for (int j = 0; j < n; j++) P[j] = P[j] && adj[u][j];
    }
    if (C.size() > best.size()) best = C;
  }
  std::sort(best.begin(), best.end());
  return best;
}

static void svd_rot2d(const std::vector<double>& X, const std::vector<double>& Y, const std::vector<double>& W, int n, double R2[4]) {
  // H = X W Y^T (2x2); R = V U^T with det correction
  double H[4] = {0, 0, 0, 0};
  for (int i = 0; i < n; i++) {
    H[0] += X[2 * i] * W[i] * Y[2 * i];
    H[1] += X[2 * i] * W[i] * Y[2 * i + 1];
    H[2] += X[2 * i + 1] * W[i] * Y[2 * i];
    H[3] += X[2 * i + 1] * W[i] * Y[2 * i + 1];
  }
  // closed-form 2x2 SVD via the polar angle: for H = U S V^T the optimal rotation V diag(1, det) U^T equals
  // the rotation by theta = atan2(H01 - H10, H00 + H11) whenever det(H) != 0 or the SVD is non-degenerate.
  const double th = std::atan2(H[1] - H[2], H[0] + H[3]);
  R2[0] = std::cos(th);
  R2[1] = -std::sin(th);
  R2[2] = std::sin(th);
  R2[3] = std::cos(th);
}

// TLS scalar estimator (adaptive voting), SURVEY App. B.7
static double tls_estimate(const std::vector<double>& X, double range) {
  const int N = (int)X.size();
  std::vector<std::pair<double, int>> h;
  h.reserve(2 * N);
  for (int i = 0; i < N; i++) {
    h.emplace_back(X[i] - range, i + 1);
    h.emplace_back(X[i] + range, -i - 1);
  }
  std::stable_sort(h.begin(), h.end(), [](const std::pair<double, int>& a, const std::pair<double, int>& b) { return a.first < b.first; });
  const double w = 1.0 / (range * range);
  double ranges_inverse_sum = range * N, dot_X_weights = 0, dot_weights_consensus = 0, sum_xi = 0, sum_xi_square = 0;
  int card = 0;
  double best_cost = std::numeric_limits<double>::infinity(), best = 0;
  for (int i = 0; i < 2 * N; i++) {
    const int idx = std::abs(h[i].second) - 1;
    const int eps = h[i].second > 0 ? 1 : -1;
    card += eps;
    dot_weights_consensus += eps * w;
    dot_X_weights += eps * w * X[idx];
    ranges_inverse_sum -= eps * range;
    sum_xi += eps * X[idx];
    sum_xi_square += eps * X[idx] * X[idx];
    const double x_hat = dot_X_weights / dot_weights_consensus;
    const double residual = card * x_hat * x_hat + sum_xi_square - 2 * sum_xi * x_hat;
    const double cost = residual + ranges_inverse_sum;
    if (cost < best_cost) {  // NaN (empty consensus set) never wins
      best_cost = cost;
      best = x_hat;
    }
  }
  return best;
}

static SolveOut teaser_quatro_solve(const float* src, int sstride, const float* dst, int dstride, const std::vector<Corr>& corr,
                                    double noise_bound, double cbar2, double gnc_factor, double cost_thr, int max_iter) {
  SolveOut o;
  for (int i = 0; i < 9; i++) o.R[i] = (i % 4 == 0) ? 1.0 : 0.0;
  o.t[0] = o.t[1] = o.t[2] = 0;
  o.valid = 0;
  o.gnc_iters = 0;
  const int n = (int)corr.size();
  if (n == 0) return o;
  std::vector<double> S(3 * (size_t)n), D(3 * (size_t)n);
  for (int i = 0; i < n; i++)
    for (int d = 0; d < 3; d++) {
      S[3 * i + d] = (double)src[(size_t)corr[i].s * sstride + d];
      D[3 * i + d] = (double)dst[(size_t)corr[i].d * dstride + d];
    }
  // TIM scale-consistency graph: | ||b_ij|| - ||a_ij|| | <= 2 * noise_bound * sqrt(cbar2)
  const double beta = 2.0 * noise_bound * std::sqrt(cbar2);
  std::vector<std::vector<unsigned char>> adj(n, std::vector<unsigned char>(n, 0));
  for (int i = 0; i < n; i++)
    for (int j = i + 1; j < n; j++) {
      double a = 0, b = 0;
      for (int d = 0; d < 3; d++) {
        const double da = S[3 * j + d] - S[3 * i + d], db = D[3 * j + d] - D[3 * i + d];
        a += da * da;
        b += db * db;
      }
      if (std::fabs(std::sqrt(a) - std::sqrt(b)) <= beta) adj[i][j] = adj[j][i] = 1;
    }
  o.clique = greedy_max_clique(n, adj);
  const int m = (int)o.clique.size();
  if (m <= 1) return o;
  // chain TIMs on the (sorted) clique
  const int nt = m - 1;
  std::vector<double> A(3 * (size_t)nt), B(3 * (size_t)nt), X(2 * (size_t)nt), Y(2 * (size_t)nt), W(nt, 1.0), res(nt);
  for (int k = 0; k < nt; k++)
    for (int d = 0; d < 3; d++) {
      A[3 * k + d] = S[3 * o.clique[k + 1] + d] - S[3 * o.clique[k] + d];
      B[3 * k + d] = D[3 * o.clique[k + 1] + d] - D[3 * o.clique[k] + d];
    }
  for (int k = 0; k < nt; k++) {
    X[2 * k] = A[3 * k]; X[2 * k + 1] = A[3 * k + 1];
    Y[2 * k] = B[3 * k]; Y[2 * k + 1] = B[3 * k + 1];
  }
  // GNC-TLS, yaw only
  double nb2 = noise_bound * noise_bound;
  if (nb2 < 1e-16) nb2 = 1e-2;
  double mu = 1, prev_cost = std::numeric_limits<double>::infinity();
  double R2[4] = {1, 0, 0, 1};
  for (int it = 0; it < max_iter; it++) {
    o.gnc_iters = it + 1;
    svd_rot2d(X, Y, W, nt, R2);
    double maxres = 0;
    for (int k = 0; k < nt; k++) {
      const double rx = B[3 * k] - (R2[0] * A[3 * k] + R2[1] * A[3 * k + 1]);
      const double ry = B[3 * k + 1] - (R2[2] * A[3 * k] + R2[3] * A[3 * k + 1]);
      const double rz = B[3 * k + 2] - A[3 * k + 2];
      res[k] = rx * rx + ry * ry + rz * rz;
      maxres = std::max(maxres, res[k]);
    }
    if (it == 0) {
      mu = 1.0 / (2.0 * maxres / nb2 - 1.0);
      if (mu <= 0) break;
    }
    const double th1 = (mu + 1) / mu * nb2, th2 = mu / (mu + 1) * nb2;
    double cost = 0;
    for (int k = 0; k < nt; k++) {
      cost += W[k] * res[k];
      if (res[k] >= th1) W[k] = 0;
      else if (res[k] <= th2) W[k] = 1;
      else W[k] = std::sqrt(nb2 * mu * (mu + 1) / res[k]) - mu;
    }
    const double cost_diff = std::fabs(cost - prev_cost);
    mu *= gnc_factor;
    prev_cost = cost;
    if (cost_diff < cost_thr) break;
  }
  o.R[0] = R2[0]; o.R[1] = R2[1]; o.R[3] = R2[2]; o.R[4] = R2[3];
  // translation: per-axis TLS over dst_i - R src_i on the clique members
  for (int d = 0; d < 3; d++) {
    std::vector<double> raw(m);
    for (int k = 0; k < m; k++) {
      const int c = o.clique[k];
      const double rs = o.R[3 * d] * S[3 * c] + o.R[3 * d + 1] * S[3 * c + 1] + o.R[3 * d + 2] * S[3 * c + 2];
      raw[k] = D[3 * c + d] - rs;
    }
    o.t[d] = tls_estimate(raw, noise_bound * std::sqrt(cbar2));
  }
  o.valid = 1;
  return o;
}

}  // namespace orq

using namespace orq;

extern "C" {

struct orc_quatro_params {
  double fpfh_normal_radius;  // QN/config/config.yaml quatro.fpfh_normal_radius (0.9)
  double fpfh_radius;         // (1.5)
  double noise_bound;         // (0.3)
  double rot_gnc_factor;      // (1.4)
  double rot_cost_thr;        // (1e-4)
  int rot_max_iter;           // (50)
  int max_corres;             // effective 200 (SURVEY §5: parameter-name typo)
  double distance_threshold;  // feature-space gate (35 in the deployment; class default 30)
  double tuple_scale;         // 0.95 (quatro_module.cc:61)
  uint64_t seed;              // replaces srand(time(NULL))
  int use_optimized_matching; // config.yaml:32 (true); 0 = Matcher::advancedMatching
  int pad_;
};

void orc_quatro_default_params(orc_quatro_params* p) {
  p->fpfh_normal_radius = 0.9;
  p->fpfh_radius = 1.5;
  p->noise_bound = 0.3;
  p->rot_gnc_factor = 1.4;
  p->rot_cost_thr = 1e-4;
  p->rot_max_iter = 50;
  p->max_corres = 200;
  p->distance_threshold = 35.0;
  p->tuple_scale = 0.95;
  p->seed = 1;
  p->use_optimized_matching = 1;
  p->pad_ = 0;
}

// normals (n x 3) and FPFH (n x 33) of one cloud
void orc_fpfh(const float* xyz, int n, int stride, double normal_radius, double fpfh_radius, float* normals_out, float* spfh_out,
              float* fpfh_out) {
  Grid g;
  g.build(xyz, n, stride, (float)std::max(normal_radius, fpfh_radius));
  std::vector<float> nrm((size_t)n * 3), sp((size_t)n * 33);
  normals(g, (float)normal_radius, nrm.data());
  spfh(g, nrm.data(), (float)fpfh_radius, sp.data());
  fpfh(g, sp.data(), nrm.data(), (float)fpfh_radius, fpfh_out);
  if (normals_out) std::memcpy(normals_out, nrm.data(), sizeof(float) * 3 * n);
  if (spfh_out) std::memcpy(spfh_out, sp.data(), sizeof(float) * 33 * n);
}

// SPFH / FPFH from GIVEN normals (stage isolation for the parity tests)
void orc_fpfh_from_normals(const float* xyz, int n, int stride, const float* nrm, double fpfh_radius, float* spfh_out, float* fpfh_out) {
  Grid g;
  g.build(xyz, n, stride, (float)fpfh_radius);
  std::vector<float> sp((size_t)n * 33);
  spfh(g, nrm, (float)fpfh_radius, sp.data());
  fpfh(g, sp.data(), nrm, (float)fpfh_radius, fpfh_out);
  if (spfh_out) std::memcpy(spfh_out, sp.data(), sizeof(float) * 33 * n);
}

// matching from GIVEN descriptors.  corr_out: up to max_corres+3 (src,dst) pairs; mutual_out: up to min(N,M) (i,j) pairs.
int orc_match(const float* src, int N, int sstride, const float* dst, int M, int dstride, const float* fsrc, const float* fdst,
              const orc_quatro_params* p, int* corr_out, int* n_mutual, int* mutual_out) {
  std::vector<Corr> mutual;
  std::vector<Corr> c = optimized_matching(src, N, sstride, dst, M, dstride, fsrc, fdst, (float)p->distance_threshold, p->max_corres,
                                           (float)p->tuple_scale, p->seed, &mutual);
  for (size_t i = 0; i < c.size(); i++) {
    corr_out[2 * i] = c[i].s;
    corr_out[2 * i + 1] = c[i].d;
  }
  if (n_mutual) *n_mutual = (int)mutual.size();
  if (mutual_out)
    for (size_t i = 0; i < mutual.size(); i++) {
      mutual_out[2 * i] = mutual[i].s;
      mutual_out[2 * i + 1] = mutual[i].d;
    }
  return (int)c.size();
}

// advancedMatching from GIVEN descriptors; corr_out must hold 2 * min(N, M) * 2 ints in the worst case (no cross check)
int orc_match_advanced(const float* src, int N, int sstride, const float* dst, int M, int dstride, const float* fsrc, const float* fdst,
                       const orc_quatro_params* p, int use_crosscheck, int use_tuple_test, int* corr_out, int cap) {
  std::vector<Corr> c = advanced_matching(src, N, sstride, dst, M, dstride, fsrc, fdst, use_crosscheck != 0, use_tuple_test != 0,
                                          (float)p->tuple_scale, p->seed);
  const int n = std::min((int)c.size(), cap);
  for (int i = 0; i < n; i++) {
    corr_out[2 * i] = c[i].s;
    corr_out[2 * i + 1] = c[i].d;
  }
  return (int)c.size();
}

// TEASER++ QUATRO solve from GIVEN correspondences.  T16 row-major.  Returns valid.
int orc_quatro_solve(const float* src, int sstride, const float* dst, int dstride, const int* corr, int ncorr,
                     const orc_quatro_params* p, double* T16, int* clique_out, int* clique_size, int* gnc_iters) {
  std::vector<Corr> c(ncorr);
  for (int i = 0; i < ncorr; i++) c[i] = {corr[2 * i], corr[2 * i + 1]};
  SolveOut o = teaser_quatro_solve(src, sstride, dst, dstride, c, p->noise_bound, 1.0, p->rot_gnc_factor, p->rot_cost_thr, p->rot_max_iter);
  for (int i = 0; i < 16; i++) T16[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int r = 0; r < 3; r++) {
    for (int cc = 0; cc < 3; cc++) T16[4 * r + cc] = o.R[3 * r + cc];
    T16[4 * r + 3] = o.t[r];
  }
  if (clique_size) *clique_size = (int)o.clique.size();
  if (clique_out)
    for (size_t i = 0; i < o.clique.size(); i++) clique_out[i] = o.clique[i];
  if (gnc_iters) *gnc_iters = o.gnc_iters;
  return o.valid;
}

// quatro<T>::align (quatro_module.cc:48-79).  Returns if_valid; T16 = Identity when invalid.
int orc_quatro_align(const float* src, int N, int sstride, const float* dst, int M, int dstride, const orc_quatro_params* p,
                     double* T16, int* n_corr_out, double* ms_fpfh, double* ms_match, double* ms_solve) {
  auto now = [] { return omp_get_wtime() * 1e3; };
  const double t0 = now();
  std::vector<float> fs((size_t)N * 33), fd((size_t)M * 33);
  orc_fpfh(src, N, sstride, p->fpfh_normal_radius, p->fpfh_radius, nullptr, nullptr, fs.data());
  orc_fpfh(dst, M, dstride, p->fpfh_normal_radius, p->fpfh_radius, nullptr, nullptr, fd.data());
  const double t1 = now();
  std::vector<int> corr(2 * (size_t)(p->use_optimized_matching ? p->max_corres + 8 : std::min(N, M)));
  const int nc = p->use_optimized_matching
                     ? orc_match(src, N, sstride, dst, M, dstride, fs.data(), fd.data(), p, corr.data(), nullptr, nullptr)
                     : orc_match_advanced(src, N, sstride, dst, M, dstride, fs.data(), fd.data(), p, 1, 1, corr.data(), std::min(N, M));
  const double t2 = now();
  for (int i = 0; i < 16; i++) T16[i] = (i % 5 == 0) ? 1.0 : 0.0;
  int valid = 0;
  if (nc > 0) valid = orc_quatro_solve(src, sstride, dst, dstride, corr.data(), nc, p, T16, nullptr, nullptr, nullptr);
  const double t3 = now();
  if (n_corr_out) *n_corr_out = nc;
  if (ms_fpfh) *ms_fpfh = t1 - t0;
  if (ms_match) *ms_match = t2 - t1;
  if (ms_solve) *ms_solve = t3 - t2;
  return valid;
}

}  // extern "C"
