// oracle/oracle_gicp.cpp -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// CPU restatement of the Nano-GICP half of the loop-closure hot path, written
// from the reference's behaviour (NOT copied).  Every function cites the
// reference lines it follows; paths are relative to the reference tree's root.
//   NG  = third_party/nano_gicp/include/nano_gicp
//   QN  = fast_lio_sam_qn
//
// Pinning status: the reference ships no tests / golden vectors (SURVEY.md §4),
// and PCL/Eigen are absent so the reference itself cannot be run here.  The one
// piece of the reference that DOES compile here is its kd-tree
// (NG/impl/nanoflann_impl.hpp): oracle/ref_nanoflann_shim.cpp wraps it into
// oracle/_ref/libref_nanoflann.so and tests/test_oracle.py pins this
// file's kNN against it index-for-index.  Everything after the kNN (covariance,
// Mahalanobis, LM) is "parity unpinned" by reference outputs and is instead
// pinned by (i) closed-form known-answer tests and (ii) ground-truth SE(3)
// recovery on synthetic pairs.
//
// Build: see oracle/Makefile (g++ -O3 -fopenmp -ffp-contract=off, no -march, as
// third_party/nano_gicp/CMakeLists.txt:14,24).
#include <dlfcn.h>
#include <omp.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <numeric>
#include <vector>

#include "linalg.hpp"

namespace orc {

// ---------------------------------------------------------------------------
// fp32 squared distance exactly as nanoflann's L2_Simple_Adaptor::evalMetric
// (NG/impl/nanoflann_impl.hpp:441-449): result=0; for x,y,z: diff=a-b; result+=diff*diff.
// -ffp-contract=off keeps it FMA-free like the reference build.
static inline float dist2_f32(const float* a, const float* b) {
  float r = 0.0f;
  for (int i = 0; i < 3; i++) {
    const float diff = a[i] - b[i];
    r += diff * diff;
  }
  return r;
}

// Deterministic tie rule (SURVEY.md App. A.3): (d2, lower index).  The
// reference keeps the first-visited point on exact-equal d2, which depends on
// its tree layout and cannot be reproduced by any other index structure.
static inline bool better(float d2a, int ia, float d2b, int ib) { return d2a < d2b || (d2a == d2b && ia < ib); }

struct KnnHeap {  // ascending insertion list, like KNNResultSet (nanoflann_impl.hpp:151-214)
  int k, count;
  int* idx;
  float* d2;
  void init(int k_, int* i_, float* d_) {
    k = k_;
    count = 0;
    idx = i_;
    d2 = d_;
    for (int j = 0; j < k; j++) {
      idx[j] = -1;
      d2[j] = std::numeric_limits<float>::max();
    }
  }
  inline float worst() const { return d2[k - 1]; }
  inline int worst_idx() const { return count == k ? idx[k - 1] : std::numeric_limits<int>::max(); }
  inline void add(float d, int i) {
    if (count == k && !better(d, i, d2[k - 1], idx[k - 1])) return;
    int j = count < k ? count : k - 1;
    while (j > 0 && better(d, i, d2[j - 1], idx[j - 1])) {
      d2[j] = d2[j - 1];
      idx[j] = idx[j - 1];
      j--;
    }
    d2[j] = d;
    idx[j] = i;
    if (count < k) count++;
  }
};

// ---------------------------------------------------------------------------
// Own exact kd-tree (median split, leaf <= 24) -- the oracle's default kNN
// backend; exactness pinned against the reference's nanoflann in tests.
struct KdTree {
  struct Node {
    int left, right;  // children (internal) or point range [left,right) (leaf)
    int dim;          // -1 => leaf
    float split;
  };
  std::vector<Node> nodes;
  std::vector<int> perm;
  std::vector<float> pts;  // permuted xyz copy (n x 3) for locality
  int n = 0;

  int build_rec(const float* xyz, int stride, int lo, int hi) {
    int id = (int)nodes.size();
    nodes.push_back(Node());
    if (hi - lo <= 24) {
      nodes[id] = {lo, hi, -1, 0.f};
      return id;
    }
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = lo; i < hi; i++)
      for (int d = 0; d < 3; d++) {
        float v = xyz[(size_t)perm[i] * stride + d];
        mn[d] = std::min(mn[d], v);
        mx[d] = std::max(mx[d], v);
      }
    int dim = 0;
    for (int d = 1; d < 3; d++)
      if (mx[d] - mn[d] > mx[dim] - mn[dim]) dim = d;
    int mid = (lo + hi) / 2;
    std::nth_element(perm.begin() + lo, perm.begin() + mid, perm.begin() + hi, [&](int a, int b) {
      float va = xyz[(size_t)a * stride + dim], vb = xyz[(size_t)b * stride + dim];
      return va < vb || (va == vb && a < b);
    });
    float split = xyz[(size_t)perm[mid] * stride + dim];
    int l = build_rec(xyz, stride, lo, mid);
    int r = build_rec(xyz, stride, mid, hi);
    nodes[id] = {l, r, dim, split};
    return id;
  }
  void build(const float* xyz, int n_, int stride) {
    n = n_;
    perm.resize(n);
    std::iota(perm.begin(), perm.end(), 0);
    nodes.clear();
    nodes.reserve(n / 8 + 16);
    if (n > 0) build_rec(xyz, stride, 0, n);
    pts.resize((size_t)n * 3);
    for (int i = 0; i < n; i++)
      for (int d = 0; d < 3; d++) pts[(size_t)i * 3 + d] = xyz[(size_t)perm[i] * stride + d];
  }
  void search(int node, const float* q, KnnHeap& h) const {
    const Node& nd = nodes[node];
    if (nd.dim < 0) {
      for (int i = nd.left; i < nd.right; i++) h.add(dist2_f32(q, &pts[(size_t)i * 3]), perm[i]);
      return;
    }
    // left subtree holds values <= split, right subtree values >= split
    float diff = q[nd.dim] - nd.split;
    int near = diff < 0 ? nd.left : nd.right, far = diff < 0 ? nd.right : nd.left;
    search(near, q, h);
    // fl(diff*diff) is a lower bound of the fp32 distance to any far-side point
    // (rounding is monotonic); strict '>' so equal-distance candidates are still seen.
    float bound = diff * diff;
    if (!(bound > h.worst())) search(far, q, h);
  }
  void knn(const float* q, int k, int* idx, float* d2) const {
    KnnHeap h;
    h.init(k, idx, d2);
    if (n > 0) search(0, q, h);
  }
};

// ---------------------------------------------------------------------------
// kNN backend switch: own kd-tree (default) or the reference's nanoflann via
// oracle/_ref/libref_nanoflann.so (used for the timed CPU baseline so the tree
// cost is the reference's own).
typedef void* (*ref_build_fn)(const float*, int, int);
typedef void (*ref_free_fn)(void*);
typedef void (*ref_knn1_fn)(void*, const float*, int, int*, float*);
static struct {
  void* lib = nullptr;
  ref_build_fn build = nullptr;
  ref_free_fn free_ = nullptr;
  ref_knn1_fn knn1 = nullptr;
} g_ref;

struct Index {
  KdTree own;
  void* ref = nullptr;
  bool use_ref = false;
  ~Index() {
    if (ref && g_ref.free_) g_ref.free_(ref);
  }
  void build(const float* xyz, int n, int stride) {
    if (g_ref.lib) {
      use_ref = true;
      ref = g_ref.build(xyz, n, stride);
    } else {
      own.build(xyz, n, stride);
    }
  }
  inline void knn(const float* q, int k, int* idx, float* d2) const {
    if (use_ref)
      g_ref.knn1(ref, q, k, idx, d2);
    else
      own.knn(q, k, idx, d2);
  }
};

static double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// ---------------------------------------------------------------------------
// NanoGICP::calculate_covariances, NG/impl/nano_gicp_impl.hpp:298-357 (PLANE):
// k-NN (self included) -> mean-subtracted 3xk -> cov = X X^T / k -> SVD ->
// U diag(1,1,1e-3) V^T.  Row/col 3 of the reference's 4x4 is identically zero
// (SURVEY App. A.2) so only the 3x3 block is produced.
static void covariances(const float* xyz, int n, int stride, const Index& index, int k, double* cov9, int* knn_idx_out, int method = 3) {
#pragma omp parallel for schedule(guided, 8)
  for (int i = 0; i < n; i++) {
    std::vector<int> idx(k);
    std::vector<float> d2(k);
    index.knn(&xyz[(size_t)i * stride], k, idx.data(), d2.data());
    if (knn_idx_out) std::memcpy(&knn_idx_out[(size_t)i * k], idx.data(), sizeof(int) * k);
    double mean[3] = {0, 0, 0};
    std::vector<double> X(3 * (size_t)k);
    int kk = 0;
    for (int j = 0; j < k; j++) {
      if (idx[j] < 0) continue;  // k > n: reference behaviour undefined (SURVEY A.3); use what exists
      for (int d = 0; d < 3; d++) {
        X[3 * kk + d] = (double)xyz[(size_t)idx[j] * stride + d];
        mean[d] += X[3 * kk + d];
      }
      kk++;
    }
    for (int d = 0; d < 3; d++) mean[d] /= k;  // rowwise().mean() over k columns (:320)
    M3 cov = m3_zero();
    for (int j = 0; j < kk; j++) {
      double v[3] = {X[3 * j] - mean[0], X[3 * j + 1] - mean[1], X[3 * j + 2] - mean[2]};
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) cov(a, b) += v[a] * v[b];
    }
    for (int a = 0; a < 9; a++) cov.m[a] /= k;  // (:321)
    // RegularizationMethod (gicp/gicp_settings.hpp:47): 0 NONE, 1 MIN_EIG, 2 NORMALIZED_MIN_EIG, 3 PLANE, 4 FROBENIUS
    M3 C = m3_zero();
    if (method == 0) {  // NONE (:323-324)
      C = cov;
    } else if (method == 4) {  // FROBENIUS (:325-330): ((C+1e-3 I)^-1 / ||.||_F)^-1
      M3 Cl = cov;
      for (int a = 0; a < 3; a++) Cl(a, a) += 1e-3;
      M3 Ci = m3_inverse(Cl);
      double nrm = 0;
      for (int a = 0; a < 9; a++) nrm += Ci.m[a] * Ci.m[a];
      nrm = std::sqrt(nrm);
      M3 Cn;
      for (int a = 0; a < 9; a++) Cn.m[a] = Ci.m[a] / nrm;
      C = m3_inverse(Cn);
    } else {
      M3 U, V;
      double s[3];
      m3_svd(cov, U, s, V);
      double vals[3] = {1.0, 1.0, 1e-3};  // PLANE (:341-343)
      if (method == 1) {                  // MIN_EIG (:344-346)
        for (int a = 0; a < 3; a++) vals[a] = std::max(s[a], 1e-3);
      } else if (method == 2) {           // NORMALIZED_MIN_EIG (:347-350)
        const double mx = std::max(s[0], std::max(s[1], s[2]));
        for (int a = 0; a < 3; a++) vals[a] = std::max(s[a] / mx, 1e-3);
      }
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) {
          double acc = 0;
          for (int c = 0; c < 3; c++) acc += U(a, c) * vals[c] * V(b, c);
          C(a, b) = acc;
        }
    }
    std::memcpy(&cov9[(size_t)i * 9], C.m, sizeof(double) * 9);
  }
}

// trans.cast<float>() then `trans_f * p.getVector4fMap()` (nano_gicp_impl.hpp:178,190).
// Summation order fixed as ((r0*x + r1*y) + r2*z) + t, no FMA (SURVEY App. A.4).
static inline void transform_query_f32(const float Tf[12], const float* p, float* q) {
  for (int r = 0; r < 3; r++) q[r] = ((Tf[4 * r + 0] * p[0] + Tf[4 * r + 1] * p[1]) + Tf[4 * r + 2] * p[2]) + Tf[4 * r + 3];
}
// pcl::transformPointCloud<PointT,float> (PCL 1.10 detail::Transformer::se3, SSE2):
// x*c0 + (y*c1 + (z*c2 + c3)); used for the output cloud (lsq_registration_impl.hpp:114)
// and inside Registration::getFitnessScore (SURVEY App. A.7 / B.3).
static inline void transform_output_f32(const float Tf[12], const float* p, float* q) {
  for (int r = 0; r < 3; r++) q[r] = Tf[4 * r + 0] * p[0] + (Tf[4 * r + 1] * p[1] + (Tf[4 * r + 2] * p[2] + Tf[4 * r + 3]));
}
static inline void iso_to_f32(const Iso& x, float Tf[12]) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) Tf[4 * r + c] = (float)x.R(r, c);
    Tf[4 * r + 3] = (float)x.t[r];
  }
}

struct GicpProblem {
  const float* src;
  int N, sstride;
  const float* tgt;
  int M, tstride;
  const Index* tgt_index;
  const double* cov_src;  // N*9
  const double* cov_tgt;  // M*9
  double max_corr_dist;
  std::vector<int> corr;
  std::vector<float> sqd;
  std::vector<double> mahal;  // N*9
};

// NanoGICP::update_correspondences, nano_gicp_impl.hpp:173-211
static void update_correspondences(GicpProblem& P, const Iso& x) {
  float Tf[12];
  iso_to_f32(x, Tf);
  P.corr.resize(P.N);
  P.sqd.resize(P.N);
  P.mahal.resize((size_t)P.N * 9);
  const float thr = (float)P.max_corr_dist;  // corr_dist_threshold_ is a double in pcl::Registration;
  const double thr2 = P.max_corr_dist * P.max_corr_dist;  // compare promotes the float d2 to double (:195)
  (void)thr;
#pragma omp parallel for schedule(guided, 8)
  for (int i = 0; i < P.N; i++) {
    float q[3];
    transform_query_f32(Tf, &P.src[(size_t)i * P.sstride], q);
    int idx;
    float d2;
    P.tgt_index->knn(q, 1, &idx, &d2);
    P.sqd[i] = d2;
    P.corr[i] = ((double)d2 < thr2) ? idx : -1;
    if (P.corr[i] < 0) continue;
    M3 CA, CB;
    std::memcpy(CA.m, &P.cov_src[(size_t)i * 9], 72);
    std::memcpy(CB.m, &P.cov_tgt[(size_t)P.corr[i] * 9], 72);
    M3 RCR = m3_add(CB, m3_mul(m3_mul(x.R, CA), m3_transpose(x.R)));  // (:205)
    M3 Minv = m3_inverse(RCR);                                         // (:208), 4x4 is block diagonal
    std::memcpy(&P.mahal[(size_t)i * 9], Minv.m, 72);
  }
}

// NanoGICP::linearize, nano_gicp_impl.hpp:213-270.  Per-thread partial sums then a
// serial sum over threads, like the reference (:218-223, 256-266).
static double linearize(GicpProblem& P, const Iso& x, double* H36, double* b6) {
  update_correspondences(P, x);
  const int nt = omp_get_max_threads();
  std::vector<double> Hs((size_t)nt * 36, 0.0), bs((size_t)nt * 6, 0.0);
  double sum_errors = 0.0;
#pragma omp parallel for reduction(+ : sum_errors) schedule(guided, 8)
  for (int i = 0; i < P.N; i++) {
    int ti = P.corr[i];
    if (ti < 0) continue;
    double a[3], bpt[3], ta[3], e[3];
    for (int d = 0; d < 3; d++) {
      a[d] = (double)P.src[(size_t)i * P.sstride + d];
      bpt[d] = (double)P.tgt[(size_t)ti * P.tstride + d];
    }
    m3_vec(x.R, a, ta);
    for (int d = 0; d < 3; d++) {
      ta[d] += x.t[d];
      e[d] = bpt[d] - ta[d];
    }
    const double* Mm = &P.mahal[(size_t)i * 9];
    double Me[3];
    for (int r = 0; r < 3; r++) Me[r] = Mm[3 * r] * e[0] + Mm[3 * r + 1] * e[1] + Mm[3 * r + 2] * e[2];
    sum_errors += e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2];
    if (!H36 || !b6) continue;
    // J = [skew(T*a) | -I]  (3x6)   (:245-247)
    double J[3][6] = {{0, -ta[2], ta[1], -1, 0, 0}, {ta[2], 0, -ta[0], 0, -1, 0}, {-ta[1], ta[0], 0, 0, 0, -1}};
    double MJ[3][6];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 6; c++) MJ[r][c] = Mm[3 * r] * J[0][c] + Mm[3 * r + 1] * J[1][c] + Mm[3 * r + 2] * J[2][c];
    double* Ht = &Hs[(size_t)omp_get_thread_num() * 36];
    double* bt = &bs[(size_t)omp_get_thread_num() * 6];
    for (int r = 0; r < 6; r++) {
      for (int c = 0; c < 6; c++) Ht[6 * r + c] += J[0][r] * MJ[0][c] + J[1][r] * MJ[1][c] + J[2][r] * MJ[2][c];
      bt[r] += J[0][r] * Me[0] + J[1][r] * Me[1] + J[2][r] * Me[2];
    }
  }
  if (H36 && b6) {
    std::fill(H36, H36 + 36, 0.0);
    std::fill(b6, b6 + 6, 0.0);
    for (int t = 0; t < nt; t++) {
      for (int j = 0; j < 36; j++) H36[j] += Hs[(size_t)t * 36 + j];
      for (int j = 0; j < 6; j++) b6[j] += bs[(size_t)t * 6 + j];
    }
  }
  return sum_errors;
}

// NanoGICP::compute_error, nano_gicp_impl.hpp:272-296 (stale correspondences + Mahalanobis)
static double compute_error(const GicpProblem& P, const Iso& x) {
  double sum_errors = 0.0;
#pragma omp parallel for reduction(+ : sum_errors) schedule(guided, 8)
  for (int i = 0; i < P.N; i++) {
    int ti = P.corr[i];
    if (ti < 0) continue;
    double a[3], ta[3], e[3];
    for (int d = 0; d < 3; d++) a[d] = (double)P.src[(size_t)i * P.sstride + d];
    m3_vec(x.R, a, ta);
    for (int d = 0; d < 3; d++) e[d] = (double)P.tgt[(size_t)ti * P.tstride + d] - (ta[d] + x.t[d]);
    const double* Mm = &P.mahal[(size_t)i * 9];
    double Me[3];
    for (int r = 0; r < 3; r++) Me[r] = Mm[3 * r] * e[0] + Mm[3 * r + 1] * e[1] + Mm[3 * r + 2] * e[2];
    sum_errors += e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2];
  }
  return sum_errors;
}

// LsqRegistration::is_converged, NG/impl/lsq_registration_impl.hpp:117-127: (1.0 / eps) * |x| as written there (:123-124),
// and a NaN anywhere in delta is not converged (the maxCoeff of an all-NaN block is NaN, and NaN < 1 is false)
static bool is_converged(const Iso& delta, double rot_eps, double trans_eps) {
  double m = 0;
  bool nan = false;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      const double v = 1.0 / rot_eps * std::fabs(delta.R(i, j) - (i == j ? 1.0 : 0.0));
      nan = nan || std::isnan(v);
      m = std::max(m, v);
    }
    const double v = 1.0 / trans_eps * std::fabs(delta.t[i]);
    nan = nan || std::isnan(v);
    m = std::max(m, v);
  }
  return !nan && m < 1;
}

}  // namespace orc

using namespace orc;

extern "C" {

struct orc_gicp_params {
  int k_correspondences;       // QN/config/config.yaml:22 -> 15
  int max_iterations;          // config.yaml:23 -> 32 (QN/src/loop_closure.cpp:11)
  double max_corr_dist;        // QN/src/fast_lio_sam_qn.cpp:24 -> 52.5
  double transformation_eps;   // config.yaml:24 -> 0.01 (loop_closure.cpp:14)
  double rotation_eps;         // lsq_registration_impl.hpp:53 -> 2e-3
  int lm_max_iterations;       // lsq_registration_impl.hpp:58 -> 10
  double lm_init_lambda_factor;  // lsq_registration_impl.hpp:59 -> 1e-9
  int regularization;          // RegularizationMethod of both clouds' covariances: 0 NONE .. 4 FROBENIUS (3 PLANE)
};

struct orc_gicp_result {
  double T[16];  // row-major final_transformation_ (x0, fp64)
  float Tf[16];  // x0.cast<float>() -- what getFinalTransformation() returns
  double fitness;
  int converged;
  int iterations;  // nr_iterations_ (index of last outer iteration)
  int n_linearize;
  int n_error;
  int lm_failed;
  int pad;
  double ms_build, ms_cov, ms_align, ms_fitness;
};

int orc_num_threads() { return omp_get_max_threads(); }
void orc_set_num_threads(int n) {
  if (n > 0) omp_set_num_threads(n);
}

int orc_use_ref_nanoflann(const char* so_path) {
  if (!so_path) {
    g_ref.lib = nullptr;
    return 0;
  }
  void* lib = dlopen(so_path, RTLD_NOW | RTLD_LOCAL);
  if (!lib) return -1;
  g_ref.build = (ref_build_fn)dlsym(lib, "ref_nf_build");
  g_ref.free_ = (ref_free_fn)dlsym(lib, "ref_nf_free");
  g_ref.knn1 = (ref_knn1_fn)dlsym(lib, "ref_nf_knn_one");
  if (!g_ref.build || !g_ref.free_ || !g_ref.knn1) return -2;
  g_ref.lib = lib;
  return 0;
}

void orc_knn(const float* pts, int n, int stride, const float* q, int nq, int qstride, int k, int* idx, float* d2) {
  Index index;
  index.build(pts, n, stride);
#pragma omp parallel for schedule(guided, 8)
  for (int i = 0; i < nq; i++) index.knn(&q[(size_t)i * qstride], k, &idx[(size_t)i * k], &d2[(size_t)i * k]);
}

void orc_knn_bruteforce(const float* pts, int n, int stride, const float* q, int nq, int qstride, int k, int* idx, float* d2) {
#pragma omp parallel for schedule(static)
  for (int i = 0; i < nq; i++) {
    KnnHeap h;
    h.init(k, &idx[(size_t)i * k], &d2[(size_t)i * k]);
    for (int j = 0; j < n; j++) h.add(dist2_f32(&q[(size_t)i * qstride], &pts[(size_t)j * stride]), j);
  }
}

void orc_covariances(const float* xyz, int n, int stride, int k, double* cov9, int* knn_idx_out) {
  Index index;
  index.build(xyz, n, stride);
  covariances(xyz, n, stride, index, k, cov9, knn_idx_out);
}

void orc_covariances_ex(const float* xyz, int n, int stride, int k, int method, double* cov9) {
  Index index;
  index.build(xyz, n, stride);
  covariances(xyz, n, stride, index, k, cov9, nullptr, method);
}

void orc_transform_queries(const double* T16, const float* xyz, int n, int stride, float* out3) {
  Iso x = iso_from_rowmajor16(T16);
  float Tf[12];
  iso_to_f32(x, Tf);
  for (int i = 0; i < n; i++) transform_query_f32(Tf, &xyz[(size_t)i * stride], &out3[(size_t)i * 3]);
}

void orc_transform_output(const float* Tf16, const float* xyz, int n, int stride, float* out3) {
  for (int i = 0; i < n; i++) transform_output_f32(Tf16, &xyz[(size_t)i * stride], &out3[(size_t)i * 3]);
}

// One linearization at pose T16 (debug tap mirroring NanoGICP::linearize).
double orc_linearize(const float* src, int N, int sstride, const float* tgt, int M, int tstride, const double* cov_src,
                     const double* cov_tgt, const double* T16, double max_corr_dist, double* H36, double* b6, int* corr_out,
                     float* sqd_out, double* mahal_out) {
  Index index;
  index.build(tgt, M, tstride);
  GicpProblem P{src, N, sstride, tgt, M, tstride, &index, cov_src, cov_tgt, max_corr_dist, {}, {}, {}};
  Iso x = iso_from_rowmajor16(T16);
  double y = linearize(P, x, H36, b6);
  if (corr_out) std::memcpy(corr_out, P.corr.data(), sizeof(int) * N);
  if (sqd_out) std::memcpy(sqd_out, P.sqd.data(), sizeof(float) * N);
  if (mahal_out) std::memcpy(mahal_out, P.mahal.data(), sizeof(double) * 9 * N);
  return y;
}

// NanoGICP::compute_error in isolation (nano_gicp_impl.hpp:272-296): correspondences and Mahalanobis matrices from one
// update_correspondences at T_lin (stale, as inside step_lm), sum of e^T M e at T_trial.
double orc_compute_error(const float* src, int N, int sstride, const float* tgt, int M, int tstride, const double* cov_src,
                         const double* cov_tgt, const double* T_lin16, const double* T_trial16, double max_corr_dist) {
  Index index;
  index.build(tgt, M, tstride);
  GicpProblem P{src, N, sstride, tgt, M, tstride, &index, cov_src, cov_tgt, max_corr_dist, {}, {}, {}};
  update_correspondences(P, iso_from_rowmajor16(T_lin16));
  return compute_error(P, iso_from_rowmajor16(T_trial16));
}

// LoopClosure::icpAlignment (QN/src/loop_closure.cpp:110-136) = setInputSource +
// calculateSourceCovariances + setInputTarget + calculateTargetCovariances +
// align (pcl::Registration::align -> LsqRegistration::computeTransformation,
// lsq_registration_impl.hpp:88-115, step_lm :160-208) + getFitnessScore.
// trace (optional): per outer iteration 64 doubles:
//   [0..15] pose at linearization (row-major), [16..51] H, [52..57] b, [58] y0,
//   [59] lambda after the step, [60] trials used, [61] accepted(1)/early-converged(2)/failed(0)
int orc_gicp_align(const float* src, int N, int sstride, const float* tgt, int M, int tstride, const orc_gicp_params* prm,
                   const double* guess16, orc_gicp_result* out, float* aligned_out3, double* trace, int trace_cap) {
  if (N <= 0 || M <= 0) return -1;
  double t0 = now_ms();
  Index sidx, tidx;
  sidx.build(src, N, sstride);  // setInputSource -> buildIndex (nano_gicp_impl.hpp:120-129)
  double t1 = now_ms();
  std::vector<double> cov_src((size_t)N * 9), cov_tgt((size_t)M * 9);
  covariances(src, N, sstride, sidx, prm->k_correspondences, cov_src.data(), nullptr, prm->regularization);
  double t2 = now_ms();
  tidx.build(tgt, M, tstride);
  double t3 = now_ms();
  covariances(tgt, M, tstride, tidx, prm->k_correspondences, cov_tgt.data(), nullptr, prm->regularization);
  double t4 = now_ms();
  // pcl::Registration::align builds PCL's own FLANN tree on the target as well
  // (SURVEY §3.4 "hidden 3rd tree build"); charged to the CPU baseline as one more build.
  {
    Index hidden;
    hidden.build(tgt, M, tstride);
  }
  double t4b = now_ms();

  GicpProblem P{src, N, sstride, tgt, M, tstride, &tidx, cov_src.data(), cov_tgt.data(), prm->max_corr_dist, {}, {}, {}};
  Iso x0 = guess16 ? iso_from_rowmajor16(guess16) : iso_identity();
  double lm_lambda = -1.0;  // lsq_registration_impl.hpp:92
  bool converged = false;
  int nr_iterations = 0, n_lin = 0, n_err = 0, lm_failed = 0;
  for (int it = 0; it < prm->max_iterations && !converged; it++) {
    nr_iterations = it;
    // ---- step_lm (:160-208)
    double H[36], b[6];
    Iso xlin = x0;
    double y0 = linearize(P, x0, H, b);
    n_lin++;
    if (lm_lambda < 0.0) {  // maxCoeff of |diag H|; a NaN there makes lambda NaN
      double mx = 0;
      bool nan = false;
      for (int d = 0; d < 6; d++) {
        nan = nan || std::isnan(H[7 * d]);
        mx = std::max(mx, std::fabs(H[7 * d]));
      }
      lm_lambda = prm->lm_init_lambda_factor * (nan ? std::nan("") : mx);
    }
    double nu = 2.0;
    Iso delta = iso_identity();
    int outcome = 0, trials = 0;
    for (int j = 0; j < prm->lm_max_iterations; j++) {
      trials = j + 1;
      double A[36], nb[6], d[6];
      std::memcpy(A, H, sizeof(A));
      for (int q = 0; q < 6; q++) {
        A[7 * q] += lm_lambda;
        nb[q] = -b[q];
      }
      ldlt6_solve(A, nb, d);
      delta.R = so3_exp_matrix(d);
      delta.t[0] = d[3];
      delta.t[1] = d[4];
      delta.t[2] = d[5];
      Iso xi = iso_mul(delta, x0);
      double yi = compute_error(P, xi);
      n_err++;
      double denom = 0;
      for (int q = 0; q < 6; q++) denom += d[q] * (lm_lambda * d[q] - b[q]);
      double rho = (y0 - yi) / denom;
      if (rho < 0) {
        if (is_converged(delta, prm->rotation_eps, prm->transformation_eps)) {
          outcome = 2;  // returns true WITHOUT updating x0 (:191-194)
          break;
        }
        lm_lambda = nu * lm_lambda;
        nu = 2 * nu;
        continue;
      }
      x0 = xi;
      lm_lambda = lm_lambda * std::max(1.0 / 3.0, 1 - std::pow(2 * rho - 1, 3));
      outcome = 1;
      break;
    }
    if (trace && it < trace_cap) {
      double* tr = &trace[(size_t)it * 64];
      std::fill(tr, tr + 64, 0.0);
      iso_to_rowmajor16(xlin, tr);
      std::memcpy(tr + 16, H, sizeof(H));
      std::memcpy(tr + 52, b, sizeof(b));
      tr[58] = y0;
      tr[59] = lm_lambda;
      tr[60] = trials;
      tr[61] = outcome;
    }
    if (outcome == 0) {  // "lm not converged!!" (:105-108)
      lm_failed = 1;
      break;
    }
    converged = is_converged(delta, prm->rotation_eps, prm->transformation_eps);
  }
  double t5 = now_ms();

  iso_to_rowmajor16(x0, out->T);
  for (int i = 0; i < 16; i++) out->Tf[i] = (float)out->T[i];
  // getFitnessScore (QN/src/loop_closure.cpp:127; SURVEY App. A.7): transform source by the
  // fp32 final transformation, serial 1-NN, mean of d2 over all N (no range cap).
  double fit = 0.0;
  {
    std::vector<float> d2s(N);
#pragma omp parallel for schedule(guided, 8)
    for (int i = 0; i < N; i++) {
      float q[3];
      transform_output_f32(out->Tf, &src[(size_t)i * sstride], q);
      if (aligned_out3) std::memcpy(&aligned_out3[(size_t)i * 3], q, 12);
      int idx;
      float d2;
      tidx.knn(q, 1, &idx, &d2);
      d2s[i] = d2;
    }
    for (int i = 0; i < N; i++) fit += (double)d2s[i];  // serial, source order
    fit /= N;
  }
  double t6 = now_ms();
  out->fitness = fit;
  out->converged = converged ? 1 : 0;
  out->iterations = nr_iterations;
  out->n_linearize = n_lin;
  out->n_error = n_err;
  out->lm_failed = lm_failed;
  out->pad = 0;
  out->ms_build = (t1 - t0) + (t3 - t2) + (t4b - t4);
  out->ms_cov = (t2 - t1) + (t4 - t3);
  out->ms_align = t5 - t4b;
  out->ms_fitness = t6 - t5;
  return 0;
}

}  // extern "C"

// ===========================================================================================
// "Next" rows of SURVEY.md §8(f): the steps either side of the registration path.
// ===========================================================================================
extern "C" {

// PosePcd::PosePcd (fast_lio_sam_qn/include/pose_pcd.hpp:21-43): pose_eig_ from the odometry quaternion (tf::Matrix3x3(q),
// restated from tf/LinearMath/Matrix3x3.h setRotation) and position; the world-frame scan goes into the LiDAR frame with
// pose_eig_.inverse() -- here by Gauss-Jordan elimination with partial pivoting (deliberately NOT the product's cofactor
// formula).  pose16_out: row-major pose_eig_ (= pose_corrected_eig_).
void orc_transform_pcd(const float* in, int n, int stride, const double* T16, float* out);
void orc_pose_pcd_ingest(const float* world, int n, int stride, const double* pos3, const double* quat_xyzw, float* out, double* pose16_out) {
  const double x = quat_xyzw[0], y = quat_xyzw[1], z = quat_xyzw[2], w = quat_xyzw[3];
  const double d = x * x + y * y + z * z + w * w, s = 2.0 / d;
  const double xs = x * s, ys = y * s, zs = z * s, wx = w * xs, wy = w * ys, wz = w * zs;
  const double xx = x * xs, xy = x * ys, xz = x * zs, yy = y * ys, yz = y * zs, zz = z * zs;
  double P[16] = {1.0 - (yy + zz), xy - wz, xz + wy, pos3[0], xy + wz, 1.0 - (xx + zz), yz - wx, pos3[1],
                  xz - wy, yz + wx, 1.0 - (xx + yy), pos3[2], 0, 0, 0, 1};
  if (pose16_out) std::memcpy(pose16_out, P, sizeof(P));
  double A[4][8];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 8; c++) A[r][c] = c < 4 ? P[4 * r + c] : (c - 4 == r ? 1.0 : 0.0);
  for (int col = 0; col < 4; col++) {
    int piv = col;
    for (int r = col + 1; r < 4; r++)
      if (std::fabs(A[r][col]) > std::fabs(A[piv][col])) piv = r;
    for (int c = 0; c < 8; c++) std::swap(A[col][c], A[piv][c]);
    const double pv = A[col][col];
    for (int c = 0; c < 8; c++) A[col][c] /= pv;
    for (int r = 0; r < 4; r++)
      if (r != col) {
        const double f = A[r][col];
        for (int c = 0; c < 8; c++) A[r][c] -= f * A[col][c];
      }
  }
  double Tinv[16];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) Tinv[4 * r + c] = A[r][4 + c];
  orc_transform_pcd(world, n, stride, Tinv, out);
}

// transformPcd (fast_lio_sam_qn/include/utilities.hpp:164-175): pcl::transformPointCloud with a Matrix4d --
// per point double math, result cast to float; other fields (intensity) copied (SURVEY App. B.2).
void orc_transform_pcd(const float* in, int n, int stride, const double* T16, float* out /* n x stride */) {
  for (int i = 0; i < n; i++) {
    const float* p = &in[(size_t)i * stride];
    float* o = &out[(size_t)i * stride];
    const double x = p[0], y = p[1], z = p[2];
    for (int d = 3; d < stride; d++) o[d] = p[d];
    for (int r = 0; r < 3; r++) o[r] = (float)(T16[4 * r] * x + T16[4 * r + 1] * y + T16[4 * r + 2] * z + T16[4 * r + 3]);
  }
}

// voxelizePcd (utilities.hpp:38-63) = pcl::VoxelGrid, leaf L on all axes, downsample_all_data (SURVEY App. B.1):
// fp32 min/max -> min_b = floor(min * (1/L)); ijk = floor(p * (1/L)) - float(min_b); idx = i + j*dx + k*dx*dy;
// sort by idx; per occupied voxel the centroid of x, y, z, intensity (fp32 running sums) in idx order.
// PCL stores idx as unsigned int (cloud_point_index_idx) and compares it unsigned: the guard below tests trunc(extent/L)+1
// per axis while dx, dy, dz are floor(max/L) - floor(min/L) + 1, up to one larger, so an index can pass 2^31 and must
// then sort after the smaller ones.  It is computed here modulo 2^32 (PCL's int arithmetic wraps to the same bits).
// Within a voxel PCL's std::sort leaves the order unspecified; ascending point index is used here.
// in/out records: (x, y, z, intensity).  Returns the number of voxels, or -1 when dx*dy*dz overflows int32
// (PCL then warns and returns the input unchanged).
int orc_voxelize(const float* in, int n, float leaf, float* out /* up to n x 4 */) {
  if (n <= 0) return 0;
  const float inv = 1.0f / leaf;
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = 0; i < n; i++)
    for (int d = 0; d < 3; d++) {
      mn[d] = std::min(mn[d], in[4 * (size_t)i + d]);
      mx[d] = std::max(mx[d], in[4 * (size_t)i + d]);
    }
  long long dd[3];
  int min_b[3], div_b[3];
  for (int d = 0; d < 3; d++) {
    dd[d] = (long long)((mx[d] - mn[d]) * inv) + 1;
    min_b[d] = (int)std::floor(mn[d] * inv);
    div_b[d] = (int)std::floor(mx[d] * inv) - min_b[d] + 1;
  }
  if (dd[0] * dd[1] * dd[2] > (long long)std::numeric_limits<int>::max()) return -1;
  std::vector<std::pair<uint32_t, int>> iv(n);
  for (int i = 0; i < n; i++) {
    uint32_t ijk[3];
    for (int d = 0; d < 3; d++) ijk[d] = (uint32_t)(int)(std::floor(in[4 * (size_t)i + d] * inv) - (float)min_b[d]);
    iv[i] = {ijk[0] + ijk[1] * (uint32_t)div_b[0] + ijk[2] * ((uint32_t)div_b[0] * (uint32_t)div_b[1]), i};
  }
  std::sort(iv.begin(), iv.end());
  int nv = 0;
  for (int a = 0; a < n;) {
    int b = a;
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    while (b < n && iv[b].first == iv[a].first) {
      for (int d = 0; d < 4; d++) s[d] += in[4 * (size_t)iv[b].second + d];
      b++;
    }
    for (int d = 0; d < 4; d++) out[4 * (size_t)nv + d] = s[d] / (float)(b - a);
    nv++;
    a = b;
  }
  return nv;
}

// LoopClosure::fetchClosestKeyframeIdx (fast_lio_sam_qn/src/loop_closure.cpp:34-56) for the query keyframe q being
// the LATEST one: candidates are idx < q (keyframes.size() - 1 == q), position distance < radius, time gap > thr,
// strictly-closer wins so the lowest index survives ties.  pos: n x 3 doubles; returns -1 when none.
int orc_fetch_closest(const double* pos, const double* stamp, int q, double radius, double tdiff_thr) {
  double shortest = radius * 3.0;
  int closest = -1;
  for (int idx = 0; idx < q; idx++) {
    const double dx = pos[3 * idx] - pos[3 * q], dy = pos[3 * idx + 1] - pos[3 * q + 1], dz = pos[3 * idx + 2] - pos[3 * q + 2];
    const double dist = std::sqrt(dx * dx + dy * dy + dz * dz);
    if (radius > dist && tdiff_thr < (stamp[q] - stamp[idx])) {
      if (dist < shortest) {
        shortest = dist;
        closest = idx;
      }
    }
  }
  return closest;
}

}  // extern "C"
