// oracle/ref_nanoflann_shim.cpp -- TEST INFRASTRUCTURE ONLY.
//
// Thin C wrapper that compiles the REFERENCE's own kd-tree
//   <reference>/third_party/nano_gicp/include/nano_gicp/impl/nanoflann_impl.hpp
// (std-only header, nanoflann v1.3.2) from where it lies, configured exactly as
// the reference configures it in nano_gicp/nanoflann.hpp:
//   * metric SO3_Adaptor<float, Adaptor>, DIM 3, int index   (nanoflann.hpp:100-102)
//   * leaf_max_size 100                                       (nanoflann.hpp:114)
//   * KNNResultSet<float,int> + findNeighbors(SearchParams()) (nanoflann.hpp:148-150)
// Output goes to oracle/_ref/libref_nanoflann.so (git-ignored, travels to the GPU
// box).  No reference source is copied into this repository; only the include
// path points at the reference tree (Makefile variable REF).  Built by oracle/Makefile target `ref`.
#include <nano_gicp/impl/nanoflann_impl.hpp>

#include <cstddef>
#include <vector>

namespace {
struct Adaptor {
  const float* xyz;
  size_t n;
  size_t stride;
  inline size_t kdtree_get_point_count() const { return n; }
  inline float kdtree_get_pt(const size_t idx, int dim) const { return xyz[idx * stride + dim]; }
  template <class BBOX>
  bool kdtree_get_bbox(BBOX&) const {
    return false;
  }
};
typedef nanoflann::KDTreeSingleIndexAdaptor<nanoflann::SO3_Adaptor<float, Adaptor>, Adaptor, 3, int> Tree;
struct Handle {
  std::vector<float> pts;  // private copy so the caller's buffer may go away
  Adaptor ad;
  Tree* tree;
};
}  // namespace

extern "C" {

void* ref_nf_build(const float* xyz, int n, int stride) {
  Handle* h = new Handle;
  h->pts.resize((size_t)n * 3);
  for (int i = 0; i < n; i++)
    for (int d = 0; d < 3; d++) h->pts[(size_t)i * 3 + d] = xyz[(size_t)i * stride + d];
  h->ad = Adaptor{h->pts.data(), (size_t)n, 3};
  h->tree = new Tree(3, h->ad, nanoflann::KDTreeSingleIndexAdaptorParams(100));
  h->tree->buildIndex();
  return h;
}

void ref_nf_free(void* hv) {
  Handle* h = (Handle*)hv;
  delete h->tree;
  delete h;
}

// one query, k results ascending (k <= n assumed, as in the reference)
void ref_nf_knn_one(void* hv, const float* q, int k, int* idx, float* d2) {
  Handle* h = (Handle*)hv;
  nanoflann::KNNResultSet<float, int> rs(k);
  rs.init(idx, d2);
  h->tree->findNeighbors(rs, q, nanoflann::SearchParams());
}

void ref_nf_knn(void* hv, const float* q, int nq, int qstride, int k, int* idx, float* d2) {
#pragma omp parallel for schedule(guided, 8)
  for (int i = 0; i < nq; i++) ref_nf_knn_one(hv, &q[(size_t)i * qstride], k, &idx[(size_t)i * k], &d2[(size_t)i * k]);
}

}  // extern "C"
