// tests/golden/ref_radius_shim.cpp -- TEST INFRASTRUCTURE ONLY (compiled by make_radius_golden.py, never shipped).
//
// Thin C wrapper that compiles the REFERENCE's own kd-tree
//   <reference>/third_party/nano_gicp/include/nano_gicp/impl/nanoflann_impl.hpp
// (std-only header, nanoflann v1.3.2) from where it lies, configured exactly as KdTreeFLANN configures it
// (nano_gicp/nanoflann.hpp:100-114: SO3_Adaptor<float, Adaptor> metric, DIM 3, int index, leaf_max_size 100), and runs
// KdTreeFLANN::radiusSearch's search (nanoflann.hpp:159-166): RadiusResultSet<float, int> through findNeighbors, then
// std::sort with IndexDist_Sorter when sorted.  No reference source is copied; only the include path points at the
// reference tree.
#include <nano_gicp/impl/nanoflann_impl.hpp>

#include <algorithm>
#include <cstddef>
#include <utility>
#include <vector>

namespace {
struct Adaptor {
  const float* xyz;
  size_t n;
  inline size_t kdtree_get_point_count() const { return n; }
  inline float kdtree_get_pt(const size_t idx, int dim) const { return xyz[idx * 3 + dim]; }
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

// xyz: n packed (x, y, z) records
void* ref_radius_build(const float* xyz, int n) {
  Handle* h = new Handle;
  h->pts.assign(xyz, xyz + (size_t)n * 3);
  h->ad = Adaptor{h->pts.data(), (size_t)n};
  h->tree = new Tree(3, h->ad, nanoflann::KDTreeSingleIndexAdaptorParams(100));
  h->tree->buildIndex();
  return h;
}

void ref_radius_free(void* hv) {
  Handle* h = (Handle*)hv;
  delete h->tree;
  delete h;
}

// One query.  `radius` is passed on unchanged (RadiusResultSet compares it with SQUARED distances).  The count is the
// result set's size -- the reference's radiusSearch takes it from findNeighbors' return value instead, which is
// result.full() (nanoflann_impl.hpp:1249), always true for a RadiusResultSet.  Writes at most cap entries; returns the
// number found.
int ref_radius_search(void* hv, const float* q, double radius, int sorted, int cap, int* idx, float* d2) {
  Handle* h = (Handle*)hv;
  std::vector<std::pair<int, float> > indices_dist;
  nanoflann::RadiusResultSet<float, int> rs(radius, indices_dist);
  h->tree->findNeighbors(rs, q, nanoflann::SearchParams());
  if (sorted) std::sort(indices_dist.begin(), indices_dist.end(), nanoflann::IndexDist_Sorter());
  const int n = (int)indices_dist.size();
  for (int i = 0; i < n && i < cap; i++) {
    idx[i] = indices_dist[i].first;
    d2[i] = indices_dist[i].second;
  }
  return n;
}

}  // extern "C"
