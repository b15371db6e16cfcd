// A client of nanoflann::KdTreeFLANN (nano_gicp/nanoflann.hpp:54-108) as code written against the reference uses it:
// NanoGICP's public source_kdtree_ / target_kdtree_, and a standalone tree over an index subset.
// usage: kdtree_client src.bin dst.bin queries.bin sq_radius   (bin = n x 4 float32: x y z intensity)
// Prints one JSON object: for every search, the per-query counts and the concatenated indices / squared distances.
#define B200REG_HOST_IMPLEMENTATION
#include <nano_gicp/nano_gicp.hpp>
#include <nano_gicp/nanoflann.hpp>
#include <nano_gicp/point_type_nano_gicp.hpp>

#if defined(B200REG_EXPECT_PCL) && !defined(B200REG_HAVE_PCL)
#error "the PCL/Eigen configuration of the facade was requested but b200reg_compat.hpp did not select it"
#endif

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>
#include <vector>

static pcl::PointCloud<PointType> load(const char* path) {
  pcl::PointCloud<PointType> c;
  std::ifstream f(path, std::ios::binary);
  float v[4];
  while (f.read(reinterpret_cast<char*>(v), sizeof(v))) {
    PointType p;
    p.x = v[0];
    p.y = v[1];
    p.z = v[2];
    p.intensity = v[3];
    c.push_back(p);
  }
  return c;
}

static bool first_key = true;
// "name": {"count": [...], "idx": [...], "d2": [...]}
template <typename Search>
static void emit(const char* name, const pcl::PointCloud<PointType>& queries, Search search) {
  std::vector<int> counts, all_idx;
  std::vector<float> all_d2;
  std::vector<int> idx;
  std::vector<float> d2;
  for (size_t i = 0; i < queries.size(); i++) {
    const int n = search(queries[i], idx, d2);
    counts.push_back(n);
    all_idx.insert(all_idx.end(), idx.begin(), idx.end());
    all_d2.insert(all_d2.end(), d2.begin(), d2.end());
  }
  std::printf("%s\"%s\": {\"count\": [", first_key ? "" : ", ", name);
  first_key = false;
  for (size_t i = 0; i < counts.size(); i++) std::printf("%s%d", i ? ", " : "", counts[i]);
  std::printf("], \"idx\": [");
  for (size_t i = 0; i < all_idx.size(); i++) std::printf("%s%d", i ? ", " : "", all_idx[i]);
  std::printf("], \"d2\": [");
  for (size_t i = 0; i < all_d2.size(); i++) std::printf("%s%.9g", i ? ", " : "", all_d2[i]);
  std::printf("]}");
}

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  pcl::PointCloud<PointType>::Ptr src(new pcl::PointCloud<PointType>(load(argv[1])));
  pcl::PointCloud<PointType>::Ptr dst(new pcl::PointCloud<PointType>(load(argv[2])));
  const pcl::PointCloud<PointType> queries = load(argv[3]);
  const double r2 = std::atof(argv[4]);
  using Tree = nanoflann::KdTreeFLANN<PointType>;

  nano_gicp::NanoGICP<PointType, PointType> gicp;
  gicp.setInputSource(src);
  gicp.setInputTarget(dst);
  std::printf("{");
  emit("source_radius", queries, [&](const PointType& q, std::vector<int>& i, std::vector<float>& d) {
    return gicp.source_kdtree_->radiusSearch(q, r2, i, d);
  });
  gicp.target_kdtree_->setSortedResults(true);
  emit("target_radius_sorted", queries, [&](const PointType& q, std::vector<int>& i, std::vector<float>& d) {
    return gicp.target_kdtree_->radiusSearch(q, r2, i, d);
  });
  emit("target_knn5", queries, [&](const PointType& q, std::vector<int>& i, std::vector<float>& d) {
    return gicp.target_kdtree_->nearestKSearch(q, 5, i, d);
  });
  // swapSourceAndTarget swaps the trees with the clouds (nano_gicp_impl.hpp:93)
  gicp.swapSourceAndTarget();
  emit("swapped_source_radius_sorted", queries, [&](const PointType& q, std::vector<int>& i, std::vector<float>& d) {
    return gicp.source_kdtree_->radiusSearch(q, r2, i, d);
  });
  emit("swapped_target_radius", queries, [&](const PointType& q, std::vector<int>& i, std::vector<float>& d) {
    return gicp.target_kdtree_->radiusSearch(q, r2, i, d);
  });
  const int same_cloud = gicp.source_kdtree_->getInputCloud() == dst && gicp.target_kdtree_->getInputCloud() == src;

  // a standalone tree over every third point of dst: results are positions in `indices`
  Tree::IndicesPtr every3(new std::vector<int>);
  for (int j = 0; j < static_cast<int>(dst->size()); j += 3) every3->push_back(j);
  Tree subset;
  subset.setEpsilon(0.1f);  // stored, not used: the engine returns the exact set
  subset.setInputCloud(dst, every3);
  emit("subset_radius", queries, [&](const PointType& q, std::vector<int>& i, std::vector<float>& d) {
    return subset.radiusSearch(q, r2, i, d);
  });
  Tree::Ptr copy = subset.makeShared();
  copy->setSortedResults(true);
  emit("subset_radius_sorted", queries, [&](const PointType& q, std::vector<int>& i, std::vector<float>& d) {
    return copy->radiusSearch(q, r2, i, d);
  });
  // k > n: the outputs are resized to k, the return value is the number found
  Tree::IndicesConstPtr four(new std::vector<int>{0, 1, 2, 3});
  Tree tiny(true);
  tiny.setInputCloud(dst, four);
  emit("tiny_knn6", queries, [&](const PointType& q, std::vector<int>& i, std::vector<float>& d) {
    return tiny.nearestKSearch(q, 6, i, d);
  });
  std::printf(", \"same_cloud\": %d}\n", same_cloud);
  return 0;
}
