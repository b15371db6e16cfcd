// A client of nanoflann::KdTreeFLANN::nearestKSearch (nano_gicp/nanoflann.hpp:140-152) with k above 32, as code written
// against the reference calls it: NanoGICP's target_kdtree_ and a standalone tree.
// usage: kdtree_knn_client cloud.bin queries.bin k   (bin = n x 4 float32: x y z intensity)
// Prints one JSON object: for every search, the per-query return values and the concatenated indices / squared distances.
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

static void emit(const char* name, bool first, const pcl::PointCloud<PointType>& queries, const nanoflann::KdTreeFLANN<PointType>& tree,
                 int k) {
  std::vector<int> counts, all_idx, idx;
  std::vector<float> all_d2, d2;
  for (size_t i = 0; i < queries.size(); i++) {
    counts.push_back(tree.nearestKSearch(queries[i], k, idx, d2));
    all_idx.insert(all_idx.end(), idx.begin(), idx.end());
    all_d2.insert(all_d2.end(), d2.begin(), d2.end());
  }
  std::printf("%s\"%s\": {\"count\": [", first ? "" : ", ", name);
  for (size_t i = 0; i < counts.size(); i++) std::printf("%s%d", i ? ", " : "", counts[i]);
  std::printf("], \"idx\": [");
  for (size_t i = 0; i < all_idx.size(); i++) std::printf("%s%d", i ? ", " : "", all_idx[i]);
  std::printf("], \"d2\": [");
  for (size_t i = 0; i < all_d2.size(); i++) std::printf("%s%.9g", i ? ", " : "", all_d2[i]);
  std::printf("]}");
}

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  pcl::PointCloud<PointType>::Ptr cloud(new pcl::PointCloud<PointType>(load(argv[1])));
  const pcl::PointCloud<PointType> queries = load(argv[2]);
  const int k = std::atoi(argv[3]);

  nano_gicp::NanoGICP<PointType, PointType> gicp;
  gicp.setInputTarget(cloud);
  nanoflann::KdTreeFLANN<PointType> tree;
  tree.setInputCloud(cloud);
  std::printf("{");
  emit("target_knn", true, queries, *gicp.target_kdtree_, k);
  emit("standalone_knn", false, queries, tree, k);
  std::printf("}\n");
  return 0;
}
