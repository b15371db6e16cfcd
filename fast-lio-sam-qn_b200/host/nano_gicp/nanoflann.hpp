// nanoflann::KdTreeFLANN<PointT> -- host facade over the C ABI (include/b200reg.h).
//
// Keeps the public surface of third_party/nano_gicp/include/nano_gicp/nanoflann.hpp:54-108, so code that includes
// <nano_gicp/nanoflann.hpp> or holds NanoGICP::source_kdtree_ / target_kdtree_ compiles unchanged.  The index is the
// engine's device-side LBVH (b200reg_clouds_create); searches run in hand-written sm_90a kernels (b200reg_knn,
// b200reg_radius_search).  Differences a maintainer should know (also in INTEGRATION.md):
//   * radiusSearch takes a SQUARED radius, like the reference: `radius` goes unchanged into RadiusResultSet<float, int>
//     (nanoflann.hpp:162), which compares it with squared distances.  radiusSearch(p, 1.5, ...) returns every point with
//     d2 < 1.5f (strict), i.e. a ball of radius sqrt(1.5) -- NOT what pcl::KdTree::radiusSearch(p, 1.5, ...) returns;
//   * radiusSearch returns ALL neighbours and their number.  The reference takes the count from findNeighbors' return value,
//     which is result.full() (nanoflann_impl.hpp:1249), always true for a RadiusResultSet: it returns exactly one entry,
//     even when it found none;
//   * order: unsorted (the default) is ascending index, sorted is ascending (d2, index).  The reference returns its kd-tree's
//     visit order, and sorts by d2 alone with ties in unspecified order;
//   * setEpsilon is stored and not used: the reference prunes approximately with eps > 0 (nanoflann_impl.hpp:1408), the
//     engine always returns the exact set, a superset of the reference's;
//   * nearestKSearch takes any k >= 1 and returns min(k, n); k > n pads with index -1 and d2 FLT_MAX; equal distances
//     resolve to the lower index; a query with a NaN coordinate gets a row of padding;
//   * Ptr / ConstPtr / IndicesPtr are std::shared_ptr (the reference uses boost::shared_ptr); the copy constructor (declared
//     but not defined by the reference) shares the device index;
//   * the calls are thread-safe (the reference's radiusSearch keeps its results in a function-local static vector).
#pragma once
#include <cstdio>
#include <memory>
#include <vector>

#include "../b200reg_compat.hpp"

namespace b200reg_host {
// A device cloud shared by the objects that search it (NanoGICP and its two KdTreeFLANN members): destroyed with the last.
using DeviceCloud = std::shared_ptr<b200reg_cloud>;
inline DeviceCloud make_device_cloud(const float* xyz, size_t n, size_t stride_bytes) {
  if (n == 0) return DeviceCloud();
  b200reg_cloud* cl = nullptr;
  const float* ptrs[1] = {xyz};
  const size_t ns[1] = {n};
  const int rc = b200reg_clouds_create(context(), 1, ptrs, ns, stride_bytes, 0, &cl);
  if (rc != 0) {
    std::fprintf(stderr, "b200reg: clouds_create failed (%d): %s\n", rc, b200reg_last_error());
    return DeviceCloud();
  }
  return DeviceCloud(cl, [](b200reg_cloud* p) { b200reg_cloud_destroy(context(), p); });
}
}  // namespace b200reg_host

namespace nanoflann {

template <typename PointT>
class KdTreeFLANN {
 public:
  typedef pcl::PointCloud<PointT> PointCloud;
  typedef typename pcl::PointCloud<PointT>::Ptr PointCloudPtr;
  typedef typename pcl::PointCloud<PointT>::ConstPtr PointCloudConstPtr;

  typedef std::shared_ptr<KdTreeFLANN<PointT>> Ptr;
  typedef std::shared_ptr<const KdTreeFLANN<PointT>> ConstPtr;
  typedef std::shared_ptr<std::vector<int>> IndicesPtr;
  typedef std::shared_ptr<const std::vector<int>> IndicesConstPtr;

  KdTreeFLANN(bool sorted = false) : sorted_(sorted) {}
  KdTreeFLANN(const KdTreeFLANN<PointT>& k) = default;

  void setEpsilon(float eps) { eps_ = eps; }
  void setSortedResults(bool sorted) { sorted_ = sorted; }
  inline Ptr makeShared() { return Ptr(new KdTreeFLANN<PointT>(*this)); }

  // indices given: the tree holds cloud[indices[j]] and every search returns positions j in `indices` (nanoflann.hpp:184-191)
  void setInputCloud(const PointCloudConstPtr& cloud, const IndicesConstPtr& indices = IndicesConstPtr()) {
    cloud_ = cloud;
    indices_ = indices;
    dev_.reset();
    if (!cloud) return;
    if (indices) {
      std::vector<float> xyz(3 * indices->size());
      for (size_t j = 0; j < indices->size(); j++) {
        const PointT& p = cloud->points[(*indices)[j]];
        xyz[3 * j] = p.x;
        xyz[3 * j + 1] = p.y;
        xyz[3 * j + 2] = p.z;
      }
      dev_ = b200reg_host::make_device_cloud(xyz.data(), indices->size(), 12);
    } else {
      dev_ = b200reg_host::make_device_cloud(reinterpret_cast<const float*>(cloud->points.data()), cloud->size(), sizeof(PointT));
    }
  }
  inline PointCloudConstPtr getInputCloud() const { return cloud_; }

  int nearestKSearch(const PointT& point, int k, std::vector<int>& k_indices, std::vector<float>& k_sqr_distances) const {
    static_assert(sizeof(int) == sizeof(int32_t), "indices are written as int32_t");
    k_indices.resize(k > 0 ? k : 0);
    k_sqr_distances.resize(k > 0 ? k : 0);
    if (!dev_ || k <= 0) return 0;
    const float q[3] = {point.x, point.y, point.z};
    const int rc = b200reg_knn(b200reg_host::context(), dev_.get(), q, 1, 12, k, reinterpret_cast<int32_t*>(k_indices.data()),
                               k_sqr_distances.data());
    if (rc != 0) {
      std::fprintf(stderr, "b200reg: nearestKSearch failed (%d): %s\n", rc, b200reg_last_error());
      return 0;
    }
    const int n = static_cast<int>(b200reg_cloud_size(dev_.get()));
    return k < n ? k : n;
  }

  // `radius` is SQUARED (see the header comment): the result holds every point with d2 < float(radius)
  int radiusSearch(const PointT& point, double radius, std::vector<int>& k_indices, std::vector<float>& k_sqr_distances) const {
    k_indices.clear();
    k_sqr_distances.clear();
    if (!dev_) return 0;
    const float q[3] = {point.x, point.y, point.z};
    int64_t off[2] = {0, 0};
    size_t cap = k_indices.capacity() > 128 ? k_indices.capacity() : 128;
    for (int attempt = 0; attempt < 2; attempt++) {
      k_indices.resize(cap);
      k_sqr_distances.resize(cap);
      const int rc = b200reg_radius_search(b200reg_host::context(), dev_.get(), q, 1, 12, radius, sorted_ ? 1 : 0, off, cap,
                                           reinterpret_cast<int32_t*>(k_indices.data()), k_sqr_distances.data());
      if (rc == 0) break;
      if (rc != B200REG_ESTATE || attempt == 1) {
        std::fprintf(stderr, "b200reg: radiusSearch failed (%d): %s\n", rc, b200reg_last_error());
        off[1] = 0;
        break;
      }
      cap = static_cast<size_t>(off[1]);  // the offsets are filled: retry with room for exactly what was found
    }
    k_indices.resize(static_cast<size_t>(off[1]));
    k_sqr_distances.resize(static_cast<size_t>(off[1]));
    return static_cast<int>(off[1]);
  }

  // facade-internal: search a device cloud that is already built (NanoGICP's source / target) -- no second upload
  void shareDeviceCloud(const PointCloudConstPtr& cloud, const b200reg_host::DeviceCloud& dev) {
    cloud_ = cloud;
    indices_.reset();
    dev_ = dev;
  }

 private:
  bool sorted_ = false;
  float eps_ = 0.f;  // stored, not reproduced (header comment)
  PointCloudConstPtr cloud_;
  IndicesConstPtr indices_;
  b200reg_host::DeviceCloud dev_;
};

}  // namespace nanoflann
