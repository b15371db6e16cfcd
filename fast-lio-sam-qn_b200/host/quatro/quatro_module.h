// quatro<PointType> -- host facade over the C ABI (include/b200reg.h); keeps the surface of
// third_party/Quatro/include/quatro/quatro_module.h:19-37 (constructor argument order and types, align()).
// FPFH, matching and the TEASER++ QUATRO solve all run on the GPU (csrc/quatro.cu); no CPU fallback.
#pragma once
#include <cstdio>

#include "../b200reg_compat.hpp"

template <typename PointType>
class quatro {
 public:
  quatro() { b200reg_default_quatro_params(&prm_); }
  // fast_lio_sam_qn/src/loop_closure.cpp:18-27 passes all ten arguments.  num_max_corres: 1..8189 with optimized
  // matching (at most num_max_corres + 3 correspondences are kept and solved); a larger value makes align() print the
  // refusal to stderr and return Identity / invalid
  quatro(const double& fpfh_normal_radi, const double& fpfh_radi, const double noise_bound, const double& rot_gnc_fact,
         const double& rot_cost_thr, const int& rot_max_iter, const bool& estimat_scale, const bool& use_optimized_matching = true,
         const double& distance_threshold = 30.0, const int& num_max_corres = 200) {
    b200reg_default_quatro_params(&prm_);
    prm_.fpfh_normal_radius = fpfh_normal_radi;
    prm_.fpfh_radius = fpfh_radi;
    prm_.noise_bound = noise_bound;
    prm_.rot_gnc_factor = rot_gnc_fact;
    prm_.rot_cost_thr = rot_cost_thr;
    prm_.rot_max_iter = rot_max_iter;
    prm_.estimate_scale = estimat_scale ? 1 : 0;
    prm_.use_optimized_matching = use_optimized_matching ? 1 : 0;
    prm_.distance_threshold = distance_threshold;
    prm_.max_corres = num_max_corres;
  }
  void setSeed(uint64_t seed) { prm_.seed = seed; }  // the reference seeds rand() with time(NULL) (matcher.cc:465)

  // returns Identity and if_valid = false when no correspondences survive (quatro_module.cc:63-66)
  Eigen::Matrix4d align(const pcl::PointCloud<PointType>& src, const pcl::PointCloud<PointType>& dst, bool& if_valid) {
    Eigen::Matrix4d out = Eigen::Matrix4d::Identity();
    if_valid = false;
    if (src.size() == 0 || dst.size() == 0) return out;
    b200reg_ctx* ctx = b200reg_host::context();
    const float* ptrs[2] = {reinterpret_cast<const float*>(src.points.data()), reinterpret_cast<const float*>(dst.points.data())};
    const size_t ns[2] = {src.size(), dst.size()};
    b200reg_cloud* cl[2] = {nullptr, nullptr};
    int rc = b200reg_clouds_create(ctx, 2, ptrs, ns, sizeof(PointType), 0, cl);
    if (rc == 0) {
      b200reg_quatro_info info;
      rc = b200reg_quatro_align(ctx, 1, &cl[0], &cl[1], &prm_, &info, nullptr);
      if (rc == 0) {
        if_valid = info.valid != 0;
        b200reg_host::from_rowmajor(info.T, out);
        last_ = info;
      }
    }
    if (rc != 0) std::fprintf(stderr, "b200reg: quatro align failed (%d): %s\n", rc, b200reg_last_error());
    b200reg_cloud_destroy(ctx, cl[0]);
    b200reg_cloud_destroy(ctx, cl[1]);
    return out;
  }
  const b200reg_quatro_info& lastInfo() const { return last_; }

 private:
  b200reg_quatro_params prm_;
  b200reg_quatro_info last_{};
};
