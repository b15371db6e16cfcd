// nano_gicp::NanoGICP<PointSource, PointTarget> -- host facade over the C ABI (include/b200reg.h).
//
// Keeps the public surface of third_party/nano_gicp/include/nano_gicp/nano_gicp.hpp:58-137 and of the base classes
// it exposes (LsqRegistration, lsq_registration.hpp:56-116; the pcl::Registration setters/getters used at
// fast_lio_sam_qn/src/loop_closure.cpp:9-16,120-133), so LoopClosure links against this header unchanged.
// Nothing is computed on the host: every call forwards to hand-written sm_90a kernels; without a GPU the process
// aborts (b200reg_host::context()).
//
// Differences a maintainer should know (also in INTEGRATION.md):
//   * the class does not derive from pcl::Registration (nothing in fast_lio_sam_qn/src uses it polymorphically);
//   * setNumThreads is accepted and ignored; RANSAC* / EuclideanFitnessEpsilon setters are stored and never read,
//     exactly like the reference's LSQ path (SURVEY.md §8b);
//   * all five RegularizationMethods are built (PLANE is the default, nano_gicp_impl.hpp:61); setCorrespondenceRandomness takes
//     any k >= 1 (k > 32 computes the covariances one warp per point, b200reg_clouds_covariances_ex);
//   * source_kdtree_/target_kdtree_ are nanoflann::KdTreeFLANN facades (nanoflann.hpp in this directory) over the SAME device
//     cloud and index the class builds for registration: no second upload, no second build;
//   * covariances live on the device and are materialised on the host lazily by getSource/TargetCovariances() as
//     Eigen::Matrix4d (4th row/column zero, like the reference's, nano_gicp_impl.hpp:354); setSource/TargetCovariances
//     upload the caller's.
//   * setDebugPrint(true) prints the reference's LM table to std::cout, row for row, but all of it when the solve has
//     finished on the device (the rows come from the solve's trace, b200reg_lm_trace), not while it runs; lastLmTrace()
//     returns the records themselves.
//   * getFitnessScore(max_range) sums the per-point squared distances the device's fitness pass found in the last align()
//     (b200reg_residuals); lastResiduals() returns those rows.
#pragma once
#include <array>
#include <cmath>
#include <cstdio>
#include <iostream>
#include <limits>
#include <memory>
#include <vector>

#include "../b200reg_compat.hpp"
#include "nanoflann.hpp"

namespace nano_gicp {

enum class RegularizationMethod { NONE, MIN_EIG, NORMALIZED_MIN_EIG, PLANE, FROBENIUS };  // gicp/gicp_settings.hpp:47
enum class LSQ_OPTIMIZER_TYPE { GaussNewton, LevenbergMarquardt };

template <typename PointSource, typename PointTarget>
class NanoGICP {
 public:
  using Scalar = float;
  using Matrix4 = Eigen::Matrix4f;
  using PointCloudSource = pcl::PointCloud<PointSource>;
  using PointCloudSourcePtr = typename PointCloudSource::Ptr;
  using PointCloudSourceConstPtr = typename PointCloudSource::ConstPtr;
  using PointCloudTarget = pcl::PointCloud<PointTarget>;
  using PointCloudTargetPtr = typename PointCloudTarget::Ptr;
  using PointCloudTargetConstPtr = typename PointCloudTarget::ConstPtr;
  using Cov = Eigen::Matrix4d;  // 4th row/col zero (nano_gicp_impl.hpp:354)
  using CovVector = std::vector<Eigen::Matrix4d, Eigen::aligned_allocator<Eigen::Matrix4d>>;  // nano_gicp.hpp:91-106
  using Matrix6d = Eigen::Matrix<double, 6, 6>;
  // per source point of the last align(), in the source cloud's order: the nearest target point at the final pose and its
  // fp32 squared distance, the values getFitnessScore() averages (b200reg_residuals)
  struct Residuals {
    std::vector<int32_t> nn;
    std::vector<float> d2;
  };

  NanoGICP() {
    source_kdtree_.reset(new nanoflann::KdTreeFLANN<PointSource>);  // nano_gicp_impl.hpp:62-63
    target_kdtree_.reset(new nanoflann::KdTreeFLANN<PointTarget>);
    b200reg_default_gicp_params(&prm_);
    prm_.k_correspondences = 20;                                 // nano_gicp_impl.hpp:57
    prm_.max_iterations = 64;                                    // lsq_registration_impl.hpp:51
    prm_.transformation_eps = 5e-4;                              // lsq_registration_impl.hpp:54
    prm_.max_corr_dist = std::sqrt(std::numeric_limits<double>::max());  // corr_dist_threshold_ = FLT_MAX-ish (:59)
    final_.fill(0.f);
    final_[0] = final_[5] = final_[10] = final_[15] = 1.f;
    final_hessian_ = Matrix6d::Identity();  // lsq_registration_impl.hpp:62
  }
  ~NanoGICP() { release(); }
  NanoGICP(const NanoGICP&) = delete;
  NanoGICP& operator=(const NanoGICP&) = delete;

  // ---- nano_gicp.hpp:82-84
  void setNumThreads(int) {}
  void setCorrespondenceRandomness(int k) {
    if (k != prm_.k_correspondences) {
      prm_.k_correspondences = k;
      src_cov_ok_ = tgt_cov_ok_ = false;
    }
  }
  void setRegularizationMethod(RegularizationMethod m) {
    if (static_cast<int>(m) != prm_.regularization) {
      prm_.regularization = static_cast<int>(m);  // same enumerator order as gicp/gicp_settings.hpp:47
      src_cov_ok_ = tgt_cov_ok_ = false;
    }
  }
  // ---- pcl::Registration setters (loop_closure.cpp:11-16)
  void setMaximumIterations(int n) { prm_.max_iterations = n; }
  void setRANSACIterations(int n) { ransac_iterations_ = n; }
  void setMaxCorrespondenceDistance(double d) { prm_.max_corr_dist = d; }
  void setTransformationEpsilon(double e) { prm_.transformation_eps = e; }
  void setEuclideanFitnessEpsilon(double e) { euclidean_fitness_epsilon_ = e; }
  void setRANSACOutlierRejectionThreshold(double t) { ransac_threshold_ = t; }
  int getMaximumIterations() const { return prm_.max_iterations; }
  double getMaxCorrespondenceDistance() const { return prm_.max_corr_dist; }
  double getTransformationEpsilon() const { return prm_.transformation_eps; }
  // ---- LsqRegistration (lsq_registration.hpp:84-92)
  void setRotationEpsilon(double e) { prm_.rotation_eps = e; }
  void setInitialLambdaFactor(double f) { prm_.lm_init_lambda_factor = f; }
  void setDebugPrint(bool lm_debug_print) { lm_debug_print_ = lm_debug_print; }

  // ---- inputs (nano_gicp_impl.hpp:120-139): pointer-identity early-out, index build, covariances cleared
  void setInputSource(const PointCloudSourceConstPtr& cloud) {
    if (input_ == cloud) return;
    input_ = cloud;
    upload(cloud, &src_);
    source_kdtree_->shareDeviceCloud(cloud, src_);
    src_cov_ok_ = false;
  }
  void setInputTarget(const PointCloudTargetConstPtr& cloud) {
    if (target_ == cloud) return;
    target_ = cloud;
    upload(cloud, &tgt_);
    target_kdtree_->shareDeviceCloud(cloud, tgt_);
    tgt_cov_ok_ = false;
  }
  void registerInputSource(const PointCloudSourceConstPtr& cloud) { setInputSource(cloud); }
  void clearSource() {
    input_.reset();
    destroy(&src_);
    src_cov_ok_ = false;
  }
  void clearTarget() {
    target_.reset();
    destroy(&tgt_);
    tgt_cov_ok_ = false;
  }
  void swapSourceAndTarget() {  // nano_gicp_impl.hpp:92-100
    std::swap(input_, target_);
    std::swap(src_, tgt_);
    std::swap(src_cov_ok_, tgt_cov_ok_);
    source_kdtree_.swap(target_kdtree_);
  }
  bool calculateSourceCovariances() { return covariances(src_.get(), &src_cov_ok_); }
  bool calculateTargetCovariances() { return covariances(tgt_.get(), &tgt_cov_ok_); }
  CovVector getSourceCovariances() { return fetch_covs(src_.get(), &src_cov_ok_); }
  CovVector getTargetCovariances() { return fetch_covs(tgt_.get(), &tgt_cov_ok_); }
  // nano_gicp.hpp:91-93, nano_gicp_impl.hpp:142-150: the caller's covariances replace the computed ones
  void setSourceCovariances(const CovVector& covs) { push_covs(src_.get(), covs, &src_cov_ok_); }
  void setTargetCovariances(const CovVector& covs) { push_covs(tgt_.get(), covs, &tgt_cov_ok_); }
  // lsq_registration.hpp:88: H of the last linearize (Identity before the first align)
  const Matrix6d& getFinalHessian() const { return final_hessian_; }

  // ---- pcl::Registration::align (SURVEY.md App. B.3): identity guess unless given
  void align(PointCloudSource& output) { align(output, Matrix4::Identity()); }
  void align(PointCloudSource& output, const Matrix4& guess) {
    converged_ = false;
    if (!src_ || !tgt_) {
      std::fprintf(stderr, "b200reg: align() called without source/target\n");
      return;
    }
    double g[16];
    b200reg_host::to_rowmajor(guess, g);
    b200reg_cloud* s[1] = {src_.get()};
    b200reg_cloud* t[1] = {tgt_.get()};
    b200reg_ctx* ctx = b200reg_host::context();
    lm_trace_.clear();
    residuals_.nn.clear();
    residuals_.d2.clear();
    if (lm_debug_print_) b200reg_ctx_set_lm_trace(ctx, 1);
    b200reg_ctx_set_residuals(ctx, 1);  // getFitnessScore(max_range) reads the fitness pass's rows
    const int rc = b200reg_gicp_align(ctx, 1, s, t, g, &prm_, &res_);
    if (lm_debug_print_) {
      if (rc == 0) fetch_lm_trace(ctx);
      b200reg_ctx_set_lm_trace(ctx, 0);
    }
    if (rc == 0) fetch_residuals(ctx);
    b200reg_ctx_set_residuals(ctx, 0);
    if (rc != 0) {
      std::fprintf(stderr, "b200reg: gicp_align failed (%d): %s\n", rc, b200reg_last_error());
      return;
    }
    if (lm_debug_print_) print_lm_trace();
    if (res_.lm_failed) std::fprintf(stderr, "lm not converged!!\n");  // lsq_registration_impl.hpp:106
    src_cov_ok_ = tgt_cov_ok_ = true;
    converged_ = res_.converged != 0;
    for (int i = 0; i < 16; i++) final_[i] = res_.Tf[i];
    for (int r = 0; r < 6; r++)
      for (int c = 0; c < 6; c++) final_hessian_(r, c) = res_.final_hessian[6 * r + c];
    // output = transformPointCloud(*input_, final_transformation_) (lsq_registration_impl.hpp:114): all fields kept
    std::vector<float> xyz(3 * input_->size());
    b200reg_transform_cloud(b200reg_host::context(), src_.get(), res_.Tf, xyz.data());
    output = *input_;
    for (size_t i = 0; i < output.size(); i++) {
      output.points[i].x = xyz[3 * i];
      output.points[i].y = xyz[3 * i + 1];
      output.points[i].z = xyz[3 * i + 2];
    }
  }
  bool hasConverged() const { return converged_; }
  Matrix4 getFinalTransformation() const {
    Matrix4 m;
    float rm[16];
    for (int i = 0; i < 16; i++) rm[i] = final_[i];
    b200reg_host::from_rowmajor(rm, m);
    return m;
  }
  // mean squared 1-NN distance of the transformed source; the default (no range cap) is what loop_closure.cpp:127 uses.
  // With a cap, pcl::Registration::getFitnessScore's rule over the last align()'s rows: a point counts iff its SQUARED
  // distance is <= max_range, summed in point order in double; DBL_MAX when none counts (a NaN max_range keeps none)
  double getFitnessScore(double max_range = std::numeric_limits<double>::max()) const {
    if (max_range == std::numeric_limits<double>::max()) return res_.fitness;
    double s = 0;
    size_t nr = 0;
    for (float v : residuals_.d2)
      if (v <= max_range) {
        s += v;
        nr++;
      }
    return nr ? s / nr : std::numeric_limits<double>::max();
  }
  int nr_iterations() const { return res_.iterations; }
  const b200reg_result& lastResult() const { return res_; }
  // every LM trial of the last align(), in execution order; empty unless setDebugPrint(true)
  const std::vector<b200reg_lm_trial>& lastLmTrace() const { return lm_trace_; }
  // the fitness pass's rows of the last align() (empty before the first and after a failed one)
  const Residuals& lastResiduals() const { return residuals_; }

  // nano_gicp.hpp:121-122: search the clouds set by setInputSource / setInputTarget (radiusSearch takes a SQUARED radius)
  std::shared_ptr<nanoflann::KdTreeFLANN<PointSource>> source_kdtree_;
  std::shared_ptr<nanoflann::KdTreeFLANN<PointTarget>> target_kdtree_;

 private:
  template <typename CloudPtr>
  void upload(const CloudPtr& cloud, b200reg_host::DeviceCloud* slot) {
    destroy(slot);
    if (!cloud || cloud->size() == 0) return;
    using P = typename std::remove_reference<decltype(cloud->points[0])>::type;
    *slot = b200reg_host::make_device_cloud(reinterpret_cast<const float*>(cloud->points.data()), cloud->size(), sizeof(P));
  }
  void fetch_lm_trace(b200reg_ctx* ctx) {
    int64_t off[2] = {0, 0};
    b200reg_lm_trace(ctx, off, 0, nullptr);  // B200REG_ESTATE unless the pair made no trial: off[1] is the count either way
    lm_trace_.resize(off[1]);
    const int rc = b200reg_lm_trace(ctx, off, lm_trace_.size(), lm_trace_.data());
    if (rc != 0) {
      std::fprintf(stderr, "b200reg: lm_trace failed (%d): %s\n", rc, b200reg_last_error());
      lm_trace_.clear();
    }
  }
  void fetch_residuals(b200reg_ctx* ctx) {
    int64_t off[2] = {0, 0};
    b200reg_residuals(ctx, off, 0, nullptr, nullptr);  // B200REG_ESTATE unless the source is empty: off[1] is the count either way
    residuals_.nn.resize(off[1]);
    residuals_.d2.resize(off[1]);
    const int rc = b200reg_residuals(ctx, off, residuals_.d2.size(), residuals_.nn.data(), residuals_.d2.data());
    if (rc != 0) {
      std::fprintf(stderr, "b200reg: residuals failed (%d): %s\n", rc, b200reg_last_error());
      residuals_.nn.clear();
      residuals_.d2.clear();
    }
  }
  // what LsqRegistration prints with lm_debug_print_ (lsq_registration_impl.hpp:95-99, 183-189), one row per trial
  void print_lm_trace() const {
    std::cout << "********************************************" << std::endl;
    std::cout << "***************** optimize *****************" << std::endl;
    std::cout << "********************************************" << std::endl;
    char line[160];
    for (const b200reg_lm_trial& r : lm_trace_) {
      if (r.trial == 0) {
        std::snprintf(line, sizeof(line), "--- LM optimization ---\n%5s %15s %15s %15s %15s %15s %5s\n", "i", "y0", "yi", "rho",
                      "lambda", "|delta|", "dec");
        std::cout << line;
      }
      double dn = 0;
      for (int k = 0; k < 6; k++) dn += r.d[k] * r.d[k];
      std::snprintf(line, sizeof(line), "%5d %15g %15g %15g %15g %15g %5c", r.trial, r.y0, r.yi, r.rho, r.lambda, std::sqrt(dn),
                    r.rho > 0.0 ? 'x' : ' ');
      std::cout << line << std::endl;
    }
  }
  void destroy(b200reg_host::DeviceCloud* slot) { slot->reset(); }  // the device cloud goes when its last user (a tree) does
  void release() {
    destroy(&src_);
    destroy(&tgt_);
  }
  bool covariances(b200reg_cloud* cl, bool* ok) {
    if (!cl) return false;
    b200reg_cloud* a[1] = {cl};
    const int rc = b200reg_clouds_covariances_ex(b200reg_host::context(), 1, a, prm_.k_correspondences, prm_.regularization);
    if (rc != 0) std::fprintf(stderr, "b200reg: covariances failed (%d): %s\n", rc, b200reg_last_error());
    *ok = rc == 0;
    return true;  // the reference returns true unconditionally (nano_gicp_impl.hpp:356)
  }
  CovVector fetch_covs(b200reg_cloud* cl, bool* ok) {
    CovVector out;
    if (!cl) return out;
    if (!*ok) covariances(cl, ok);
    const size_t n = b200reg_cloud_size(cl);
    std::vector<double> c9(9 * n);
    b200reg_get_covariances(b200reg_host::context(), cl, c9.data());
    out.resize(n);
    for (size_t i = 0; i < n; i++) {
      Cov m;
      for (int r = 0; r < 4; r++)
        for (int c = 0; c < 4; c++) m(r, c) = (r < 3 && c < 3) ? c9[9 * i + 3 * r + c] : 0.0;
      out[i] = m;
    }
    return out;
  }
  void push_covs(b200reg_cloud* cl, const CovVector& covs, bool* ok) {
    if (!cl) return;
    if (covs.size() != b200reg_cloud_size(cl)) {
      std::fprintf(stderr, "b200reg: %zu covariances for a cloud of %zu points\n", covs.size(), b200reg_cloud_size(cl));
      return;
    }
    std::vector<double> c9(9 * covs.size());
    for (size_t i = 0; i < covs.size(); i++)
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) c9[9 * i + 3 * r + c] = covs[i](r, c);
    const int rc = b200reg_set_covariances(b200reg_host::context(), cl, c9.data(), covs.size());
    if (rc != 0) std::fprintf(stderr, "b200reg: set_covariances failed (%d): %s\n", rc, b200reg_last_error());
    *ok = rc == 0;
  }

  b200reg_gicp_params prm_;
  b200reg_result res_{};
  PointCloudSourceConstPtr input_;
  PointCloudTargetConstPtr target_;
  b200reg_host::DeviceCloud src_, tgt_;
  bool src_cov_ok_ = false, tgt_cov_ok_ = false, converged_ = false;
  bool lm_debug_print_ = false;  // lsq_registration.hpp:92
  std::vector<b200reg_lm_trial> lm_trace_;
  Residuals residuals_;
  std::array<float, 16> final_;
  Matrix6d final_hessian_;
  int ransac_iterations_ = 0;
  double euclidean_fitness_epsilon_ = 0, ransac_threshold_ = 0;
};

}  // namespace nano_gicp
