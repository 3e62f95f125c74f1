// fast_gicp::FastVGICPCuda -- mirror of the reference's include/fast_gicp/gicp/fast_vgicp_cuda.hpp:27-85 and
// impl/fast_vgicp_cuda_impl.hpp:22-178 on top of the C ABI (include/vgicp_b200.h) instead of FastVGICPCudaCore.
// Same public interface, same state machine (pointer-equality caching, swap, clear), same quirks (SURVEY Q1-Q3, Q7).
#pragma once
#include <stdexcept>

#include "../../../../include/vgicp_b200.h"
#include "lsq_registration.hpp"

namespace fast_gicp {

// Robust kernel of the Mahalanobis residual (an extension, not in the reference): VGICP_ROBUST_* of include/vgicp_b200.h
enum class RobustKernel { NONE, HUBER, CAUCHY, GEMAN_MCCLURE };

template <typename PointSource, typename PointTarget>
class FastVGICPCuda : public LsqRegistration<PointSource, PointTarget> {
public:
  using Scalar = float;
  using Base = LsqRegistration<PointSource, PointTarget>;
  using Matrix4 = typename Base::Matrix4;
  using PointCloudSource = typename Base::PointCloudSource;
  using PointCloudSourceConstPtr = typename Base::PointCloudSourceConstPtr;
  using PointCloudTarget = typename Base::PointCloudTarget;
  using PointCloudTargetConstPtr = typename Base::PointCloudTargetConstPtr;
  using Ptr = std::shared_ptr<FastVGICPCuda<PointSource, PointTarget>>;

protected:
  using Base::input_;
  using pcl::Registration<PointSource, PointTarget, Scalar>::target_;

public:
  explicit FastVGICPCuda(int device = 0) : Base() {  // impl:22-32
    this->reg_name_ = "FastVGICPCuda";
    k_correspondences_ = 20;
    voxel_resolution_ = 1.0;
    regularization_method_ = RegularizationMethod::PLANE;
    neighbor_search_method_ = NearestNeighborMethod::CPU_PARALLEL_KDTREE;
    int rc = vgicp_create(device, &vgicp_cuda_);
    if (rc != VGICP_OK) throw std::runtime_error("FastVGICPCuda: vgicp_create failed (a CUDA device with an sm_90a image is required; there is no CPU fallback)");
    check(vgicp_set_resolution(vgicp_cuda_, voxel_resolution_));
    check(vgicp_set_kernel_params(vgicp_cuda_, 0.5, 3.0));
  }
  virtual ~FastVGICPCuda() override { vgicp_destroy(vgicp_cuda_); }
  FastVGICPCuda(const FastVGICPCuda&) = delete;
  FastVGICPCuda& operator=(const FastVGICPCuda&) = delete;

  void setCorrespondenceRandomness(int) {}                                                     // impl:38 (empty in the reference)
  void setResolution(double resolution) { check(vgicp_set_resolution(vgicp_cuda_, resolution)); }  // impl:41-43
  void setKernelWidth(double kernel_width, double max_dist = -1.0) {                           // impl:46-51
    if (max_dist <= 0.0) max_dist = kernel_width * 5.0;
    check(vgicp_set_kernel_params(vgicp_cuda_, kernel_width, max_dist));
  }
  void setRegularizationMethod(RegularizationMethod method) { regularization_method_ = method; }
  void setNeighborSearchMethod(NeighborSearchMethod method, double radius = -1.0) {            // impl:59-61
    check(vgicp_set_neighbor_search_method(vgicp_cuda_, static_cast<int>(method), radius));
  }
  void setNearestNeighborSearchMethod(NearestNeighborMethod method) { neighbor_search_method_ = method; }
  // scale = delta in Mahalanobis units (ignored for NONE); a setting of the core, kept across input changes and swaps
  void setRobustKernel(RobustKernel kind, double scale = 1.0) { check(vgicp_set_robust_kernel(vgicp_cuda_, static_cast<int>(kind), scale)); }

  // Local map for scan-to-map odometry (an extension).  Afterwards the target on the device is no longer the cloud given to
  // setInputTarget: target_ becomes a fresh empty placeholder, so align still has a target and setInputTarget(that cloud) reloads it.
  void appendSourceToTarget(const Matrix4& T) {  // T: e.g. getFinalTransformation()
    double Td[16];
    for (int i = 0; i < 16; i++) Td[i] = static_cast<double>(T.v[i]);
    checkStrict(vgicp_append_source_to_target(vgicp_cuda_, Td));
    target_ = pcl::make_shared<PointCloudTarget>();
  }
  // keep the target points within `radius` of `center`, then at most the newest `max_points` of them (0 = no cap)
  void cropTarget(const double center[3], double radius, size_t max_points = 0) {
    checkStrict(vgicp_crop_target(vgicp_cuda_, center, radius, max_points));
    target_ = pcl::make_shared<PointCloudTarget>();
  }
  // keep at most `max_points_per_voxel` target points per cell of a `leaf_size` grid, the oldest (call after appendSourceToTarget)
  void thinTarget(double leaf_size, int max_points_per_voxel) {
    checkStrict(vgicp_thin_target(vgicp_cuda_, leaf_size, max_points_per_voxel));
    target_ = pcl::make_shared<PointCloudTarget>();
  }
  // remove the target points the current source, placed by T, sees through (call after align, before appendSourceToTarget);
  // params: NULL = vgicp_carve_default_params; returns the number of points removed
  size_t carveTarget(const Matrix4& T, const vgicp_carve_params* params = nullptr) {
    double Td[16];
    for (int i = 0; i < 16; i++) Td[i] = static_cast<double>(T.v[i]);
    vgicp_carve_params P;
    if (params) P = *params; else vgicp_carve_default_params(&P);
    size_t removed = 0;
    checkStrict(vgicp_carve_target(vgicp_cuda_, Td, &P, &removed));
    target_ = pcl::make_shared<PointCloudTarget>();
    return removed;
  }

  // Motion compensation (an extension): every source point becomes Exp((t_i - t_ref) twist) p_i, the point in the sensor frame at
  // t_ref (include/vgicp_b200.h), then the source covariances are recomputed as setInputSource computes them.  t: n float
  // timestamps stride_bytes apart, e.g. &cloud->points[0].time and sizeof(PointT); twist = [omega, v] per time unit.  Afterwards
  // input_ is a copy of the cloud given to setInputSource (its fields stay for align's output), so setInputSource(that cloud)
  // reloads the raw points.
  void deskewSource(const float* t, size_t n, size_t stride_bytes, const double twist[6], double t_ref = 0.0) {
    if (!input_) throw std::runtime_error("FastVGICPCuda: deskewSource needs an input source");
    checkStrict(vgicp_deskew_source(vgicp_cuda_, t, n, stride_bytes, twist, t_ref));
    sourceCovariances();
    input_ = pcl::make_shared<PointCloudSource>(*input_);
  }
  // deskewSource with the timestamps and t_ref stored by setSourceTimestamps (no upload): the same points, the same state after
  void deskewSourceStored(const double twist[6]) {
    if (!input_) throw std::runtime_error("FastVGICPCuda: deskewSourceStored needs an input source");
    checkStrict(vgicp_deskew_source_stored(vgicp_cuda_, twist));
    sourceCovariances();
    input_ = pcl::make_shared<PointCloudSource>(*input_);
  }

  // Continuous-time registration (an extension): the pose at t_ref and the sweep's body twist estimated together
  // (vgicp_align_ct, include/vgicp_b200.h).  setSourceTimestamps takes one timestamp per point of the current source, as
  // deskewSource does; setInputSource with another cloud and swapSourceAndTarget drop them, deskewSource keeps them.
  void setSourceTimestamps(const float* t, size_t n, size_t stride_bytes, double t_ref = 0.0) {
    if (!input_) throw std::runtime_error("FastVGICPCuda: setSourceTimestamps needs an input source");
    checkStrict(vgicp_set_source_timestamps(vgicp_cuda_, t, n, stride_bytes, t_ref));
  }
  // Sets getFinalTransformation() (cast to float like align), hasConverged() and getFinalTwist(); `result` (optional) receives the
  // whole record (double pose, twist, the 12 x 12 system, counters).  The guess is cast to float, like align's.
  void alignCT(const Matrix4& guess, const double twist_guess[6], const double twist_prior[6], const double twist_weight[6], vgicp_align_ct_result* result = nullptr) {
    if (!input_ || !target_) throw std::runtime_error("FastVGICPCuda: alignCT needs an input source and target");
    multiPrelude();
    double g[16];
    for (int i = 0; i < 16; i++) g[i] = static_cast<double>(guess.v[i]);
    const vgicp_lsq_params P = this->lsqParams();
    vgicp_align_ct_result r;
    this->converged_ = false;
    checkStrict(vgicp_align_ct(vgicp_cuda_, g, twist_guess, twist_prior, twist_weight, &P, &r));
    if (r.lm_failed) std::cerr << "lm not converged!!" << std::endl;
    this->nr_iterations_ = r.nr_iterations;
    this->converged_ = r.converged != 0;
    for (int i = 0; i < 16; i++) this->final_transformation_.v[i] = static_cast<float>(r.T[i]);
    for (int j = 0; j < 6; j++) final_twist_[j] = r.twist[j];
    if (result) *result = r;
  }
  const double* getFinalTwist() const { return final_twist_; }

  // Multi-source alignment (an extension): each source registered against the current target with this object's k and
  // regularisation, the optimisers' evaluations sharing launches (vgicp_align_sources).  T_out[i] and converged_out[i] are what
  // setInputSource(sources[i]) + align(output, guesses[i]) would give (guesses empty: identity); the input source,
  // getFinalTransformation(), hasConverged() and the final Hessian are left alone.  RBF covariances are not batched: with
  // GPU_RBF_KERNEL selected this throws.
  void alignSources(const std::vector<PointCloudSourceConstPtr>& sources, const std::vector<Matrix4>& guesses, std::vector<Matrix4>& T_out, std::vector<bool>& converged_out) {
    T_out.clear();
    converged_out.clear();
    if (!target_) throw std::runtime_error("FastVGICPCuda: alignSources needs an input target");
    if (neighbor_search_method_ == NearestNeighborMethod::GPU_RBF_KERNEL)
      throw std::runtime_error("FastVGICPCuda: alignSources computes k-NN covariances; GPU_RBF_KERNEL is not available here");
    if (!guesses.empty() && guesses.size() != sources.size()) throw std::invalid_argument("FastVGICPCuda: alignSources needs one guess per source");
    if (sources.empty()) return;
    multiPrelude();
    const int n = static_cast<int>(sources.size());
    std::vector<const float*> xyz(sources.size());
    std::vector<size_t> sizes(sources.size());
    for (int i = 0; i < n; i++) {
      xyz[i] = sources[i]->empty() ? nullptr : &sources[i]->points[0].x;
      sizes[i] = sources[i]->size();
    }
    std::vector<double> g;
    if (!guesses.empty()) {
      g.resize(16 * guesses.size());
      for (int i = 0; i < n; i++)
        for (int k = 0; k < 16; k++) g[16 * i + k] = static_cast<double>(guesses[i].v[k]);
    }
    const vgicp_lsq_params P = this->lsqParams();
    std::vector<vgicp_align_result> r(sources.size());
    checkStrict(vgicp_align_sources(vgicp_cuda_, xyz.data(), sizes.data(), sizeof(PointSource), 0, k_correspondences_, static_cast<int>(regularization_method_),
                                    g.empty() ? nullptr : g.data(), n, &P, r.data()));
    T_out.resize(sources.size());
    converged_out.resize(sources.size());
    for (int i = 0; i < n; i++) {
      for (int k = 0; k < 16; k++) T_out[i].v[k] = static_cast<float>(r[i].T[k]);
      converged_out[i] = r[i].converged != 0;
    }
  }

  virtual void swapSourceAndTarget() override {  // impl:69-72
    check(vgicp_swap_source_and_target(vgicp_cuda_));
    input_.swap(target_);
  }
  virtual void clearSource() override { input_.reset(); }  // impl:75-77
  virtual void clearTarget() override { target_.reset(); }  // impl:80-82

  virtual void setInputSource(const PointCloudSourceConstPtr& cloud) override {  // impl:85-111
    if (cloud == input_) return;
    pcl::Registration<PointSource, PointTarget, Scalar>::setInputSource(cloud);
    check(vgicp_set_source_cloud(vgicp_cuda_, cloud->empty() ? nullptr : &cloud->points[0].x, cloud->size(), sizeof(PointSource)));
    sourceCovariances();
  }

  virtual void setInputTarget(const PointCloudTargetConstPtr& cloud) override {  // impl:114-141
    if (cloud == target_) return;
    pcl::Registration<PointSource, PointTarget, Scalar>::setInputTarget(cloud);
    check(vgicp_set_target_cloud(vgicp_cuda_, cloud->empty() ? nullptr : &cloud->points[0].x, cloud->size(), sizeof(PointTarget)));
    switch (neighbor_search_method_) {
      case NearestNeighborMethod::CPU_PARALLEL_KDTREE:
      case NearestNeighborMethod::GPU_BRUTEFORCE:
        check(vgicp_find_target_neighbors(vgicp_cuda_, k_correspondences_));
        check(vgicp_calculate_target_covariances(vgicp_cuda_, static_cast<int>(regularization_method_)));
        break;
      case NearestNeighborMethod::GPU_RBF_KERNEL:
        check(vgicp_calculate_target_covariances_rbf(vgicp_cuda_, static_cast<int>(regularization_method_)));
        break;
    }
    check(vgicp_create_target_voxelmap(vgicp_cuda_));
  }

  vgicp_handle handle() const { return vgicp_cuda_; }

protected:
  virtual void computeTransformation(PointCloudSource& output, const Matrix4& guess) override {  // impl:144-148
    multiPrelude();
    Base::computeTransformation(output, guess);
  }
  virtual vgicp_handle multiHandle() const override { return vgicp_cuda_; }
  virtual void multiPrelude() override { check(vgicp_set_resolution(vgicp_cuda_, voxel_resolution_)); }

  virtual void transformSource(PointCloudSource& output, const Matrix4& T) override {  // pcl::transformPointCloud on the device
    output = *input_;
    if (output.empty()) return;
    double Td[16];
    for (int i = 0; i < 16; i++) Td[i] = static_cast<double>(T.v[i]);
    check(vgicp_transform_source(vgicp_cuda_, Td, &output.points[0].x, output.size(), sizeof(PointSource)));
  }

  virtual double linearize(const Isometry3d& trans, Matrix6d* H = nullptr, Vector6d* b = nullptr) override {  // impl:170-173
    check(vgicp_update_correspondences(vgicp_cuda_, trans.m));
    double err = 0.0;
    check(vgicp_compute_error(vgicp_cuda_, trans.m, H ? H->data() : nullptr, b ? b->data() : nullptr, &err));
    return err;
  }
  virtual double compute_error(const Isometry3d& trans) override {  // impl:176-178
    double err = 0.0;
    check(vgicp_compute_error(vgicp_cuda_, trans.m, nullptr, nullptr, &err));
    return err;
  }

private:
  void check(int rc) const {
    if (rc != VGICP_OK && rc != VGICP_ERR_UNSUPPORTED) throw std::runtime_error(std::string("FastVGICPCuda: ") + vgicp_last_error(vgicp_cuda_));
    if (rc == VGICP_ERR_UNSUPPORTED) std::cerr << vgicp_last_error(vgicp_cuda_) << std::endl;  // the reference prints and carries on
  }
  void sourceCovariances() {  // impl:96-110
    switch (neighbor_search_method_) {
      case NearestNeighborMethod::CPU_PARALLEL_KDTREE:  // the same exact neighbour sets, computed on the GPU
      case NearestNeighborMethod::GPU_BRUTEFORCE:
        check(vgicp_find_source_neighbors(vgicp_cuda_, k_correspondences_));
        check(vgicp_calculate_source_covariances(vgicp_cuda_, static_cast<int>(regularization_method_)));
        break;
      case NearestNeighborMethod::GPU_RBF_KERNEL:
        check(vgicp_calculate_source_covariances_rbf(vgicp_cuda_, static_cast<int>(regularization_method_)));
        break;
    }
  }
  void checkStrict(int rc) const {  // the extensions have no reference behaviour to follow: every failure throws
    if (rc != VGICP_OK) throw std::runtime_error(std::string("FastVGICPCuda: ") + vgicp_last_error(vgicp_cuda_));
  }

  int k_correspondences_;
  double voxel_resolution_;
  RegularizationMethod regularization_method_;
  NearestNeighborMethod neighbor_search_method_;
  vgicp_handle vgicp_cuda_ = nullptr;
  double final_twist_[6] = {0, 0, 0, 0, 0, 0};
};

}  // namespace fast_gicp
