// fast_gicp::FastVGICPCuda -- mirror of the reference's include/fast_gicp/gicp/fast_vgicp_cuda.hpp:27-85 and
// impl/fast_vgicp_cuda_impl.hpp:22-178 on top of the C ABI (include/vgicp_b200.h) instead of FastVGICPCudaCore.
// Same public interface, same state machine (pointer-equality caching, swap, clear), same quirks (SURVEY Q1-Q3, Q7).
#pragma once
#include <stdexcept>

#include "../../../../include/vgicp_b200.h"
#include "lsq_registration.hpp"

namespace fast_gicp {

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

  int k_correspondences_;
  double voxel_resolution_;
  RegularizationMethod regularization_method_;
  NearestNeighborMethod neighbor_search_method_;
  vgicp_handle vgicp_cuda_ = nullptr;
};

}  // namespace fast_gicp
