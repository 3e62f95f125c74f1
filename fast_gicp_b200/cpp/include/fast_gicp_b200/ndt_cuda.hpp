// fast_gicp::NDTCuda -- mirror of the reference's include/fast_gicp/ndt/ndt_cuda.hpp:22-71 and impl/ndt_cuda_impl.hpp:11-90 on the C
// ABI (the NDT problems of the same handle, include/vgicp_b200.h "NDT").
#pragma once
#include <stdexcept>

#include "../../../../include/vgicp_b200.h"
#include "lsq_registration.hpp"

namespace fast_gicp {

enum class NDTDistanceMode { P2D, D2D };  // ndt_settings.hpp:6

template <typename PointSource, typename PointTarget>
class NDTCuda : public LsqRegistration<PointSource, PointTarget> {
public:
  using Scalar = float;
  using Base = LsqRegistration<PointSource, PointTarget>;
  using Matrix4 = typename Base::Matrix4;
  using PointCloudSource = typename Base::PointCloudSource;
  using PointCloudSourceConstPtr = typename Base::PointCloudSourceConstPtr;
  using PointCloudTargetConstPtr = typename Base::PointCloudTargetConstPtr;
  using Ptr = std::shared_ptr<NDTCuda<PointSource, PointTarget>>;

protected:
  using Base::input_;
  using pcl::Registration<PointSource, PointTarget, Scalar>::target_;

public:
  explicit NDTCuda(int device = 0) : Base() {  // ndt_cuda_impl.hpp:11-14 + NDTCudaCore ctor ndt_cuda.cu:13-23
    this->reg_name_ = "NDTCuda";
    if (vgicp_create(device, &ndt_cuda_) != VGICP_OK) throw std::runtime_error("NDTCuda: vgicp_create failed (a CUDA device with an sm_90a image is required)");
    check(vgicp_set_problem(ndt_cuda_, 2));                                     // distance_mode = D2D
    check(vgicp_set_neighbor_search_method(ndt_cuda_, VGICP_DIRECT7, 0.0));     // DIRECT7
  }
  virtual ~NDTCuda() override { vgicp_destroy(ndt_cuda_); }
  NDTCuda(const NDTCuda&) = delete;
  NDTCuda& operator=(const NDTCuda&) = delete;

  void setDistanceMode(NDTDistanceMode mode) { check(vgicp_set_problem(ndt_cuda_, mode == NDTDistanceMode::P2D ? 1 : 2)); }
  void setResolution(double resolution) { check(vgicp_set_resolution(ndt_cuda_, resolution)); }
  void setNeighborSearchMethod(NeighborSearchMethod method, double radius = -1.0) { check(vgicp_set_neighbor_search_method(ndt_cuda_, static_cast<int>(method), radius)); }

  virtual void swapSourceAndTarget() override {
    check(vgicp_swap_source_and_target(ndt_cuda_));
    input_.swap(target_);
  }
  virtual void clearSource() override { input_.reset(); }
  virtual void clearTarget() override { target_.reset(); }

  virtual void setInputSource(const PointCloudSourceConstPtr& cloud) override {
    if (cloud == input_) return;
    pcl::Registration<PointSource, PointTarget, Scalar>::setInputSource(cloud);
    check(vgicp_set_source_cloud(ndt_cuda_, cloud->empty() ? nullptr : &cloud->points[0].x, cloud->size(), sizeof(PointSource)));
  }
  virtual void setInputTarget(const PointCloudTargetConstPtr& cloud) override {
    if (cloud == target_) return;
    pcl::Registration<PointSource, PointTarget, Scalar>::setInputTarget(cloud);
    check(vgicp_set_target_cloud(ndt_cuda_, cloud->empty() ? nullptr : &cloud->points[0].x, cloud->size(), sizeof(PointTarget)));
  }
  vgicp_handle handle() const { return ndt_cuda_; }

protected:
  virtual void computeTransformation(PointCloudSource& output, const Matrix4& guess) override {  // ndt_cuda_impl.hpp:70-74
    multiPrelude();
    Base::computeTransformation(output, guess);
  }
  virtual vgicp_handle multiHandle() const override { return ndt_cuda_; }
  virtual void multiPrelude() override { check(vgicp_ndt_create_voxelmaps(ndt_cuda_)); }
  virtual void transformSource(PointCloudSource& output, const Matrix4& T) override {
    output = *input_;
    if (output.empty()) return;
    double Td[16];
    for (int i = 0; i < 16; i++) Td[i] = static_cast<double>(T.v[i]);
    check(vgicp_transform_source(ndt_cuda_, Td, &output.points[0].x, output.size(), sizeof(PointSource)));
  }
  virtual double linearize(const Isometry3d& trans, Matrix6d* H = nullptr, Vector6d* b = nullptr) override {  // :77-80
    check(vgicp_update_correspondences(ndt_cuda_, trans.m));
    double err = 0.0;
    check(vgicp_compute_error(ndt_cuda_, trans.m, H ? H->data() : nullptr, b ? b->data() : nullptr, &err));
    return err;
  }
  virtual double compute_error(const Isometry3d& trans) override {  // :83-85
    double err = 0.0;
    check(vgicp_compute_error(ndt_cuda_, trans.m, nullptr, nullptr, &err));
    return err;
  }

private:
  void check(int rc) const {
    if (rc != VGICP_OK) throw std::runtime_error(std::string("NDTCuda: ") + vgicp_last_error(ndt_cuda_));
  }
  vgicp_handle ndt_cuda_ = nullptr;
};

}  // namespace fast_gicp
