// fast_gicp::LsqRegistration -- host-side optimiser, mirror of the reference's
// include/fast_gicp/gicp/lsq_registration.hpp:16-85 and impl/lsq_registration_impl.hpp:9-168 (same members, same LM /
// Gauss-Newton logic in double); the 6x6 solve and SE(3) exponential come from csrc/lsq_math.hpp instead of Eigen.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../../include/vgicp_b200.h"
#include "../../../csrc/lsq_math.hpp"
#include "compat.hpp"
#include "gicp_settings.hpp"

namespace fast_gicp {

using Matrix6d = Eigen::Matrix<double, 6, 6>;
using Vector6d = Eigen::Matrix<double, 6, 1>;
using Isometry3d = vgicp::Iso3d;  // 4x4 column-major double, memory image of Eigen::Isometry3d

template <typename PointSource, typename PointTarget>
class LsqRegistration : public pcl::Registration<PointSource, PointTarget, float> {
public:
  using Scalar = float;
  using Base = pcl::Registration<PointSource, PointTarget, Scalar>;
  using Matrix4 = typename Base::Matrix4;
  using PointCloudSource = typename Base::PointCloudSource;
  using PointCloudSourcePtr = typename PointCloudSource::Ptr;
  using PointCloudSourceConstPtr = typename PointCloudSource::ConstPtr;
  using PointCloudTarget = typename Base::PointCloudTarget;
  using PointCloudTargetPtr = typename PointCloudTarget::Ptr;
  using PointCloudTargetConstPtr = typename PointCloudTarget::ConstPtr;
  using Ptr = std::shared_ptr<LsqRegistration<PointSource, PointTarget>>;

protected:
  using Base::converged_;
  using Base::final_transformation_;
  using Base::input_;
  using Base::max_iterations_;
  using Base::nr_iterations_;
  using Base::transformation_epsilon_;

public:
  LsqRegistration() {  // lsq_registration_impl.hpp:9-22
    this->reg_name_ = "LsqRegistration";
    max_iterations_ = 64;
    rotation_epsilon_ = 2e-3;
    transformation_epsilon_ = 5e-4;
    lsq_optimizer_type_ = LSQ_OPTIMIZER_TYPE::LevenbergMarquardt;
    lm_debug_print_ = false;
    lm_max_iterations_ = 10;
    lm_init_lambda_factor_ = 1e-9;
    lm_lambda_ = -1.0;
    final_hessian_.setIdentity();
  }
  virtual ~LsqRegistration() {}

  void setRotationEpsilon(double eps) { rotation_epsilon_ = eps; }
  void setInitialLambdaFactor(double f) { lm_init_lambda_factor_ = f; }
  void setDebugPrint(bool p) { lm_debug_print_ = p; }
  void setOptimizerType(LSQ_OPTIMIZER_TYPE t) { lsq_optimizer_type_ = t; }  // (protected member in the reference)
  const Matrix6d& getFinalHessian() const { return final_hessian_; }

  double evaluateCost(const Eigen::Matrix4f& relative_pose, Matrix6d* H = nullptr, Vector6d* b = nullptr) {  // :48-50
    Isometry3d T;
    for (int i = 0; i < 16; i++) T.m[i] = static_cast<double>(relative_pose.v[i]);
    return this->linearize(T, H, b);
  }

  virtual void swapSourceAndTarget() {}
  virtual void clearSource() {}
  virtual void clearTarget() {}

  // Multi-hypothesis alignment (not in the reference): one registration of the source per initial guess, the evaluations of all
  // hypotheses sharing launches on the device (vgicp_align_multi).  T_out[i] and converged_out[i] are the final transformation and
  // convergence flag of that registration; getFinalTransformation(), hasConverged() and the final Hessian are left alone.
  void alignMulti(const std::vector<Matrix4>& guesses, std::vector<Matrix4>& T_out, std::vector<bool>& converged_out) {
    T_out.clear();
    converged_out.clear();
    if (!input_ || !this->target_ || guesses.empty()) return;  // (pcl's align returns without inputs)
    multiPrelude();
    const int n = static_cast<int>(guesses.size());
    std::vector<double> g(16 * guesses.size());
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 16; k++) g[16 * i + k] = static_cast<double>(guesses[i].v[k]);
    const vgicp_lsq_params P = lsqParams();
    std::vector<vgicp_align_result> r(guesses.size());
    multiCheck(vgicp_align_multi(multiHandle(), g.data(), n, &P, r.data()));
    T_out.resize(guesses.size());
    converged_out.resize(guesses.size());
    for (int i = 0; i < n; i++) {
      for (int k = 0; k < 16; k++) T_out[i].v[k] = static_cast<float>(r[i].T[k]);
      converged_out[i] = r[i].converged != 0;
    }
  }

  // Scores poses in one launch: err[i] is the error of linearize(poses[i]) and n_corr[i] its number of (source point, voxel)
  // correspondences (vgicp_evaluate_poses).  A pose without overlap scores 0 with no correspondences.
  void evaluatePoses(const std::vector<Eigen::Matrix4d>& poses, std::vector<double>& err, std::vector<int64_t>& n_corr) {
    err.clear();
    n_corr.clear();
    if (!input_ || !this->target_ || poses.empty()) return;
    multiPrelude();
    std::vector<double> T(16 * poses.size());
    for (size_t i = 0; i < poses.size(); i++) std::memcpy(&T[16 * i], poses[i].data(), 16 * sizeof(double));
    err.resize(poses.size());
    n_corr.resize(poses.size());
    multiCheck(vgicp_evaluate_poses(multiHandle(), T.data(), static_cast<int>(poses.size()), err.data(), nullptr, nullptr, n_corr.data()));
  }

protected:
  // this optimiser's settings for the optimisers inside the library (vgicp_align_multi, vgicp_align_ct)
  vgicp_lsq_params lsqParams() const {
    vgicp_lsq_params P;
    vgicp_lsq_default_params(&P);
    P.max_iterations = max_iterations_;
    P.rotation_epsilon = rotation_epsilon_;
    P.transformation_epsilon = transformation_epsilon_;
    P.use_gauss_newton = lsq_optimizer_type_ == LSQ_OPTIMIZER_TYPE::GaussNewton ? 1 : 0;
    P.lm_max_iterations = lm_max_iterations_;
    P.lm_init_lambda_factor = lm_init_lambda_factor_;
    return P;
  }
  // the device handle and the computeTransformation prelude of a subclass, for alignMulti / evaluatePoses
  virtual vgicp_handle multiHandle() const = 0;
  virtual void multiPrelude() {}
  void multiCheck(int rc) const {
    if (rc != VGICP_OK) throw std::runtime_error(this->reg_name_ + ": " + vgicp_last_error(multiHandle()));
  }

  virtual void transformSource(PointCloudSource& output, const Matrix4& T) {  // pcl::transformPointCloud (:78)
    output = *input_;
    for (auto& p : output.points) {
      const float x = p.x, y = p.y, z = p.z;
      p.x = T(0, 0) * x + T(0, 1) * y + T(0, 2) * z + T(0, 3);
      p.y = T(1, 0) * x + T(1, 1) * y + T(1, 2) * z + T(1, 3);
      p.z = T(2, 0) * x + T(2, 1) * y + T(2, 2) * z + T(2, 3);
    }
  }

  virtual void computeTransformation(PointCloudSource& output, const Matrix4& guess) override {  // :53-79
    Isometry3d x0;
    for (int i = 0; i < 16; i++) x0.m[i] = static_cast<double>(guess.v[i]);
    lm_lambda_ = -1.0;
    converged_ = false;
    for (int i = 0; i < max_iterations_ && !converged_; i++) {
      nr_iterations_ = i;
      Isometry3d delta;
      if (!step_optimize(x0, delta)) {
        std::cerr << "lm not converged!!" << std::endl;
        break;
      }
      converged_ = is_converged(delta);
    }
    for (int i = 0; i < 16; i++) final_transformation_.v[i] = static_cast<float>(x0.m[i]);
    transformSource(output, final_transformation_);
  }

  bool is_converged(const Isometry3d& delta) const { return vgicp::is_converged(delta, rotation_epsilon_, transformation_epsilon_); }  // :82-91

  virtual double linearize(const Isometry3d& trans, Matrix6d* H = nullptr, Vector6d* b = nullptr) = 0;
  virtual double compute_error(const Isometry3d& trans) = 0;

  bool step_optimize(Isometry3d& x0, Isometry3d& delta) {  // :94-103
    return lsq_optimizer_type_ == LSQ_OPTIMIZER_TYPE::GaussNewton ? step_gn(x0, delta) : step_lm(x0, delta);
  }

  bool step_gn(Isometry3d& x0, Isometry3d& delta) {  // :106-120
    Matrix6d H;
    Vector6d b;
    linearize(x0, &H, &b);
    double nb[6], d[6];
    for (int i = 0; i < 6; i++) nb[i] = -b[i];
    vgicp::ldlt_solve<6>(H.data(), nb, d);
    delta = vgicp::se3_exp(d);
    x0 = vgicp::iso_mul(delta, x0);
    final_hessian_ = H;
    return true;
  }

  bool step_lm(Isometry3d& x0, Isometry3d& delta) {  // :123-168
    Matrix6d H;
    Vector6d b;
    double y0 = linearize(x0, &H, &b);
    if (lm_lambda_ < 0.0) {
      double mx = 0.0;
      for (int i = 0; i < 6; i++) mx = std::fmax(mx, std::fabs(H(i, i)));
      lm_lambda_ = lm_init_lambda_factor_ * mx;
    }
    double nu = 2.0;
    for (int i = 0; i < lm_max_iterations_; i++) {
      Matrix6d Hl = H;
      for (int q = 0; q < 6; q++) Hl(q, q) += lm_lambda_;
      double nb[6], d[6];
      for (int q = 0; q < 6; q++) nb[q] = -b[q];
      vgicp::ldlt_solve<6>(Hl.data(), nb, d);
      delta = vgicp::se3_exp(d);
      Isometry3d xi = vgicp::iso_mul(delta, x0);
      double yi = compute_error(xi);
      double den = 0.0, dn = 0.0;
      for (int q = 0; q < 6; q++) { den += d[q] * (lm_lambda_ * d[q] - b[q]); dn += d[q] * d[q]; }
      double rho = (y0 - yi) / den;
      if (lm_debug_print_) {
        if (i == 0) std::printf("--- LM optimization ---\n%5s %15s %15s %15s %15s %15s %5s\n", "i", "y0", "yi", "rho", "lambda", "|delta|", "dec");
        std::printf("%5d %15g %15g %15g %15g %15g %5c\n", i, y0, yi, rho, lm_lambda_, std::sqrt(dn), rho > 0.0 ? 'x' : ' ');
      }
      if (rho < 0) {
        if (is_converged(delta)) return true;
        lm_lambda_ = nu * lm_lambda_;
        nu = 2 * nu;
        continue;
      }
      x0 = xi;
      lm_lambda_ = lm_lambda_ * std::fmax(1.0 / 3.0, 1 - std::pow(2 * rho - 1, 3));
      final_hessian_ = H;
      return true;
    }
    return false;
  }

protected:
  double rotation_epsilon_;
  LSQ_OPTIMIZER_TYPE lsq_optimizer_type_;
  int lm_max_iterations_;
  double lm_init_lambda_factor_;
  double lm_lambda_;
  bool lm_debug_print_;
  Matrix6d final_hessian_;
};

}  // namespace fast_gicp
