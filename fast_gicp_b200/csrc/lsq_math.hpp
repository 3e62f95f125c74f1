// lsq_math.hpp -- small fixed-size double-precision helpers for the host side of the registration loop:
// SE(3) exponential (reference include/fast_gicp/so3/so3.hpp:58-104), 6x6 pivoted LDL^T solve (stands in for
// Eigen::LDLT<Matrix<double,6,6>>, lsq_registration_impl.hpp:111,134), isometry product, convergence test
// (lsq_registration_impl.hpp:82-91).  Header-only, no dependencies (Eigen is not available in this environment).
#pragma once
#include <math.h>

namespace vgicp {

// 4x4 column-major isometry image, identical to Eigen::Isometry3d::data()
struct Iso3d {
  double m[16];
  double& operator()(int r, int c) { return m[c * 4 + r]; }
  double operator()(int r, int c) const { return m[c * 4 + r]; }
};

inline Iso3d iso_identity() {
  Iso3d T;
  for (int i = 0; i < 16; i++) T.m[i] = (i % 5 == 0) ? 1.0 : 0.0;
  return T;
}

// delta * x0 for affine 4x4 (last row 0 0 0 1)
inline Iso3d iso_mul(const Iso3d& A, const Iso3d& B) {
  Iso3d C;
  for (int c = 0; c < 4; c++)
    for (int r = 0; r < 3; r++) {
      double s = A(r, 0) * B(0, c) + A(r, 1) * B(1, c) + A(r, 2) * B(2, c);
      if (c == 3) s += A(r, 3);
      C(r, c) = s;
    }
  C(3, 0) = C(3, 1) = C(3, 2) = 0.0;
  C(3, 3) = 1.0;
  return C;
}

// so3.hpp:80-104 (rotation-first 6-vector [omega, v]); so3_exp :58-77; Eigen's Quaternion::toRotationMatrix
inline Iso3d se3_exp(const double* a) {
  const double ox = a[0], oy = a[1], oz = a[2];
  const double theta_sq = ox * ox + oy * oy + oz * oz;
  const double theta = sqrt(theta_sq);
  double imag_factor, real_factor;
  if (theta_sq < 1e-10) {
    const double theta_quad = theta_sq * theta_sq;
    imag_factor = 0.5 - 1.0 / 48.0 * theta_sq + 1.0 / 3840.0 * theta_quad;
    real_factor = 1.0 - 1.0 / 8.0 * theta_sq + 1.0 / 384.0 * theta_quad;
  } else {
    const double half_theta = 0.5 * theta;
    imag_factor = sin(half_theta) / theta;
    real_factor = cos(half_theta);
  }
  const double qw = real_factor, qx = imag_factor * ox, qy = imag_factor * oy, qz = imag_factor * oz;
  const double tx = 2.0 * qx, ty = 2.0 * qy, tz = 2.0 * qz;
  const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  Iso3d T = iso_identity();
  T(0, 0) = 1.0 - (tyy + tzz); T(0, 1) = txy - twz;         T(0, 2) = txz + twy;
  T(1, 0) = txy + twz;         T(1, 1) = 1.0 - (txx + tzz); T(1, 2) = tyz - twx;
  T(2, 0) = txz - twy;         T(2, 1) = tyz + twx;         T(2, 2) = 1.0 - (txx + tyy);
  // V = I + (1-cos)/th^2 * Om + (th - sin)/th^3 * Om^2   (V = R when theta < 1e-10)
  double V[3][3];
  if (theta < 1e-10) {
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) V[r][c] = T(r, c);
  } else {
    const double Om[3][3] = {{0.0, -oz, oy}, {oz, 0.0, -ox}, {-oy, ox, 0.0}};
    const double c1 = (1.0 - cos(theta)) / theta_sq;
    const double c2 = (theta - sin(theta)) / (theta_sq * theta);
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        const double om2 = Om[r][0] * Om[0][c] + Om[r][1] * Om[1][c] + Om[r][2] * Om[2][c];
        V[r][c] = (r == c ? 1.0 : 0.0) + c1 * Om[r][c] + c2 * om2;
      }
  }
  for (int r = 0; r < 3; r++) T(r, 3) = V[r][0] * a[3] + V[r][1] * a[4] + V[r][2] * a[5];
  return T;
}

// Solve A x = rhs, A symmetric N x N column-major; LDL^T with diagonal pivoting.  N = 6: the pose step; N = 12: pose and twist
// (vgicp_align_ct).
template <int N>
inline void ldlt_solve(const double* A_in, const double* rhs, double* x) {
  double A[N][N];
  int perm[N];
  for (int r = 0; r < N; r++) {
    perm[r] = r;
    for (int c = 0; c < N; c++) A[r][c] = A_in[c * N + r];
  }
  for (int k = 0; k < N; k++) {
    int p = k;
    double best = fabs(A[k][k]);
    for (int i = k + 1; i < N; i++)
      if (fabs(A[i][i]) > best) { best = fabs(A[i][i]); p = i; }
    if (p != k) {
      for (int j = 0; j < N; j++) { double t = A[k][j]; A[k][j] = A[p][j]; A[p][j] = t; }
      for (int j = 0; j < N; j++) { double t = A[j][k]; A[j][k] = A[j][p]; A[j][p] = t; }
      int t = perm[k]; perm[k] = perm[p]; perm[p] = t;
    }
    const double d = A[k][k];
    if (d == 0.0) continue;
    for (int i = k + 1; i < N; i++) A[i][k] /= d;
    for (int j = k + 1; j < N; j++)
      for (int i = j; i < N; i++) {
        A[i][j] -= A[i][k] * d * A[j][k];
        A[j][i] = A[i][j];
      }
  }
  double y[N];
  for (int i = 0; i < N; i++) y[i] = rhs[perm[i]];
  for (int i = 0; i < N; i++)
    for (int j = 0; j < i; j++) y[i] -= A[i][j] * y[j];
  for (int i = 0; i < N; i++) y[i] = (A[i][i] != 0.0) ? y[i] / A[i][i] : 0.0;
  for (int i = N - 1; i >= 0; i--)
    for (int j = i + 1; j < N; j++) y[i] -= A[j][i] * y[j];
  for (int i = 0; i < N; i++) x[perm[i]] = y[i];
}

// lsq_registration_impl.hpp:82-91
inline bool is_converged(const Iso3d& delta, double rotation_epsilon, double transformation_epsilon) {
  double mr = 0.0, mt = 0.0;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      const double v = fabs(delta(r, c) - (r == c ? 1.0 : 0.0)) / rotation_epsilon;
      if (v > mr) mr = v;
    }
  for (int r = 0; r < 3; r++) {
    const double v = fabs(delta(r, 3)) / transformation_epsilon;
    if (v > mt) mt = v;
  }
  return (mr > mt ? mr : mt) < 1.0;
}

}  // namespace vgicp
