// vgicp_deskew.cuh -- kernel of vgicp_deskew_source: motion compensation of the source cloud from per-point timestamps and a
// constant body twist, in place on the device.  The arithmetic include/vgicp_b200.h documents is spelled as IEEE single
// operations (__f*_rn; this unit is compiled with contraction on), and the SE(3) exponential uses truncated Taylor series instead
// of sin / cos, so that numpy float32 rebuilds the same bytes and nothing depends on the CUDA math library.
#pragma once
#include <cuda_runtime.h>

namespace vgicp {

// Horner step h * q + c
__device__ __forceinline__ float horner_step(float h, float q, float c) { return __fadd_rn(__fmul_rn(h, q), c); }

// Point i becomes Exp(s xi) p_i with s = t_i - t_ref (rotation-first xi = [omega, nu], both already cast to float):
//   w = s omega, u = s nu, q = (w0 w0 + w1 w1) + w2 w2 (= theta^2),
//   A = sin(theta)/theta, B = (1 - cos(theta))/theta^2, C = (theta - sin(theta))/theta^3 as Horner polynomials in q,
//   K = [w]x, K2 = w w^T - q I, R = (I + A K) + B K2, V = (I + B K) + C K2 (entry by entry),
//   p'_j = ((R_j0 p0 + R_j1 p1) + R_j2 p2) + ((V_j0 u0 + V_j1 u1) + V_j2 u2).
// The coefficients are the float32 roundings of the series' coefficients; A keeps 7 terms, B and C 6, which keeps the truncation
// below 2^-24 relative for theta <= pi/2 (the host rejects larger rotations).
// One point: Exp(s xi) p.  Shared by k_deskew_points and the continuous-time evaluation kernels (vgicp_kernels.cuh), which
// must place a point exactly where vgicp_deskew_source would store it.
__device__ __forceinline__ float3 deskew_point(float4 p, float s, float o0, float o1, float o2, float n0, float n1, float n2) {
  const float w[3] = {__fmul_rn(s, o0), __fmul_rn(s, o1), __fmul_rn(s, o2)};
  const float u[3] = {__fmul_rn(s, n0), __fmul_rn(s, n1), __fmul_rn(s, n2)};
  const float q = __fadd_rn(__fadd_rn(__fmul_rn(w[0], w[0]), __fmul_rn(w[1], w[1])), __fmul_rn(w[2], w[2]));
  float A = 1.6059044e-10f;
  A = horner_step(A, q, -2.5052108e-08f);
  A = horner_step(A, q, 2.7557319e-06f);
  A = horner_step(A, q, -0.0001984127f);
  A = horner_step(A, q, 0.008333334f);
  A = horner_step(A, q, -0.16666667f);
  A = horner_step(A, q, 1.0f);
  float B = -2.0876756e-09f;
  B = horner_step(B, q, 2.755732e-07f);
  B = horner_step(B, q, -2.4801588e-05f);
  B = horner_step(B, q, 0.0013888889f);
  B = horner_step(B, q, -0.041666668f);
  B = horner_step(B, q, 0.5f);
  float C = -1.6059044e-10f;
  C = horner_step(C, q, 2.5052108e-08f);
  C = horner_step(C, q, -2.7557319e-06f);
  C = horner_step(C, q, 0.0001984127f);
  C = horner_step(C, q, -0.008333334f);
  C = horner_step(C, q, 0.16666667f);
  const float K[9] = {0.0f, -w[2], w[1], w[2], 0.0f, -w[0], -w[1], w[0], 0.0f};  // row-major
  const float pv[3] = {p.x, p.y, p.z};
  float out[3];
#pragma unroll
  for (int j = 0; j < 3; j++) {
    float R[3], V[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const float d = j == k ? 1.0f : 0.0f;
      const float k2 = j == k ? __fsub_rn(__fmul_rn(w[j], w[k]), q) : __fmul_rn(w[j], w[k]);
      R[k] = __fadd_rn(__fadd_rn(d, __fmul_rn(A, K[j * 3 + k])), __fmul_rn(B, k2));
      V[k] = __fadd_rn(__fadd_rn(d, __fmul_rn(B, K[j * 3 + k])), __fmul_rn(C, k2));
    }
    const float rp = __fadd_rn(__fadd_rn(__fmul_rn(R[0], pv[0]), __fmul_rn(R[1], pv[1])), __fmul_rn(R[2], pv[2]));
    const float vu = __fadd_rn(__fadd_rn(__fmul_rn(V[0], u[0]), __fmul_rn(V[1], u[1])), __fmul_rn(V[2], u[2]));
    out[j] = __fadd_rn(rp, vu);
  }
  return make_float3(out[0], out[1], out[2]);
}

__global__ void k_deskew_points(float4* __restrict__ pts, const float* __restrict__ times, int n, float t_ref, float o0, float o1, float o2, float n0, float n1,
                                float n2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = pts[i];
  const float s = __fsub_rn(times[i], t_ref);
  const float3 q = deskew_point(p, s, o0, o1, o2, n0, n1, n2);
  pts[i] = make_float4(q.x, q.y, q.z, 0.0f);
}

// vgicp_set_source_timestamps_device: the caller's strided timestamps packed into `times`, with what the host path finds in its
// pass: stats[0] = the number of non-finite values, stats[1] = ~key(min), stats[2] = key(max) over the finite ones, key() the
// order-preserving map of a float onto an unsigned (stats zeroed before the launch; min and max are exact in any order)
__device__ __forceinline__ unsigned time_key(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__global__ void k_gather_times(const unsigned char* __restrict__ src, size_t stride, int n, float* __restrict__ times, unsigned* __restrict__ stats) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned bad = 0, nlo = 0, hi = 0;  // neutral values of the three reductions
  if (i < n) {
    const float v = *reinterpret_cast<const float*>(src + (size_t)i * stride);
    times[i] = v;
    if (isfinite(v)) {
      nlo = ~time_key(v);
      hi = time_key(v);
    } else {
      bad = 1;
    }
  }
  bad = __reduce_add_sync(0xffffffffu, bad);
  nlo = __reduce_max_sync(0xffffffffu, nlo);
  hi = __reduce_max_sync(0xffffffffu, hi);
  if ((threadIdx.x & 31) == 0) {
    if (bad) atomicAdd(&stats[0], bad);
    atomicMax(&stats[1], nlo);
    atomicMax(&stats[2], hi);
  }
}

}  // namespace vgicp
