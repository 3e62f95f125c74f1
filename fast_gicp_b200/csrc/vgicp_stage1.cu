// vgicp_stage1.cu -- stage 1 kernels: exact k-NN, covariance estimation, regularisation, RBF covariances.
//
// This translation unit is compiled with --fmad=false: every fused multiply-add it wants is spelled __fmaf_rn, every
// other a*b+c stays two roundings, so the per-point results (neighbour order, raw covariance, eigen-decomposition,
// regularised covariance) are a pure function of the input bits and can be checked bit-for-bit against a CPU
// restatement compiled with -ffp-contract=off.  The closed-form 3x3 eigen-solver amplifies 1-ulp differences on
// line-like neighbourhoods (lidar rings) into percent-level differences of the covariance, so "close" is not
// good enough here.
#include "vgicp_stage1.cuh"
#include "vgicp_sort.cuh"

#include <math.h>
#include <stdint.h>
#include <stdlib.h>

namespace vgicp {

// ---------------------------------------------------------------------------------------------------------------
// Stage 1a: exact brute-force k-NN inside one cloud (self included).  One query per thread, targets staged through
// shared memory in tiles (every thread reads the same target -> broadcast, conflict-free), per-thread ascending
// top-k list in shared memory laid out [k][thread] (conflict-free).  d2 = (dx*dx + dy*dy) + dz*dz, no contraction.
// Replaces brute_force_knn.cu:16-60 (global-memory heap per thread) and the CPU kd-tree of
// fast_vgicp_cuda_impl.hpp:152-167.  Output rows ascending in (d2, index).
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kKnnThreads) k_knn_bruteforce(const float4* __restrict__ pts, int n, int k, int* __restrict__ nbr) {
  extern __shared__ float smem_knn[];
  float4* tile = reinterpret_cast<float4*>(smem_knn);                       // kKnnTile float4
  float* ld = smem_knn + 4 * kKnnTile;                                      // [k][kKnnThreads]
  int* li = reinterpret_cast<int*>(ld + (size_t)k * kKnnThreads);           // [k][kKnnThreads]
  const int tid = threadIdx.x;
  const int q = blockIdx.x * kKnnThreads + tid;
  const bool active = q < n;
  float4 qp = active ? pts[q] : make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = 0; j < k; j++) {
    ld[j * kKnnThreads + tid] = __int_as_float(0x7f800000);  // +inf
    li[j * kKnnThreads + tid] = -1;
  }
  float worst = __int_as_float(0x7f800000);
  for (int base = 0; base < n; base += kKnnTile) {
    __syncthreads();
    for (int j = tid; j < kKnnTile; j += kKnnThreads) {
      int g = base + j;
      tile[j] = g < n ? pts[g] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    if (!active) continue;
    const int lim = min(kKnnTile, n - base);
#pragma unroll 4
    for (int j = 0; j < lim; j++) {
      float4 t = tile[j];
      float dx = __fsub_rn(t.x, qp.x), dy = __fsub_rn(t.y, qp.y), dz = __fsub_rn(t.z, qp.z);
      float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      if (d < worst) {  // targets arrive in increasing index, so ties keep the smaller index: ascending (d2, index)
        int p = k - 1;
        while (p > 0 && ld[(p - 1) * kKnnThreads + tid] > d) {
          ld[p * kKnnThreads + tid] = ld[(p - 1) * kKnnThreads + tid];
          li[p * kKnnThreads + tid] = li[(p - 1) * kKnnThreads + tid];
          p--;
        }
        ld[p * kKnnThreads + tid] = d;
        li[p * kKnnThreads + tid] = base + j;
        worst = ld[(k - 1) * kKnnThreads + tid];
      }
    }
  }
  if (active)
    for (int j = 0; j < k; j++) nbr[(size_t)q * k + j] = li[j * kKnnThreads + tid];
}

// ---------------------------------------------------------------------------------------------------------------
// 3x3 helpers (registers).  Full matrices are row-major m[r*3+c] here.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void inv3_general(const float* m, float* o) {  // Eigen Matrix3f::inverse(): cofactors / det (column 0 expansion)
  float c00 = m[4] * m[8] - m[5] * m[7];
  float c10 = m[7] * m[2] - m[8] * m[1];
  float c20 = m[1] * m[5] - m[2] * m[4];
  float det = (c00 * m[0] + c10 * m[3]) + c20 * m[6];
  float id = 1.0f / det;
  o[0] = c00 * id; o[1] = c10 * id; o[2] = c20 * id;
  o[3] = (m[5] * m[6] - m[3] * m[8]) * id;
  o[4] = (m[8] * m[0] - m[6] * m[2]) * id;
  o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  o[6] = (m[3] * m[7] - m[4] * m[6]) * id;
  o[7] = (m[6] * m[1] - m[7] * m[0]) * id;
  o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}
__device__ __forceinline__ void mul3(const float* a, const float* b, float* o) {
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) o[r * 3 + c] = (a[r * 3] * b[c] + a[r * 3 + 1] * b[3 + c]) + a[r * 3 + 2] * b[6 + c];
}
__device__ __forceinline__ float3 cross3(float3 a, float3 b) { return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

// Eigen SelfAdjointEigenSolver<Matrix3f>::computeDirect restated (closed-form roots + cross-product eigenvectors);
// s: symmetric, row-major.  evec columns: V[r*3+c].
__device__ __forceinline__ void eig3_extract_kernel(const float* m, float* res /*3*/, float* rep /*3 or null*/) {
  int i0 = 0;
  float best = fabsf(m[0]);
  if (fabsf(m[4]) > best) { best = fabsf(m[4]); i0 = 1; }
  if (fabsf(m[8]) > best) { best = fabsf(m[8]); i0 = 2; }
  int i1 = (i0 + 1) % 3, i2 = (i0 + 2) % 3;
  float3 r = make_float3(m[0 * 3 + i0], m[1 * 3 + i0], m[2 * 3 + i0]);
  float3 a = make_float3(m[0 * 3 + i1], m[1 * 3 + i1], m[2 * 3 + i1]);
  float3 b = make_float3(m[0 * 3 + i2], m[1 * 3 + i2], m[2 * 3 + i2]);
  float3 c0 = cross3(r, a), c1 = cross3(r, b);
  float n0 = (c0.x * c0.x + c0.y * c0.y) + c0.z * c0.z;
  float n1 = (c1.x * c1.x + c1.y * c1.y) + c1.z * c1.z;
  if (rep) { rep[0] = r.x; rep[1] = r.y; rep[2] = r.z; }
  if (n0 > n1) {
    float s = sqrtf(n0);
    res[0] = c0.x / s; res[1] = c0.y / s; res[2] = c0.z / s;
  } else {
    float s = sqrtf(n1);
    res[0] = c1.x / s; res[1] = c1.y / s; res[2] = c1.z / s;
  }
}

__device__ void eig3_direct(const float* cov /*row-major sym*/, float* evals, float* V /*V[r*3+c], column c = eigenvector c*/) {
  float s[9];
#pragma unroll
  for (int i = 0; i < 9; i++) s[i] = cov[i];
  // selfadjointView<Lower>
  s[1] = s[3]; s[2] = s[6]; s[5] = s[7];
  float shift = ((s[0] + s[4]) + s[8]) / 3.0f;
  s[0] -= shift; s[4] -= shift; s[8] -= shift;
  float scale = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; i++) scale = fmaxf(scale, fabsf(s[i]));
  if (scale > 0.0f) {
#pragma unroll
    for (int i = 0; i < 9; i++) s[i] = s[i] / scale;
  }
  {  // computeRoots
    const float s_inv3 = 1.0f / 3.0f;
    const float s_sqrt3 = sqrtf(3.0f);
    float c0 = s[0] * s[4] * s[8] + 2.0f * s[3] * s[6] * s[7] - s[0] * s[7] * s[7] - s[4] * s[6] * s[6] - s[8] * s[3] * s[3];
    float c1 = s[0] * s[4] - s[3] * s[3] + s[0] * s[8] - s[6] * s[6] + s[4] * s[8] - s[7] * s[7];
    float c2 = s[0] + s[4] + s[8];
    float c2_over_3 = c2 * s_inv3;
    float a_over_3 = fmaxf((c2 * c2_over_3 - c1) * s_inv3, 0.0f);
    float half_b = 0.5f * (c0 + c2_over_3 * (2.0f * c2_over_3 * c2_over_3 - c1));
    float q = fmaxf(a_over_3 * a_over_3 * a_over_3 - half_b * half_b, 0.0f);
    float rho = sqrtf(a_over_3);
    // atan2 / cos / sin evaluated in double and rounded once: the float results are then the correctly rounded ones
    // whatever libm is underneath (CUDA's atan2f/cosf/sinf are 2-ulp functions; line-like neighbourhoods amplify
    // a 1-ulp difference in theta into a visibly different normal).
    float theta = (float)atan2((double)sqrtf(q), (double)half_b) * s_inv3;
    float cos_theta = (float)cos((double)theta), sin_theta = (float)sin((double)theta);
    evals[0] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
    evals[1] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
    evals[2] = c2_over_3 + 2.0f * rho * cos_theta;
  }
  const float eps = 1.1920929e-07f;
  float v0[3], v1[3], v2[3];  // eigenvector columns
  if ((evals[2] - evals[0]) <= eps) {
    v0[0] = 1; v0[1] = 0; v0[2] = 0; v1[0] = 0; v1[1] = 1; v1[2] = 0; v2[0] = 0; v2[1] = 0; v2[2] = 1;
  } else {
    float d0 = evals[2] - evals[1];
    float d1 = evals[1] - evals[0];
    bool k_is_2 = d0 > d1;  // k = index of the most distinct eigenvalue, l = the other extreme
    if (k_is_2) d0 = d1;
    float ek = k_is_2 ? evals[2] : evals[0];
    float el = k_is_2 ? evals[0] : evals[2];
    float tmp[9];
#pragma unroll
    for (int i = 0; i < 9; i++) tmp[i] = s[i];
    tmp[0] -= ek; tmp[4] -= ek; tmp[8] -= ek;
    float vk[3], vl[3];
    eig3_extract_kernel(tmp, vk, vl);
    if (d0 <= 2.0f * eps * d1) {
      float dot = (vk[0] * vl[0] + vk[1] * vl[1]) + vk[2] * vl[2];
      float t0 = vl[0] - dot * vl[0], t1 = vl[1] - dot * vl[1], t2 = vl[2] - dot * vl[2];
      float nn = sqrtf((t0 * t0 + t1 * t1) + t2 * t2);
      if (nn > 0.0f) { vl[0] = t0 / nn; vl[1] = t1 / nn; vl[2] = t2 / nn; }
    } else {
#pragma unroll
      for (int i = 0; i < 9; i++) tmp[i] = s[i];
      tmp[0] -= el; tmp[4] -= el; tmp[8] -= el;
      eig3_extract_kernel(tmp, vl, nullptr);
    }
#pragma unroll
    for (int i = 0; i < 3; i++) { v0[i] = k_is_2 ? vl[i] : vk[i]; v2[i] = k_is_2 ? vk[i] : vl[i]; }
    float3 c = cross3(make_float3(v2[0], v2[1], v2[2]), make_float3(v0[0], v0[1], v0[2]));
    float nn = sqrtf((c.x * c.x + c.y * c.y) + c.z * c.z);
    if (nn > 0.0f) { v1[0] = c.x / nn; v1[1] = c.y / nn; v1[2] = c.z / nn; } else { v1[0] = c.x; v1[1] = c.y; v1[2] = c.z; }
  }
#pragma unroll
  for (int r = 0; r < 3; r++) { V[r * 3 + 0] = v0[r]; V[r * 3 + 1] = v1[r]; V[r * 3 + 2] = v2[r]; }
#pragma unroll
  for (int i = 0; i < 3; i++) evals[i] = evals[i] * scale + shift;
}

// covariance_regularization.cu: PLANE :105-116 (V diag(1e-3,1,1) V^-1), MIN_EIG :84-101, FROBENIUS :74-82.
// c: row-major 3x3 in/out.
__device__ void regularize_cov(float* c, int method) {
  if (method == 3 /*PLANE*/ || method == 1 /*MIN_EIG*/) {
    float ev[3], V[9], Vi[9], Vd[9];
    eig3_direct(c, ev, V);
    float l0 = 1e-3f, l1 = 1.0f, l2 = 1.0f;
    if (method == 1) { l0 = fmaxf(1e-3f, ev[0]); l1 = fmaxf(1e-3f, ev[1]); l2 = fmaxf(1e-3f, ev[2]); }
    inv3_general(V, Vi);
#pragma unroll
    for (int r = 0; r < 3; r++) { Vd[r * 3] = V[r * 3] * l0; Vd[r * 3 + 1] = V[r * 3 + 1] * l1; Vd[r * 3 + 2] = V[r * 3 + 2] * l2; }
    mul3(Vd, Vi, c);
  } else if (method == 4 /*FROBENIUS*/) {
    float C[9], Ci[9];
#pragma unroll
    for (int i = 0; i < 9; i++) C[i] = c[i];
    C[0] += 1e-3f; C[4] += 1e-3f; C[8] += 1e-3f;
    inv3_general(C, Ci);
    float nn = 0.0f;  // Frobenius norm, summed in Eigen's (column-major) coefficient order
#pragma unroll
    for (int cidx = 0; cidx < 3; cidx++)
#pragma unroll
      for (int r = 0; r < 3; r++) nn += Ci[r * 3 + cidx] * Ci[r * 3 + cidx];
    nn = sqrtf(nn);
#pragma unroll
    for (int i = 0; i < 9; i++) Ci[i] = Ci[i] / nn;
    inv3_general(Ci, c);
  }
}

__device__ __forceinline__ void store_cov_sym(const float* c /*row-major 3x3*/, float4* __restrict__ covA, float2* __restrict__ covB, int i) {
  // the regularised matrix is symmetric up to float rounding of V*L*V^-1; the packed store keeps the mean of the
  // two triangles (changes the final pose by ~1e-7 m, see DESIGN.md)
  covA[i] = make_float4(c[0], 0.5f * (c[1] + c[3]), 0.5f * (c[2] + c[6]), c[4]);
  covB[i] = make_float2(0.5f * (c[5] + c[7]), c[8]);
}

// Stage 1b: covariance_estimation.cu:26-34 fused with the regulariser.
__global__ void __launch_bounds__(128) k_covariance_knn(const float4* __restrict__ pts, const int* __restrict__ nbr, int n, int k, int method, float4* __restrict__ covA,
                                                       float2* __restrict__ covB) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float mx = 0.f, my = 0.f, mz = 0.f;
  float cxx = 0.f, cxy = 0.f, cxz = 0.f, cyy = 0.f, cyz = 0.f, czz = 0.f;
  const int* row = nbr + (size_t)i * k;
  for (int j = 0; j < k; j++) {
    float4 p = pts[row[j]];
    mx = __fadd_rn(mx, p.x); my = __fadd_rn(my, p.y); mz = __fadd_rn(mz, p.z);
    cxx = __fmaf_rn(p.x, p.x, cxx); cxy = __fmaf_rn(p.x, p.y, cxy); cxz = __fmaf_rn(p.x, p.z, cxz);
    cyy = __fmaf_rn(p.y, p.y, cyy); cyz = __fmaf_rn(p.y, p.z, cyz); czz = __fmaf_rn(p.z, p.z, czz);
  }
  float kf = (float)k;
  mx = __fdiv_rn(mx, kf); my = __fdiv_rn(my, kf); mz = __fdiv_rn(mz, kf);
  float c[9];
  c[0] = __fmaf_rn(-mx, mx, __fdiv_rn(cxx, kf));
  c[1] = c[3] = __fmaf_rn(-mx, my, __fdiv_rn(cxy, kf));
  c[2] = c[6] = __fmaf_rn(-mx, mz, __fdiv_rn(cxz, kf));
  c[4] = __fmaf_rn(-my, my, __fdiv_rn(cyy, kf));
  c[5] = c[7] = __fmaf_rn(-my, mz, __fdiv_rn(cyz, kf));
  c[8] = __fmaf_rn(-mz, mz, __fdiv_rn(czz, kf));
  regularize_cov(c, method);
  store_cov_sym(c, covA, covB, i);
}

// The same for a slice of the cloud when stage 1 is sharded over several GPUs (SURVEY 8e): thread t takes the point at sorted
// position pos_begin + t of the k-NN grid (the slice whose neighbour rows this rank computed) and stores its covariance into the
// covariance arrays of EVERY rank -- plain peer stores over NVLink into IPC-mapped memory, own copy included -- so that each rank
// ends up with the covariances of the whole cloud without a collective call.
struct CovPeers {
  float4* covA[8];
  float2* covB[8];
  int nranks;
};
__global__ void __launch_bounds__(128) k_covariance_knn_sharded(const float4* __restrict__ pts, const int* __restrict__ nbr, const float4* __restrict__ sorted, int pos_begin, int pos_end,
                                                               int k, int method, CovPeers peers) {
  const int pos = pos_begin + blockIdx.x * blockDim.x + threadIdx.x;
  if (pos >= pos_end) return;
  const int i = __float_as_int(sorted[pos].w);
  float mx = 0.f, my = 0.f, mz = 0.f;
  float cxx = 0.f, cxy = 0.f, cxz = 0.f, cyy = 0.f, cyz = 0.f, czz = 0.f;
  const int* row = nbr + (size_t)i * k;
  for (int j = 0; j < k; j++) {
    float4 p = pts[row[j]];
    mx = __fadd_rn(mx, p.x); my = __fadd_rn(my, p.y); mz = __fadd_rn(mz, p.z);
    cxx = __fmaf_rn(p.x, p.x, cxx); cxy = __fmaf_rn(p.x, p.y, cxy); cxz = __fmaf_rn(p.x, p.z, cxz);
    cyy = __fmaf_rn(p.y, p.y, cyy); cyz = __fmaf_rn(p.y, p.z, cyz); czz = __fmaf_rn(p.z, p.z, czz);
  }
  float kf = (float)k;
  mx = __fdiv_rn(mx, kf); my = __fdiv_rn(my, kf); mz = __fdiv_rn(mz, kf);
  float c[9];
  c[0] = __fmaf_rn(-mx, mx, __fdiv_rn(cxx, kf));
  c[1] = c[3] = __fmaf_rn(-mx, my, __fdiv_rn(cxy, kf));
  c[2] = c[6] = __fmaf_rn(-mx, mz, __fdiv_rn(cxz, kf));
  c[4] = __fmaf_rn(-my, my, __fdiv_rn(cyy, kf));
  c[5] = c[7] = __fmaf_rn(-my, mz, __fdiv_rn(cyz, kf));
  c[8] = __fmaf_rn(-mz, mz, __fdiv_rn(czz, kf));
  regularize_cov(c, method);
  const float4 a4 = make_float4(c[0], 0.5f * (c[1] + c[3]), 0.5f * (c[2] + c[6]), c[4]);
  const float2 b2 = make_float2(0.5f * (c[5] + c[7]), c[8]);
  for (int r = 0; r < peers.nranks; r++) {
    peers.covA[r][i] = a4;
    peers.covB[r][i] = b2;
  }
}

// exp(x) for x <= 0 from IEEE single operations only (Cephes' expf: n = rint(x log2 e), two-step reduction r = x - n ln 2,
// degree-5 polynomial, scale by 2^n), every operation spelled, so that the CPU checker evaluates the identical sequence.
// Why not expf: the reference calls CUDA's expf, a 2-ulp function that no CPU libm reproduces bit for bit; this one has the same
// accuracy class (about 1 ulp) and makes the RBF stage testable bit-for-bit like the rest of this file.
__device__ __forceinline__ float exp_det(float x) {
  if (x < -87.0f) return 0.0f;
  const float n = rintf(__fmul_rn(x, 1.44269504088896341f));
  float r = __fmaf_rn(n, -0.693359375f, x);
  r = __fmaf_rn(n, 2.12194440e-4f, r);
  float p = 1.9875691500e-4f;
  p = __fmaf_rn(p, r, 1.3981999507e-3f);
  p = __fmaf_rn(p, r, 8.3334519073e-3f);
  p = __fmaf_rn(p, r, 4.1665795894e-2f);
  p = __fmaf_rn(p, r, 1.6666665459e-1f);
  p = __fmaf_rn(p, r, 5.0000001201e-1f);
  p = __fadd_rn(__fmaf_rn(p, __fmul_rn(r, r), r), 1.0f);
  return __fmul_rn(p, __int_as_float(((int)n + 127) << 23));
}

// bounding boxes of the 512-point blocks of the (zero-padded) cloud: box[b] = {min xyz, max xyz}
__global__ void __launch_bounds__(128) k_rbf_block_boxes(const float4* __restrict__ pts, int n, float* __restrict__ boxes) {
  __shared__ float red[4][6];
  const int b = blockIdx.x, tid = threadIdx.x;
  float lo[3] = {__int_as_float(0x7f800000), __int_as_float(0x7f800000), __int_as_float(0x7f800000)};
  float hi[3] = {__int_as_float(0xff800000), __int_as_float(0xff800000), __int_as_float(0xff800000)};
  for (int j = tid; j < kRbfBlock; j += 128) {
    const int g = b * kRbfBlock + j;
    const float4 p = g < n ? pts[g] : make_float4(0.f, 0.f, 0.f, 0.f);  // the padding sits at the origin (:126-129)
    lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
    hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
  }
#pragma unroll
  for (int d = 0; d < 3; d++)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  if ((tid & 31) == 0)
    for (int d = 0; d < 3; d++) { red[tid >> 5][d] = lo[d]; red[tid >> 5][3 + d] = hi[d]; }
  __syncthreads();
  if (tid < 6) {
    float v = red[0][tid];
    for (int w = 1; w < 4; w++) v = tid < 3 ? fminf(v, red[w][tid]) : fmaxf(v, red[w][tid]);
    boxes[b * 6 + tid] = v;
  }
}

// Stage 1b': covariance_estimation_rbf.cu:59-151.  The reference accumulates, per query, one partial {sum w, sum w p, sum w p p^T}
// per block of 512 consecutive points (sequentially inside the block, :59-90) and adds the partials in block order (:92-114); the
// cloud is padded to a multiple of 512 with points at the origin (:126-129) which pick up weight whenever the query is within
// max_dist of the origin -- all reproduced.  All nine entries of sum w p p^T are kept ((w p_r) p_c and (w p_c) p_r round differently
// and the reference's Matrix3f holds both).
// Parallel shape: the blocks of one query are independent, so EIGHT lanes share a query and take the blocks 8 r + lane of round r
// (16 queries per 128-thread block); after each round the query's first lane adds the eight partials in block order.  That is 8x the
// threads of a thread-per-query loop (4288 warps instead of 536 at 17 k points: the loop is a latency chain per thread).
// A block whose bounding box is farther than max_dist from the query contributes an all-zero partial (x + 0 == x) and is skipped; the
// float box distance uses the same operations as the per-point distance and rounding is monotone, so it never exceeds it.
constexpr int kRbfLanes = 8;                          // lanes (blocks in flight) per query
constexpr int kRbfQueries = 128 / kRbfLanes;          // queries per thread block
constexpr int kRbfTileStride = kRbfBlock + 1;         // float4 per staged tile (+1: the eight tiles start in different banks)
__global__ void __launch_bounds__(128) k_covariance_rbf(const float4* __restrict__ pts, int n, float exp_factor, float max_dist, int method, const float* __restrict__ boxes,
                                                       float4* __restrict__ covA, float2* __restrict__ covB) {
  extern __shared__ float4 rbf_tiles[];                                 // [kRbfLanes][kRbfTileStride]
  __shared__ float part[kRbfQueries][kRbfLanes][13];                    // one partial per (query, lane) and round
  const int tid = threadIdx.x, ql = tid / kRbfLanes, l = tid % kRbfLanes;
  const int q = blockIdx.x * kRbfQueries + ql;
  const bool active = q < n;
  const float4 x = pts[active ? q : n - 1];
  const float max_dist_sq = max_dist * max_dist;
  float sw = 0.f, m[3] = {0.f, 0.f, 0.f}, c[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // running totals (lane 0 of the query); c row-major
  const int nblocks = (n + kRbfBlock - 1) / kRbfBlock;
  for (int r0 = 0; r0 < nblocks; r0 += kRbfLanes) {
    __syncthreads();  // the previous round's tiles and partials are consumed
    for (int j = tid; j < kRbfLanes * kRbfBlock; j += 128) {
      const int t = j / kRbfBlock, jj = j % kRbfBlock;
      const int g = (r0 + t) * kRbfBlock + jj;
      rbf_tiles[t * kRbfTileStride + jj] = g < n ? pts[g] : make_float4(0.f, 0.f, 0.f, 0.f);  // padding at the origin, :126-129
    }
    __syncthreads();
    const int b = r0 + l;
    float psw = 0.f, pm[3] = {0.f, 0.f, 0.f}, pc[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    bool need = false;
    if (b < nblocks) {
      const float* bx = boxes + b * 6;
      const float dx = fmaxf(fmaxf(bx[0] - x.x, x.x - bx[3]), 0.f), dy = fmaxf(fmaxf(bx[1] - x.y, x.y - bx[4]), 0.f), dz = fmaxf(fmaxf(bx[2] - x.z, x.z - bx[5]), 0.f);
      need = !((dx * dx + dy * dy) + dz * dz > max_dist_sq);
    }
    if (need) {
      const float4* tile = rbf_tiles + l * kRbfTileStride;
      for (int j = 0; j < kRbfBlock; j++) {
        const float4 p = tile[j];
        const float dx = x.x - p.x, dy = x.y - p.y, dz = x.z - p.z;
        const float sq = (dx * dx + dy * dy) + dz * dz;
        if (sq > max_dist_sq) continue;
        const float w = exp_det(-exp_factor * sq);
        psw += w;
        const float wx = w * p.x, wy = w * p.y, wz = w * p.z;
        pm[0] += wx; pm[1] += wy; pm[2] += wz;
        pc[0] += wx * p.x; pc[1] += wx * p.y; pc[2] += wx * p.z;
        pc[3] += wy * p.x; pc[4] += wy * p.y; pc[5] += wy * p.z;
        pc[6] += wz * p.x; pc[7] += wz * p.y; pc[8] += wz * p.z;
      }
    }
    float* pp = part[ql][l];
    pp[0] = psw;
#pragma unroll
    for (int d = 0; d < 3; d++) pp[1 + d] = pm[d];
#pragma unroll
    for (int d = 0; d < 9; d++) pp[4 + d] = pc[d];
    __syncthreads();
    if (l == 0) {  // the reference's finalisation order: partials added block by block
      for (int t = 0; t < kRbfLanes && r0 + t < nblocks; t++) {
        const float* s = part[ql][t];
        sw += s[0];
#pragma unroll
        for (int d = 0; d < 3; d++) m[d] += s[1 + d];
#pragma unroll
        for (int d = 0; d < 9; d++) c[d] += s[4 + d];
      }
    }
  }
  if (!active || l != 0) return;
  // NormalDistribution::finalize :47-53:  mean = sum/sw ; cov = (cov - mean*sum^T)/sw
  float mean[3] = {m[0] / sw, m[1] / sw, m[2] / sw};
  float cc[9];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int col = 0; col < 3; col++) cc[r * 3 + col] = (c[r * 3 + col] - mean[r] * m[col]) / sw;
  regularize_cov(cc, method);
  store_cov_sym(cc, covA, covB, q);
}


// ---------------------------------------------------------------------------------------------------------------
// Stage 1a': exact k-NN on a Morton-ordered multi-level grid, one THREAD per query.
//
// Why: lidar clouds are surfaces whose density falls with range; the 20-NN radius spans 0.2 m .. several metres, so no single
// cell size fits.  The points are sorted ONCE by the Morton code of their finest cell (cell size s_0 = extent / 2^(L+1)); a cell
// of level l (size s_0 * 2^l) is then a contiguous run of the sorted array, and one hash table maps (level, cell) -> [start, end).
// The table is filled from the sorted codes alone (a point starts / ends the cells of every level at which its code differs
// from its predecessor's / successor's): no per-level scatter, one sorted copy of the cloud for all levels.
//
// Query (thread i = sorted position i, so the threads of a warp are spatial neighbours and mostly walk the same cells):
//   1. the 2k+1 points around position i in Morton order seed a max-heap of the k best (d2, index) keys -> an upper bound B on
//      the k-th distance;
//   2. the finest level l with 0.999 s_l >= B: every point within B of the query lies in the 3x3x3 block of its cell there;
//   3. the block's cells whose box lies within the (shrinking) k-th distance are looked up and scanned, skipping the window.
// That is exact by construction (no certificate, no restart).  Blocks with very many candidates and queries whose bound exceeds
// the coarsest level (tiny clouds, far outliers) are handed to a block-cooperative kernel.
// Top-k: a binary max-heap of 64-bit keys ((bits of d2) << 32 | index; d2 >= 0, so unsigned order == ascending (d2, index)) in
// shared memory, [k][thread] (bank = thread: conflict-free whatever heap slot each lane touches); heap-sorted in place at the
// end, so rows come out as the unique ascending (d2, index) list -- identical to the CPU checker.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kGridMaxLevels = 12;
constexpr unsigned long long kGridEmpty = 0xFFFFFFFFFFFFFFFFULL;

struct __align__(16) CellEntry {
  unsigned long long key;  // (Morton prefix of the cell << 4) | level, kGridEmpty when free
  unsigned start, end;     // the cell's points are sorted[start .. end)
};

struct GridArgs {
  const float4* pts;
  int n, k, L;
  unsigned* bbox_min;          // [3] ordered-uint min xyz (initialised to 0xFFFFFFFF)
  unsigned* bbox_max;          // [3] ordered-uint max xyz (initialised to 0)
  unsigned long long* codes;   // [n] Morton codes of the finest cells, sorted
  float4* sorted;              // [n] points in that order, original index in .w
  CellEntry* table;
  unsigned tmask;
  int* level_hist;             // [kGridMaxLevels + 2] histogram over the points of "first level shared with the predecessor"
  int* l_min;                  // finest level present in the table
  unsigned* done_blocks;       // ticket of k_grid_levels
  int* defer_count;            // queries handed to the block-cooperative kernel
  int* defer_cursor;
  int2* defer_queue;           // [n] (sorted position, level of the block to scan; L = whole cloud)
  int q_begin, q_end;          // sorted positions searched by this launch (multi-GPU: a slice per rank)
  int* nbr;
};

__device__ __forceinline__ unsigned f2ord(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

__global__ void k_grid_bbox(const float4* __restrict__ pts, int n, unsigned* __restrict__ bbox_min, unsigned* __restrict__ bbox_max) {
  float lo[3] = {__int_as_float(0x7f800000), __int_as_float(0x7f800000), __int_as_float(0x7f800000)};
  float hi[3] = {__int_as_float(0xff800000), __int_as_float(0xff800000), __int_as_float(0xff800000)};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float4 p = pts[i];
    lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
    hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
  }
#pragma unroll
  for (int d = 0; d < 3; d++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int d = 0; d < 3; d++) {
      atomicMin(&bbox_min[d], f2ord(lo[d]));
      atomicMax(&bbox_max[d], f2ord(hi[d]));
    }
  }
}

struct GridGeom {
  float minx, miny, minz;
  float s0, inv_s0;  // finest cell size
  int cmax;          // largest cell coordinate of the finest level: 2^(L+1) - 1
};
__device__ __forceinline__ GridGeom grid_geom(const unsigned* __restrict__ bmin, const unsigned* __restrict__ bmax, int L) {
  GridGeom g;
  g.minx = ord2f(bmin[0]); g.miny = ord2f(bmin[1]); g.minz = ord2f(bmin[2]);
  float ex = ord2f(bmax[0]) - g.minx, ey = ord2f(bmax[1]) - g.miny, ez = ord2f(bmax[2]) - g.minz;
  float e = fmaxf(fmaxf(ex, ey), fmaxf(ez, 1e-3f));
  g.s0 = ldexpf(e, -(L + 1));  // coarsest level: 4 cells along the longest axis
  g.inv_s0 = 1.0f / g.s0;
  g.cmax = (2 << L) - 1;
  return g;
}
// finest-level cell of a point; the far face of the bounding box is clamped into the last cell (its box is closed there)
__device__ __forceinline__ int3 grid_cell0(const GridGeom& g, float x, float y, float z) {
  int cx = (int)floorf((x - g.minx) * g.inv_s0), cy = (int)floorf((y - g.miny) * g.inv_s0), cz = (int)floorf((z - g.minz) * g.inv_s0);
  return make_int3(min(max(cx, 0), g.cmax), min(max(cy, 0), g.cmax), min(max(cz, 0), g.cmax));
}
__device__ __forceinline__ unsigned long long spread3(unsigned v) {  // bit i of v -> bit 3 i
  unsigned long long x = v & 0x1fffffu;
  x = (x | x << 32) & 0x1f00000000ffffULL;
  x = (x | x << 16) & 0x1f0000ff0000ffULL;
  x = (x | x << 8) & 0x100f00f00f00f00fULL;
  x = (x | x << 4) & 0x10c30c30c30c30c3ULL;
  x = (x | x << 2) & 0x1249249249249249ULL;
  return x;
}
__device__ __forceinline__ unsigned long long morton3(int x, int y, int z) { return (spread3((unsigned)x) << 2) | (spread3((unsigned)y) << 1) | spread3((unsigned)z); }
__device__ __forceinline__ unsigned grid_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return (unsigned)k;
}
// first level at which two finest-cell codes fall into the same cell (0 when equal)
__device__ __forceinline__ int shared_level(unsigned long long a, unsigned long long b) {
  const unsigned long long x = a ^ b;
  return x ? (63 - __clzll((long long)x)) / 3 + 1 : 0;
}

// Morton codes of the finest cells + the digit histograms of the sort
__global__ void __launch_bounds__(kSortThreads) k_grid_codes(GridArgs a, int passes, unsigned* __restrict__ hist) {
  __shared__ unsigned sh[kSortMaxPasses * kSortBins];
  for (int i = threadIdx.x; i < passes * kSortBins; i += kSortThreads) sh[i] = 0;
  __syncthreads();
  const GridGeom g = grid_geom(a.bbox_min, a.bbox_max, a.L);
  const int n_round = (a.n + 31) & ~31;
  for (int i = blockIdx.x * kSortThreads + threadIdx.x; i < n_round; i += gridDim.x * kSortThreads) {
    const bool valid = i < a.n;
    unsigned long long code = 0;
    if (valid) {
      const float4 p = a.pts[i];
      const int3 c = grid_cell0(g, p.x, p.y, p.z);
      code = morton3(c.x, c.y, c.z);
      a.codes[i] = code;
    }
    sort_hist_add(sh, passes, valid, code);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < passes * kSortBins; i += kSortThreads)
    if (sh[i]) atomicAdd(&hist[i], sh[i]);
}

// cells per level (from the sorted codes) -> the finest level whose cells, together with all coarser ones, fit half the table
__global__ void __launch_bounds__(256) k_grid_levels(GridArgs a) {
  __shared__ int sh[kGridMaxLevels + 2];
  __shared__ bool is_last;
  if (threadIdx.x < kGridMaxLevels + 2) sh[threadIdx.x] = 0;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const int ld = i > 0 ? min(shared_level(a.codes[i], a.codes[i - 1]), a.L) : a.L;  // starts a cell at every level below ld
    atomicAdd(&sh[ld], 1);
  }
  __syncthreads();
  if (threadIdx.x < kGridMaxLevels + 2 && sh[threadIdx.x]) atomicAdd(&a.level_hist[threadIdx.x], sh[threadIdx.x]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(a.done_blocks, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last || threadIdx.x != 0) return;
  __threadfence();
  // cells of level l = points with ld > l; walk from the coarsest level down while the total stays within half the table
  const long long cap = ((long long)a.tmask + 1) / 2;
  long long cells = 0, total = 0;
  int l_min = a.L - 1;
  for (int l = a.L - 1; l >= 0; l--) {
    cells += *reinterpret_cast<volatile int*>(&a.level_hist[l + 1]);
    if (total + cells > cap && l < a.L - 1) break;
    total += cells;
    l_min = l;
  }
  *a.l_min = l_min;
}

// table fill: position i opens the cells of the levels at which its code differs from its predecessor's and closes those at
// which it differs from its successor's.  The opener and the closer of a cell find the same slot (insert-or-find by CAS on the key)
// and write different fields of it.
__device__ __forceinline__ CellEntry* table_slot(const GridArgs& a, unsigned long long key) {
  unsigned pos = grid_hash(key) & a.tmask;
  for (;;) {
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(&a.table[pos].key);
    if (cur == kGridEmpty) {
      const unsigned long long old = atomicCAS(&a.table[pos].key, kGridEmpty, key);
      cur = (old == kGridEmpty) ? key : old;
    }
    if (cur == key) return &a.table[pos];
    pos = (pos + 1) & a.tmask;
  }
}
__global__ void __launch_bounds__(256) k_grid_table(GridArgs a) {  // blockIdx.y = level - l_min: a thread per (point, level), two slot operations at most
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int l = *a.l_min + (int)blockIdx.y;
  if (i >= a.n || l >= a.L) return;
  const unsigned long long c = a.codes[i];
  const int ls = i > 0 ? min(shared_level(c, a.codes[i - 1]), a.L) : a.L;
  const int le = i + 1 < a.n ? min(shared_level(c, a.codes[i + 1]), a.L) : a.L;
  if (l >= ls && l >= le) return;
  CellEntry* e = table_slot(a, ((c >> (3 * l)) << 4) | (unsigned)l);
  if (l < ls) e->start = (unsigned)i;
  if (l < le) e->end = (unsigned)i + 1u;
}

__device__ __forceinline__ bool cell_range(const GridArgs& a, unsigned long long key, int& start, int& end) {
  unsigned pos = grid_hash(key) & a.tmask;
  for (;;) {
    const uint4 e = __ldg(reinterpret_cast<const uint4*>(&a.table[pos]));
    const unsigned long long cur = ((unsigned long long)e.y << 32) | e.x;
    if (cur == key) { start = (int)e.z; end = (int)e.w; return true; }
    if (cur == kGridEmpty) return false;
    pos = (pos + 1) & a.tmask;
  }
}

typedef unsigned long long tkey;
constexpr tkey kKeyInf = 0x7f8000007fffffffULL;  // (+inf, INT_MAX)
__device__ __forceinline__ tkey make_key(float d, int i) { return ((tkey)__float_as_uint(d) << 32) | (unsigned)i; }
__device__ __forceinline__ int key_index(tkey e) { return (int)(unsigned)(e & 0xffffffffULL); }
__device__ __forceinline__ float knn_d2(float4 q, float4 t) {  // (dx*dx + dy*dy) + dz*dz, no contraction
  float dx = __fsub_rn(t.x, q.x), dy = __fsub_rn(t.y, q.y), dz = __fsub_rn(t.z, q.z);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// compare-exchange step of a bitonic network over the 32 lanes: lane keeps the smaller key when keep_min
__device__ __forceinline__ void cmpx(tkey& e, int stride, bool keep_min) {
  tkey o = __shfl_xor_sync(0xffffffffu, e, stride);
  if ((o < e) == keep_min) e = o;  // keys are distinct except (inf, INT_MAX) padding, where either choice is the same
}

constexpr int kSearchWarps = 8;          // queries per block of the search kernel
constexpr int kWarpBuf = 128;            // per-warp buffer of candidate keys within the bound
constexpr int kDeferCandidates = 2048;   // blocks with more candidates than this go to the block-cooperative kernel (density transitions)

// Smallest-ish threshold T on distance bits with at least k of the warp's values <= T (each lane holds NV values; absent = 0xFFFFFFFF):
// bisection on the bit pattern (non-negative floats order like their bits), one ballot per value and step, stopping as soon as at
// most `limit` values qualify.  `hi` must qualify on entry.  All lanes return the same T.
template <int NV>
__device__ __forceinline__ unsigned warp_tighten(const unsigned (&v)[NV], int k, int limit, unsigned hi) {
  unsigned lo = 0;
  while (hi - lo > 1u) {
    const unsigned mid = lo + ((hi - lo) >> 1);
    int c = 0;
#pragma unroll
    for (int j = 0; j < NV; j++) c += __popc(__ballot_sync(0xffffffffu, v[j] <= mid));
    if (c >= k) {
      hi = mid;
      if (c <= limit) break;
    } else {
      lo = mid;
    }
  }
  return hi;
}

// finest level l >= l_min with 0.998 s_l >= B (L when there is none); s = that level's cell size
__device__ __forceinline__ int level_for(float B, int l_min, int L, float s0, float& s) {
  int l = l_min;
  s = ldexpf(s0, l);
  while (l < L && !(B <= 0.998f * s)) { l++; s *= 2.0f; }  // (also runs to L when B is inf / NaN)
  return l;
}

// One warp per query (sorted position i); every step is warp-synchronous, so the lanes never diverge:
//   1. the 64 points around position i in Morton order (two coalesced loads): the k-th smallest of their distances, found by a
//      warp bisection (ballot + popc per step), bounds the k-th distance from above;
//   2. the finest level l with 0.998 s_l >= bound: every point within the bound of the query lies in the 3x3x3 block of its cell
//      there (window points included); 27 lanes look the block's cells up in parallel, cells whose box is beyond the bound are dropped;
//   3. the cells' runs are flattened into one index space (prefix sum over the lanes) and read 32 candidates at a time; those within
//      the bound are appended (ballot + prefix) to the warp's buffer in shared memory -- nothing is sorted while scanning;
//   4. the buffer is tightened to at most 32 (64 for k > 32) keys by another bisection, the survivors are sorted once across the
//      lanes (bitonic network on 64-bit keys) and the first k are the row, ascending in (d2, index).
// Alternatives tried and dropped (all exact, all slower on the 17 k-point fixture cloud):
//   one thread per query, max-heap of the k best in shared memory  (low lane efficiency, dependent shared-memory chains, a long tail)
//   one thread per query, bisection + append buffer + rank sort
//   this kernel with four consecutive queries per warp sharing the 27 table lookups  (fewer, longer warps)
//   eight lanes per query, four queries per warp (segmented ballots / shuffles)
template <bool WIDE>
__global__ void __launch_bounds__(kSearchWarps * 32) k_knn_search(GridArgs a, int force_whole_cloud) {
  __shared__ tkey sbuf[kSearchWarps][kWarpBuf];
  __shared__ tkey sfin[kSearchWarps][64];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  const int i = a.q_begin + blockIdx.x * kSearchWarps + wid;
  if (i >= a.q_end) return;
  const int k = a.k, L = a.L;
  const GridGeom g = grid_geom(a.bbox_min, a.bbox_max, L);
  const float4 q = __ldg(&a.sorted[i]);
  const int qi = __float_as_int(q.w);
  if (force_whole_cloud) {
    if (lane == 0) a.defer_queue[atomicAdd(a.defer_count, 1)] = make_int2(i, L);
    return;
  }
  tkey* buf = sbuf[wid];
  // 1. Morton window -> bound on the k-th distance (k <= 64 <= window size whenever n >= 64; a smaller cloud is all window)
  unsigned T;
  {
    int w0 = i - 32;
    if (w0 > a.n - 64) w0 = a.n - 64;
    if (w0 < 0) w0 = 0;
    unsigned v[2];
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int p = w0 + u * 32 + lane;
      v[u] = 0xFFFFFFFFu;
      if (p < a.n) v[u] = __float_as_uint(knn_d2(q, __ldg(&a.sorted[p])));
    }
    // bracket: the largest window distance qualifies (>= k valid points); most of the steps of a bisection from [0, inf) would only
    // locate its binade
    unsigned mx = max(v[0] == 0xFFFFFFFFu ? 0u : v[0], v[1] == 0xFFFFFFFFu ? 0u : v[1]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    T = warp_tighten<2>(v, k, k + 2, mx);
  }
  const int l_min = *a.l_min;
  float s;
  const int l = level_for(sqrtf(__uint_as_float(T)), l_min, L, g.s0, s);
  if (l >= L) {  // the bound exceeds the coarsest cells (tiny cloud, far outlier): whole cloud, block-cooperative
    if (lane == 0) a.defer_queue[atomicAdd(a.defer_count, 1)] = make_int2(i, L);
    return;
  }
  // 2. the block's cells, one per lane
  int st = 0, cn = 0;
  if (lane < 27) {
    const int3 c0 = grid_cell0(g, q.x, q.y, q.z);
    const int cl_max = g.cmax >> l;
    const int cx = (c0.x >> l) + lane / 9 - 1, cy = (c0.y >> l) + (lane / 3) % 3 - 1, cz = (c0.z >> l) + lane % 3 - 1;
    if ((unsigned)cx <= (unsigned)cl_max && (unsigned)cy <= (unsigned)cl_max && (unsigned)cz <= (unsigned)cl_max) {
      // distance from the query to the cell's box against the bound (+ slack for the rounding of the cell boundaries)
      const float fx = q.x - g.minx, fy = q.y - g.miny, fz = q.z - g.minz;
      const float lx = cx * s, ly = cy * s, lz = cz * s;
      const float ex = fmaxf(fmaxf(lx - fx, fx - (lx + s)), 0.f), ey = fmaxf(fmaxf(ly - fy, fy - (ly + s)), 0.f), ez = fmaxf(fmaxf(lz - fz, fz - (lz + s)), 0.f);
      const float reach = sqrtf(__uint_as_float(T)) + 2e-3f * s;
      if (ex * ex + ey * ey + ez * ez <= reach * reach) {
        int en;
        if (cell_range(a, (morton3(cx, cy, cz) << 4) | (unsigned)l, st, en)) cn = en - st;
      }
    }
  }
  // 3. flatten the runs and scan
  int incl = cn;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  const int excl = incl - cn;
  if (total > kDeferCandidates) {  // block-cooperative kernel (scans the block afresh)
    if (lane == 0) a.defer_queue[atomicAdd(a.defer_count, 1)] = make_int2(i, l);
    return;
  }
  int cnt = 0;  // keys in the buffer (warp-uniform)
  constexpr int U = 2;
  for (int base = 0; base < total; base += 32 * U) {
    float4 c[U];
    bool valid[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int j = base + u * 32 + lane;
      valid[u] = j < total;
      c[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (base + u * 32 < total) {  // warp-uniform
        int cell = 0;  // largest lane index whose exclusive prefix is <= j (runs of equal prefixes end at the non-empty cell)
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
          const int e = __shfl_sync(0xffffffffu, excl, (cell + step) & 31);
          if (e <= j) cell += step;
        }
        const int cs = __shfl_sync(0xffffffffu, st, cell);
        const int ce = __shfl_sync(0xffffffffu, excl, cell);
        if (valid[u]) c[u] = __ldg(&a.sorted[cs + (j - ce)]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (base + u * 32 >= total) break;
      const float d2 = knn_d2(q, c[u]);
      const bool pass = valid[u] && __float_as_uint(d2) <= T;
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      if (pass) buf[cnt + __popc(m & lt)] = make_key(d2, __float_as_int(c[u].w));
      cnt += __popc(m);
      if (cnt > kWarpBuf - 32) {  // the next batch might not fit: tighten the bound to about the k-th distance of the buffered keys
        __syncwarp();
        unsigned v[kWarpBuf / 32];
#pragma unroll
        for (int t = 0; t < kWarpBuf / 32; t++) v[t] = t * 32 + lane < cnt ? (unsigned)(buf[t * 32 + lane] >> 32) : 0xFFFFFFFFu;
        T = warp_tighten<kWarpBuf / 32>(v, k, k + (k >> 2) + 1, T);
        tkey keep[kWarpBuf / 32];
#pragma unroll
        for (int t = 0; t < kWarpBuf / 32; t++) keep[t] = t * 32 + lane < cnt ? buf[t * 32 + lane] : kKeyInf;
        __syncwarp();
        int w = 0;
#pragma unroll
        for (int t = 0; t < kWarpBuf / 32; t++) {
          const bool kp = v[t] <= T;
          const unsigned mm = __ballot_sync(0xffffffffu, kp);
          if (kp) buf[w + __popc(mm & lt)] = keep[t];
          w += __popc(mm);
        }
        cnt = w;
        __syncwarp();
        if (cnt > kWarpBuf - 32) {  // ties (duplicate points) that a distance threshold cannot separate: cooperative kernel
          if (lane == 0) a.defer_queue[atomicAdd(a.defer_count, 1)] = make_int2(i, l);
          return;
        }
      }
    }
  }
  __syncwarp();
  // 4. at most 32 (64) survivors -> one sort
  constexpr int NF = WIDE ? 2 : 1;
  {
    unsigned v[kWarpBuf / 32];
    tkey keep[kWarpBuf / 32];
#pragma unroll
    for (int t = 0; t < kWarpBuf / 32; t++) {
      keep[t] = t * 32 + lane < cnt ? buf[t * 32 + lane] : kKeyInf;
      v[t] = t * 32 + lane < cnt ? (unsigned)(keep[t] >> 32) : 0xFFFFFFFFu;
    }
    if (cnt > 32 * NF) T = warp_tighten<kWarpBuf / 32>(v, k, 32 * NF, T);
    tkey* fin = sfin[wid];
    fin[lane] = kKeyInf;
    fin[32 + lane] = kKeyInf;
    __syncwarp();
    int w = 0;
#pragma unroll
    for (int t = 0; t < kWarpBuf / 32; t++) {
      const bool kp = v[t] <= T;
      const unsigned mm = __ballot_sync(0xffffffffu, kp);
      const int dst = w + __popc(mm & lt);
      if (kp && dst < 64) fin[dst] = keep[t];
      w += __popc(mm);
    }
    __syncwarp();
    if (w > 32 * NF) {  // more equal distances than the sort holds: cooperative kernel
      if (lane == 0) a.defer_queue[atomicAdd(a.defer_count, 1)] = make_int2(i, l);
      return;
    }
    tkey e0 = fin[lane], e1 = WIDE ? fin[32 + lane] : kKeyInf;
    // bitonic sort of the 32 (64) keys across the lanes
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        const bool up = (lane & size) == 0 || size == 32;
        const bool lower = (lane & stride) == 0;
        cmpx(e0, stride, lower == up);
        if (WIDE) cmpx(e1, stride, lower != up);  // the second register is sorted descending: (e0, e1) is then bitonic
      }
    }
    if (WIDE) {  // size == 32 sorted e1 descending over the lanes; merge the bitonic 64
      const tkey lo_ = e0 < e1 ? e0 : e1, hi_ = e0 < e1 ? e1 : e0;
      e0 = lo_;
      e1 = hi_;
#pragma unroll
      for (int stride = 16; stride > 0; stride >>= 1) {
        cmpx(e0, stride, (lane & stride) == 0);
        cmpx(e1, stride, (lane & stride) == 0);
      }
    }
    int* row = a.nbr + (size_t)qi * k;
    if (lane < k) row[lane] = key_index(e0);
    if (WIDE && 32 + lane < k) row[32 + lane] = key_index(e1);
  }
}

// ---- warp-level sorted top-k (k <= 64) for the block-cooperative kernel: rank r lives in lane r & 31, register r >> 5.
// WIDE=false (k <= 32) keeps a single register set. ----
struct WarpTopK {
  tkey e0, e1;
  tkey worst;  // entry of rank k-1, broadcast
};

__device__ __forceinline__ void topk_reset(WarpTopK& t) { t.e0 = t.e1 = t.worst = kKeyInf; }

// Merge a batch of 32 candidates into the sorted list (k <= 32): bitonic-sort the batch (15 steps), take the element-wise
// minimum with the reversed list (the 32 smallest of the 64, a bitonic sequence), bitonic-merge (5 steps).
__device__ __forceinline__ void topk_merge32(WarpTopK& t, int k, int lane, tkey c) {
#pragma unroll
  for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      bool up = (lane & size) == 0 || size == 32;
      bool lower = (lane & stride) == 0;
      cmpx(c, stride, lower == up);
    }
  }
  if (__all_sync(0xffffffffu, t.e0 == kKeyInf)) {  // (the vote must not sit behind a per-lane short-circuit)
    t.e0 = c;  // empty list: the sorted batch is the list
  } else {
    tkey r = __shfl_sync(0xffffffffu, c, 31 - lane);
    if (r < t.e0) t.e0 = r;
#pragma unroll
    for (int stride = 16; stride > 0; stride >>= 1) cmpx(t.e0, stride, (lane & stride) == 0);
  }
  t.worst = __shfl_sync(0xffffffffu, t.e0, k - 1);
}

// all 32 lanes call this with their candidate (valid=false for padding lanes)
template <bool WIDE>
__device__ __forceinline__ void topk_offer(WarpTopK& t, int k, int lane, bool valid, float cd, int ci) {
  const tkey c = make_key(cd, ci);
  const bool pass = valid && c < t.worst;
  unsigned m = __ballot_sync(0xffffffffu, pass);
  if (!WIDE && __popc(m) > 3) {  // many entrants: one sort-merge instead of one insertion each
    topk_merge32(t, k, lane, pass ? c : kKeyInf);
    return;
  }
  while (m) {
    int src = __ffs(m) - 1;
    m &= m - 1;
    tkey n = __shfl_sync(0xffffffffu, c, src);
    if (!(n < t.worst)) continue;  // worst moved since the ballot (warp-uniform branch)
    int p = __popc(__ballot_sync(0xffffffffu, t.e0 < n));  // rank of the new entry
    tkey up0 = __shfl_up_sync(0xffffffffu, t.e0, 1);
    const int kr = k - 1;
    if (WIDE) {
      p += __popc(__ballot_sync(0xffffffffu, t.e1 < n));
      tkey up1 = __shfl_up_sync(0xffffffffu, t.e1, 1);
      tkey carry = __shfl_sync(0xffffffffu, t.e0, 31);  // rank 31 -> 32 crosses registers
      int r1 = 32 + lane;
      if (r1 > p) t.e1 = (lane == 0) ? carry : up1;
      else if (r1 == p) t.e1 = n;
    }
    if (lane > p) t.e0 = up0;
    else if (lane == p) t.e0 = n;
    if (WIDE) {
      tkey w0 = __shfl_sync(0xffffffffu, t.e0, kr & 31), w1 = __shfl_sync(0xffffffffu, t.e1, kr & 31);
      t.worst = (kr < 32) ? w0 : w1;
    } else {
      t.worst = __shfl_sync(0xffffffffu, t.e0, kr);
    }
  }
}

// scan one contiguous run of the sorted array; the 32-point batches are dealt round-robin to `nw` cooperating warps (warp `wi`
// takes batches wi, wi+nw, ...), four loads in flight
template <bool WIDE>
__device__ __forceinline__ void scan_run_strided(WarpTopK& t, int k, int lane, float4 q, const float4* __restrict__ sorted, int start, int count, int wi, int nw) {
  constexpr int U = 4;
  for (int off = wi * 32; off < count; off += 32 * U * nw) {
    float4 c[U];
    bool valid[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      int j = off + u * 32 * nw + lane;
      valid[u] = j < count;
      c[u] = valid[u] ? __ldg(&sorted[start + j]) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < U; u++)
      if (off + u * 32 * nw < count) topk_offer<WIDE>(t, k, lane, valid[u], knn_d2(q, c[u]), __float_as_int(c[u].w));
  }
}

constexpr int kKnnGridWarps = 16;  // warps per block of the cooperative kernel (a whole-cloud item is 17 k .. 1 M candidates)

// Block-cooperative continuation for the deferred queries: the 8 warps of a block split the candidates of one query -- the runs
// of the 27 cells of its block at the recorded level, or the whole cloud -- each keeps its own sorted top-k, warp 0 merges the
// eight lists through shared memory.  The block at that level contains the k nearest by construction (k_knn_search step 2).
template <bool WIDE>
__global__ void __launch_bounds__(kKnnGridWarps * 32) k_knn_deferred(GridArgs a) {
  __shared__ tkey se[kKnnGridWarps][64];
  __shared__ int s_next;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int k = a.k, L = a.L;
  const GridGeom g = grid_geom(a.bbox_min, a.bbox_max, L);
  const int n_items = *a.defer_count;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) s_next = atomicAdd(a.defer_cursor, 1);
    __syncthreads();
    const int h = s_next;
    if (h >= n_items) return;
    const int2 item = a.defer_queue[h];
    const float4 q = __ldg(&a.sorted[item.x]);
    const int qi = __float_as_int(q.w);
    WarpTopK t;
    topk_reset(t);
    if (item.y < L) {
      const int l = item.y;
      const int3 c0 = grid_cell0(g, q.x, q.y, q.z);
      const int cl_max = g.cmax >> l;
      int st = 0, en = 0;
      if (lane < 27) {
        const int cx = (c0.x >> l) + lane / 9 - 1, cy = (c0.y >> l) + (lane / 3) % 3 - 1, cz = (c0.z >> l) + lane % 3 - 1;
        if ((unsigned)cx <= (unsigned)cl_max && (unsigned)cy <= (unsigned)cl_max && (unsigned)cz <= (unsigned)cl_max) {
          if (!cell_range(a, (morton3(cx, cy, cz) << 4) | (unsigned)l, st, en)) st = en = 0;
        }
      }
      for (int c = 0; c < 27; c++) {
        const int s0 = __shfl_sync(0xffffffffu, st, c), e0 = __shfl_sync(0xffffffffu, en, c);
        if (e0 > s0) scan_run_strided<WIDE>(t, k, lane, q, a.sorted, s0, e0 - s0, wid, kKnnGridWarps);
      }
    } else {
      scan_run_strided<WIDE>(t, k, lane, q, a.sorted, 0, a.n, wid, kKnnGridWarps);
    }
    // merge the per-warp lists in warp 0
    se[wid][lane] = t.e0;
    se[wid][32 + lane] = t.e1;
    __syncthreads();
    if (wid == 0) {
      for (int ww = 1; ww < kKnnGridWarps; ww++) {
        tkey e = se[ww][lane];
        topk_offer<WIDE>(t, k, lane, lane < k, __uint_as_float((unsigned)(e >> 32)), key_index(e));
        if (WIDE) {
          e = se[ww][32 + lane];
          topk_offer<WIDE>(t, k, lane, 32 + lane < k, __uint_as_float((unsigned)(e >> 32)), key_index(e));
        }
      }
      int* row = a.nbr + (size_t)qi * k;
      if (lane < k) row[lane] = key_index(t.e0);
      if (WIDE && 32 + lane < k) row[32 + lane] = key_index(t.e1);
    }
  }
}

// regulariser over voxel covariances (NDT).  The finalised covariance (S_rc - mean_r * S_c)/n is symmetric only up to rounding;
// Eigen's selfadjointView<Lower> reads the lower triangle, which is what the packed record holds.
__global__ void k_regularize_voxels(VoxelRec* __restrict__ vox, const int* __restrict__ nv_ptr, int method) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= *nv_ptr) return;
  VoxelRec r = vox[v];
  float c[9] = {r.c0.x, r.c0.y, r.c0.z, r.c0.y, r.c0.w, r.c1.x, r.c0.z, r.c1.x, r.c1.y};
  regularize_cov(c, method);
  r.c0 = make_float4(c[0], 0.5f * (c[1] + c[3]), 0.5f * (c[2] + c[6]), c[4]);
  r.c1 = make_float4(0.5f * (c[5] + c[7]), c[8], 0.f, 0.f);
  vox[v] = r;
}

// ---------------------------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------------------------
cudaError_t launch_regularize_voxels(VoxelRec* vox, const int* nv_ptr, int vmax, int method, cudaStream_t stream) {
  k_regularize_voxels<<<(vmax + 127) / 128, 128, 0, stream>>>(vox, nv_ptr, method);
  return cudaGetLastError();
}

size_t knn_smem_bytes(int k) { return sizeof(float4) * kKnnTile + (size_t)k * kKnnThreads * (sizeof(float) + sizeof(int)); }

cudaError_t launch_knn_bruteforce(const float4* pts, int n, int k, int* nbr, cudaStream_t stream) {
  // per device and thread-safe: set on every call (a host-side attribute write; this engine is the A/B legacy path)
  cudaError_t e = cudaFuncSetAttribute(k_knn_bruteforce, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)knn_smem_bytes(kMaxK));
  if (e != cudaSuccess) return e;
  k_knn_bruteforce<<<(n + kKnnThreads - 1) / kKnnThreads, kKnnThreads, knn_smem_bytes(k), stream>>>(pts, n, k, nbr);
  return cudaGetLastError();
}

size_t knn_grid_scratch_bytes(int n, int* levels_out, unsigned* table_size_out) {
  int L = 8;
  for (long m = 16384; m * 4 <= (long)n && L < kGridMaxLevels; m *= 4) L++;
  if (n < 4096) L = 6;
  unsigned T = 1024;
  while (T < 4u * (unsigned)n) T <<= 1;
  if (levels_out) *levels_out = L;
  if (table_size_out) *table_size_out = T;
  const size_t sort_bytes = (sort_scratch_bytes(n, sort_num_passes(3 * (L + 1))) + 15) & ~(size_t)15;
  return 4096 + (size_t)T * sizeof(CellEntry) + sort_bytes + (size_t)n * (8 + 8 + 4 + 4 + 16 + 8) + 256;
}

// scratch layout:  [0xFF-filled : bbox min (16 B) | cell table]
//                  [zero-filled : bbox max (16 B) | counters (256 B) | sort scratch (digit histograms, tickets, look-back state)]
//                  [uninitialised: Morton codes x2 | sort values x2 | sorted points | deferred-query queue]
// q_begin/q_end: sorted positions whose neighbours are searched (whole cloud: 0, n); the build always covers the whole cloud.
cudaError_t launch_knn_grid(const float4* pts, int n, int k, int* nbr, unsigned char* scratch, size_t scratch_bytes, int force_bruteforce, int q_begin, int q_end, int* launches,
                            const float4** sorted_out, cudaStream_t stream) {
  int L;
  unsigned T;
  size_t need = knn_grid_scratch_bytes(n, &L, &T);
  if (scratch_bytes < need || (reinterpret_cast<uintptr_t>(scratch) & 15)) return cudaErrorInvalidValue;
  if (q_end > n) q_end = n;
  if (q_begin < 0) q_begin = 0;
  const int key_bits = 3 * (L + 1);
  const int passes = sort_num_passes(key_bits);
  GridArgs a;
  a.pts = pts; a.n = n; a.k = k; a.L = L; a.tmask = T - 1; a.nbr = nbr; a.q_begin = q_begin; a.q_end = q_end;
  unsigned char* p = scratch;
  unsigned char* ff_begin = p;
  a.bbox_min = reinterpret_cast<unsigned*>(p); p += 16;
  a.table = reinterpret_cast<CellEntry*>(p); p += (size_t)T * sizeof(CellEntry);
  const size_t ff_bytes = (size_t)(p - ff_begin);
  unsigned char* z_begin = p;
  a.bbox_max = reinterpret_cast<unsigned*>(p); p += 16;
  int* counters = reinterpret_cast<int*>(p); p += 256;
  a.level_hist = counters;  // [0 .. kGridMaxLevels + 1]
  a.l_min = counters + 16;
  a.done_blocks = reinterpret_cast<unsigned*>(counters + 17);
  a.defer_count = counters + 18;
  a.defer_cursor = counters + 19;
  unsigned char* sort_scratch = p;
  p += (sort_scratch_bytes(n, passes) + 15) & ~(size_t)15;
  const size_t z_bytes = (size_t)(p - z_begin);
  unsigned long long* codes0 = reinterpret_cast<unsigned long long*>(p); p += (size_t)n * 8;
  unsigned long long* codes1 = reinterpret_cast<unsigned long long*>(p); p += (size_t)n * 8;
  unsigned* vals0 = reinterpret_cast<unsigned*>(p); p += (size_t)n * 4;
  unsigned* vals1 = reinterpret_cast<unsigned*>(p); p += (size_t)n * 4;
  p = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p) + 15) & ~(uintptr_t)15);
  a.sorted = reinterpret_cast<float4*>(p); p += (size_t)n * 16;
  a.defer_queue = reinterpret_cast<int2*>(p); p += (size_t)n * 8;
  a.codes = codes0;
  if (sorted_out) *sorted_out = a.sorted;
  cudaError_t e;
  int nl = 0;
  const int nb = (n + 255) / 256;
  if ((e = cudaMemsetAsync(ff_begin, 0xFF, ff_bytes, stream)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(z_begin, 0, z_bytes, stream)) != cudaSuccess) return e;
  k_grid_bbox<<<nb < 4 * kNumSMs ? nb : 4 * kNumSMs, 256, 0, stream>>>(pts, n, a.bbox_min, a.bbox_max);
  k_grid_codes<<<nb < 8 * kNumSMs ? nb : 8 * kNumSMs, kSortThreads, 0, stream>>>(a, passes, reinterpret_cast<unsigned*>(sort_scratch));
  nl += 2;
  if ((e = launch_sort_pairs<unsigned long long>(codes0, vals0, codes1, vals1, n, key_bits, sort_scratch, true, pts, a.sorted, &nl, stream)) != cudaSuccess) return e;
  a.codes = (passes & 1) ? codes1 : codes0;
  k_grid_levels<<<nb < 4 * kNumSMs ? nb : 4 * kNumSMs, 256, 0, stream>>>(a);
  k_grid_table<<<dim3(nb, L), 256, 0, stream>>>(a);
  nl += 2;
  const int nq = q_end > q_begin ? q_end - q_begin : 0;
  if (nq > 0) {
    const int sblocks = (nq + kSearchWarps - 1) / kSearchWarps;
    if (k <= 32) k_knn_search<false><<<sblocks, kSearchWarps * 32, 0, stream>>>(a, force_bruteforce);
    else k_knn_search<true><<<sblocks, kSearchWarps * 32, 0, stream>>>(a, force_bruteforce);
    int hblocks = (nq + kKnnGridWarps - 1) / kKnnGridWarps;
    if (hblocks > 4 * kNumSMs) hblocks = 4 * kNumSMs;  // persistent: items pulled from a counter
    if (k <= 32) k_knn_deferred<false><<<hblocks, kKnnGridWarps * 32, 0, stream>>>(a);
    else k_knn_deferred<true><<<hblocks, kKnnGridWarps * 32, 0, stream>>>(a);
    nl += 2;
  }
  if (launches) *launches = nl;
  return cudaGetLastError();
}

cudaError_t launch_covariance_knn(const float4* pts, const int* nbr, int n, int k, int method, float4* covA, float2* covB, cudaStream_t stream) {
  k_covariance_knn<<<(n + 127) / 128, 128, 0, stream>>>(pts, nbr, n, k, method, covA, covB);
  return cudaGetLastError();
}

cudaError_t launch_covariance_knn_sharded(const float4* pts, const int* nbr, const float4* sorted, int pos_begin, int pos_end, int k, int method, float4* const* covA_peers,
                                         float2* const* covB_peers, int nranks, cudaStream_t stream) {
  if (nranks < 1 || nranks > 8) return cudaErrorInvalidValue;
  CovPeers peers;
  for (int r = 0; r < 8; r++) { peers.covA[r] = r < nranks ? covA_peers[r] : nullptr; peers.covB[r] = r < nranks ? covB_peers[r] : nullptr; }
  peers.nranks = nranks;
  const int cnt = pos_end - pos_begin;
  if (cnt > 0) k_covariance_knn_sharded<<<(cnt + 127) / 128, 128, 0, stream>>>(pts, nbr, sorted, pos_begin, pos_end, k, method, peers);
  return cudaGetLastError();
}

cudaError_t launch_covariance_rbf(const float4* pts, int n, float exp_factor, float max_dist, int method, float* boxes, float4* covA, float2* covB, cudaStream_t stream) {
  k_rbf_block_boxes<<<(n + kRbfBlock - 1) / kRbfBlock, 128, 0, stream>>>(pts, n, boxes);
  const size_t smem = sizeof(float4) * kRbfLanes * kRbfTileStride;
  cudaError_t e = cudaFuncSetAttribute(k_covariance_rbf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_covariance_rbf<<<(n + kRbfQueries - 1) / kRbfQueries, 128, smem, stream>>>(pts, n, exp_factor, max_dist, method, boxes, covA, covB);
  return cudaGetLastError();
}

}  // namespace vgicp
