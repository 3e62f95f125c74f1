// vgicp_local_map.cuh -- kernels of the local-map operations (vgicp_append_source_to_target, vgicp_crop_target): the target
// cloud grows by the registered source and is compacted by a crop, both in place on the device, so that scan-to-map odometry
// never moves the map over PCIe.  Included after vgicp_kernels.cuh (Pose, transform_point).  The arithmetic the header
// documents is spelled as IEEE single operations (__f*_rn): this unit is compiled with contraction on.
#pragma once
#include <cuda_runtime.h>

namespace vgicp {

constexpr int kCropThreads = 1024;  // points per block of the crop's scan (one look-back state word per block)

// Appended row i: point = transform_point(T, a_i), the bytes vgicp_transform_source returns; covariance = R C_i R^T with
//   M_ik = (R_i0 C_0k + R_i1 C_1k) + R_i2 C_2k,   N_ij = (M_i0 R_j0 + M_i1 R_j1) + M_i2 R_j2,
// stored symmetric-packed like set_covariances: the diagonal of N, and 0.5f (N_ij + N_ji) off it.
__global__ void k_append_transformed(const float4* __restrict__ src_pts, const float4* __restrict__ src_covA, const float2* __restrict__ src_covB, int n, const Pose T,
                                     float4* __restrict__ dst_pts, float4* __restrict__ dst_covA, float2* __restrict__ dst_covB) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = src_pts[i];
  const float3 q = transform_point(T, p.x, p.y, p.z);
  dst_pts[i] = make_float4(q.x, q.y, q.z, 0.0f);
  const float4 a = src_covA[i];
  const float2 b = src_covB[i];
  const float C[9] = {a.x, a.y, a.z, a.y, a.w, b.x, a.z, b.x, b.y};  // row-major (symmetric)
  const float* R = T.r;                                            // row-major
  float M[9], N[9];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int k = 0; k < 3; k++) M[r * 3 + k] = __fadd_rn(__fadd_rn(__fmul_rn(R[r * 3 + 0], C[0 + k]), __fmul_rn(R[r * 3 + 1], C[3 + k])), __fmul_rn(R[r * 3 + 2], C[6 + k]));
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) N[r * 3 + c] = __fadd_rn(__fadd_rn(__fmul_rn(M[r * 3 + 0], R[c * 3 + 0]), __fmul_rn(M[r * 3 + 1], R[c * 3 + 1])), __fmul_rn(M[r * 3 + 2], R[c * 3 + 2]));
  dst_covA[i] = make_float4(N[0], __fmul_rn(0.5f, __fadd_rn(N[1], N[3])), __fmul_rn(0.5f, __fadd_rn(N[2], N[6])), N[4]);
  dst_covB[i] = make_float2(__fmul_rn(0.5f, __fadd_rn(N[5], N[7])), N[8]);
}

// Crop, pass 1: point i passes when d^2 = (dx dx + dy dy) + dz dz <= r2 (dx = p.x - c.x, ...); rank[i] = number of passing points
// before i, or -1.  The total lands in *count.  Block scan, then the decoupled look-back of k_table_assign_ids over the totals
// the preceding blocks publish in `state` (epoch << 32 | total; the epoch changes every launch, so the array never needs clearing).
// A block only ever waits for blocks with a smaller index, which the hardware scheduled before it.
__global__ void __launch_bounds__(kCropThreads) k_crop_rank(const float4* __restrict__ pts, int n, float cx, float cy, float cz, float r2, int* __restrict__ rank,
                                                            int* __restrict__ count, unsigned long long* state_words, unsigned epoch) {
  __shared__ int warp_sums[32];
  __shared__ int s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int i = blockIdx.x * kCropThreads + tid;
  int flag = 0;
  if (i < n) {
    const float4 p = pts[i];
    const float dx = __fsub_rn(p.x, cx), dy = __fsub_rn(p.y, cy), dz = __fsub_rn(p.z, cz);
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    flag = d2 <= r2 ? 1 : 0;
  }
  int v = flag;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) warp_sums[wid] = v;
  __syncthreads();
  if (wid == 0) {
    int w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    warp_sums[lane] = w;
    const int total = __shfl_sync(0xffffffffu, w, 31);
    volatile unsigned long long* state = state_words;
    if (lane == 0) {
      state[blockIdx.x] = ((unsigned long long)epoch << 32) | (unsigned)total;
      __threadfence();
    }
    int base = 0;  // lanes split the predecessors
    for (int p = (int)blockIdx.x - 1 - lane; p >= 0; p -= 32) {
      unsigned long long sv;
      while ((unsigned)((sv = state[p]) >> 32) != epoch) {}
      base += (int)(unsigned)(sv & 0xffffffffULL);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) base += __shfl_xor_sync(0xffffffffu, base, o);
    if (lane == 0) {
      s_base = base;
      if (blockIdx.x == gridDim.x - 1) *count = base + total;
    }
  }
  __syncthreads();
  if (i < n) rank[i] = flag ? s_base + (wid > 0 ? warp_sums[wid - 1] : 0) + v - 1 : -1;
}

// Crop, pass 2: passing point i with rank r >= first goes to row r - first of the output arrays (stable compaction of the newest
// ranks; first = number of passing points dropped by the cap)
__global__ void k_crop_scatter(const float4* __restrict__ pts, const float4* __restrict__ covA, const float2* __restrict__ covB, const int* __restrict__ rank, int n, int first,
                               float4* __restrict__ out_pts, float4* __restrict__ out_covA, float2* __restrict__ out_covB) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = rank[i];
  if (r < first) return;  // failed the radius test (-1), or one of the oldest passing points
  out_pts[r - first] = pts[i];
  out_covA[r - first] = covA[i];
  out_covB[r - first] = covB[i];
}

}  // namespace vgicp
