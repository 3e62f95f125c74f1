// vgicp_stage1.cuh -- launchers of the stage 1 kernels (vgicp_stage1.cu, compiled with --fmad=false).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace vgicp {

struct VoxelRec {
  float4 mean_n;  // mean xyz, num_points as int bits in w
  float4 c0;      // cxx cxy cxz cyy
  float4 c1;      // cyz czz 0 0
};

constexpr int kMaxK = 64;       // k-NN list capacity
constexpr int kRbfBlock = 512;  // covariance_estimation_rbf.cu:60 BLOCK_SIZE

// exact k-NN of every point inside its own cloud (k <= 64), rows ascending in (d2, index), on a Morton-ordered multi-level grid: one
// warp per query, a block-cooperative scan for the queries the grid does not narrow down (every query of a cloud below 256 points);
// scratch from knn_grid_scratch_bytes(), 16-byte aligned.  [q_begin, q_end): the sorted positions whose rows are computed (0, n = all;
// a slice per rank when stage 1 is sharded)
size_t knn_grid_scratch_bytes(int n, int* levels_out, unsigned* table_size_out);
cudaError_t launch_knn_grid(const float4* pts, int n, int k, int* nbr, unsigned char* scratch, size_t scratch_bytes, int q_begin, int q_end, int* launches,
                            const float4** sorted_out, cudaStream_t stream);
// covariances of the points at sorted positions [pos_begin, pos_end) of that grid, stored into the covariance arrays of all `nranks`
// ranks (peer-mapped pointers; the own arrays included)
cudaError_t launch_covariance_knn_sharded(const float4* pts, const int* nbr, const float4* sorted, int pos_begin, int pos_end, int k, int method, float4* const* covA_peers,
                                         float2* const* covB_peers, int nranks, cudaStream_t stream);
// covariance_estimation + covariance_regularization(method) fused; symmetric-packed output
cudaError_t launch_covariance_knn(const float4* pts, const int* nbr, int n, int k, int method, float4* covA, float2* covB, cudaStream_t stream);
// covariance_estimation_rbf + covariance_regularization(method); boxes: scratch of 6 floats per 512-point block (2 launches)
cudaError_t launch_covariance_rbf(const float4* pts, int n, float exp_factor, float max_dist, int method, float* boxes, float4* covA, float2* covB, cudaStream_t stream);

// covariance_regularization(method) over the covariances of a voxel array (NDT: MIN_EIG on voxel covariances, ndt_cuda.cu:129,140);
// launched for `vmax` voxels, the exact count is read from *nv_ptr on the device
cudaError_t launch_regularize_voxels(VoxelRec* vox, const int* nv_ptr, int vmax, int method, cudaStream_t stream);

}  // namespace vgicp
