// vgicp_local_map.cuh -- kernels of the local-map operations (vgicp_append_source_to_target, vgicp_thin_target,
// vgicp_crop_target): the target cloud grows by the registered source and is compacted by a voxel cap and a crop, all in place on
// the device, so that scan-to-map odometry never moves the map over PCIe.  Included after vgicp_kernels.cuh (Pose,
// transform_point, vgicp_scan.cuh, vgicp_sort.cuh).  The arithmetic the header documents is spelled as IEEE single operations (__f*_rn): this
// unit is compiled with contraction on.
#pragma once
#include <cuda_runtime.h>

namespace vgicp {

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

// Crop, pass 1: point i passes when d^2 = (dx dx + dy dy) + dz dz <= r2 (dx = p.x - c.x, ...) or, when `keep` is given, when
// keep[i] != 0 (the radius is then not tested: a carve keeps non-finite points); rank[i] = number of passing points before i
// (block_rank), or -1.  The total lands in *count.
__global__ void __launch_bounds__(kRankThreads) k_crop_rank(const float4* __restrict__ pts, const unsigned char* __restrict__ keep, int n, float cx, float cy, float cz,
                                                            float r2, int* __restrict__ rank, int* __restrict__ count, unsigned long long* state_words, unsigned epoch) {
  const int i = blockIdx.x * kRankThreads + threadIdx.x;
  int flag = 0;
  if (i < n) {
    if (keep) {
      flag = keep[i] ? 1 : 0;
    } else {
      const float4 p = pts[i];
      const float dx = __fsub_rn(p.x, cx), dy = __fsub_rn(p.y, cy), dz = __fsub_rn(p.z, cz);
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      flag = d2 <= r2 ? 1 : 0;
    }
  }
  const int r = block_rank(flag, state_words, epoch, count);
  if (i < n) rank[i] = flag ? r : -1;
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

// Thinning (vgicp_thin_target): row i is kept iff fewer than M earlier rows share its cell c_a = floorf(p_a * inv).  The rows are
// sorted stably by a u64 cell key, so the rows of one cell are contiguous and in array order; sorted position j is then kept iff
// j < M or key[j - M] != key[j].  k_crop_rank with the resulting mask (and r2 = +inf) and k_crop_scatter compact the target.
constexpr int kThinBoxThreads = 256;

// one pass over the target: the cells' box (kBoxWords), the number of non-finite points in word 6 and a cell outside
// [-2^31, 2^31) in word 7 (st zeroed by the caller)
__global__ void __launch_bounds__(kThinBoxThreads) k_thin_box(const float4* __restrict__ pts, int n, float inv, unsigned* __restrict__ st) {
  unsigned mx[6] = {0, 0, 0, 0, 0, 0}, nonfinite = 0, range = 0;
  for (int i = blockIdx.x * kThinBoxThreads + threadIdx.x; i < n; i += gridDim.x * kThinBoxThreads) {
    const float4 p = pts[i];
    int c[3];
    const int s = cell_of(p.x, p.y, p.z, inv, 0, c);
    nonfinite += s == 0;
    range |= s == 2;
    if (s == 1) box_add(mx, c);
  }
  box_flush(mx, nonfinite, range, st);
}

// key of every point, (c_x - min_x) | (c_y - min_y) << b_x | (c_z - min_z) << (b_x + b_y), and the digit counts of all sort passes
// (every cell is valid: the box pass refused the target otherwise).  sh_x / sh_z: the shifts of the y and z fields; a field of
// width 0 is always 0, which also covers a shift of 64.
__global__ void __launch_bounds__(kSortThreads) k_thin_keys(const float4* __restrict__ pts, int n, float inv, int3 lo, int sh_y, int sh_z, int passes,
                                                            unsigned long long* __restrict__ keys, unsigned* __restrict__ hist) {
  __shared__ unsigned sh[kSortMaxPasses * kSortBins];
  sort_hist_zero(sh, passes);
  const int n_round = (n + 31) & ~31;
  for (int i = blockIdx.x * kSortThreads + threadIdx.x; i < n_round; i += gridDim.x * kSortThreads) {  // warp-uniform trip count
    const bool valid = i < n;
    unsigned long long key = 0;
    if (valid) {
      const float4 p = pts[i];
      int c[3];
      cell_of(p.x, p.y, p.z, inv, 0, c);
      const unsigned long long dy = (unsigned)c[1] - (unsigned)lo.y, dz = (unsigned)c[2] - (unsigned)lo.z;
      key = (unsigned long long)((unsigned)c[0] - (unsigned)lo.x) | (dy ? dy << sh_y : 0ull) | (dz ? dz << sh_z : 0ull);
      keys[i] = key;
    }
    sort_hist_add(sh, passes, valid, key);
  }
  sort_hist_flush(sh, passes, hist);
}

// sorted position j is kept iff j < M or key[j - M] != key[j]; the flag goes to the point's original index (vals == nullptr: the
// keys were not sorted, sorted position = original index)
__global__ void k_thin_keep(const unsigned long long* __restrict__ keys, const unsigned* __restrict__ vals, int n, int M, unsigned char* __restrict__ keep) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const bool k = j < M || keys[j - M] != keys[j];
  keep[vals ? vals[j] : (unsigned)j] = k ? 1 : 0;
}

// Carving (vgicp_carve_target): the scan's range image, then one test per map point against the least range in its window.  The
// pixel and the range follow the header's recipe; a point has a pixel iff carve_pixel returns true.
struct CarveImage {
  int W, H;
  float wq, e_lo, inv_de;  // W * 0.25f, (float)tan(elevation_min), (float)(H / (tan(elevation_max) - tan(elevation_min)))
};

__device__ __forceinline__ bool carve_pixel(const CarveImage& im, float x, float y, float z, int* row, int* col, float* r) {
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;
  const float s = __fadd_rn(fabsf(x), fabsf(y));
  if (s == 0.0f) return false;
  const float q = __fdiv_rn(fabsf(y), s);
  const float a = y >= 0.0f ? (x >= 0.0f ? q : __fsub_rn(2.0f, q)) : (x < 0.0f ? __fadd_rn(2.0f, q) : __fsub_rn(4.0f, q));
  const float xy = __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y));
  const float u = __fmul_rn(__fsub_rn(__fdiv_rn(z, __fsqrt_rn(xy)), im.e_lo), im.inv_de);
  if (!(u >= 0.0f && u < (float)im.H)) return false;  // (also a NaN or infinite u when x x + y y underflows)
  const int c = (int)floorf(__fmul_rn(a, im.wq));
  *col = c == im.W ? 0 : c;
  *row = (int)floorf(u);
  *r = __fsqrt_rn(__fadd_rn(xy, __fmul_rn(z, z)));
  return true;
}

// one thread per source point: the least range per pixel (img filled with 0xFFFFFFFF, "no return", by the caller)
__global__ void k_carve_image(const float4* __restrict__ src, int n, const CarveImage im, unsigned* __restrict__ img) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = src[i];
  int row, col;
  float r;
  if (carve_pixel(im, p.x, p.y, p.z, &row, &col, &r)) atomicMin(img + (size_t)row * im.W + col, __float_as_uint(r));
}

// one thread per target point: into the sensor frame by Ti (row-major 3x4), the pixel, the least range r_min in the window, and
// keep[i] = 0 iff r < r_min - (margin + margin_rel r_min)
__global__ void k_carve_keep(const float4* __restrict__ pts, int n, const Pose Ti, const CarveImage im, const unsigned* __restrict__ img, int window, float margin,
                             float margin_rel, unsigned char* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 m = pts[i];
  float s[3];
#pragma unroll
  for (int j = 0; j < 3; j++)
    s[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(Ti.r[j * 3 + 0], m.x), __fmul_rn(Ti.r[j * 3 + 1], m.y)), __fmul_rn(Ti.r[j * 3 + 2], m.z)), Ti.t[j]);
  int row, col;
  float r;
  bool removed = false;
  if (carve_pixel(im, s[0], s[1], s[2], &row, &col, &r)) {
    unsigned best = 0xFFFFFFFFu;
    const int r0 = row - window < 0 ? 0 : row - window, r1 = row + window >= im.H ? im.H - 1 : row + window;
    for (int rr = r0; rr <= r1; rr++) {
      const unsigned* line = img + (size_t)rr * im.W;
      for (int dc = -window; dc <= window; dc++) {
        int cc = (col + dc) % im.W;
        if (cc < 0) cc += im.W;
        best = min(best, __ldg(line + cc));
      }
    }
    if (best != 0xFFFFFFFFu) {
      const float r_min = __uint_as_float(best);
      removed = r < __fsub_rn(r_min, __fadd_rn(margin, __fmul_rn(margin_rel, r_min)));
    }
  }
  keep[i] = removed ? 0 : 1;
}

}  // namespace vgicp
