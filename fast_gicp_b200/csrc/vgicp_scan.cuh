// vgicp_scan.cuh -- device primitives shared by the stable compactions and the cell grids of both native libraries: the block rank
// with its decoupled look-back (voxel ids, crop and thinning, the approximate and the exact voxel grid), and the cell of a point
// with the box of cells (thinning, exact voxel grid).
#pragma once
#include <cuda_runtime.h>

#include "vgicp_devbuf.hpp"

namespace vgicp {

constexpr int kRankThreads = 1024;  // block size of every block_rank kernel (one look-back state word per block)

// Exclusive rank of this thread's flag among the flagged threads of the whole grid, in thread order; call with every thread of a
// kRankThreads block.  Block scan, then a decoupled look-back over the totals the preceding blocks publish in `state_words`
// (epoch << 32 | total; the epoch changes every launch, so the array never needs clearing).  A block only ever waits for blocks
// with a smaller index, which the hardware scheduled before it.  The last block writes the grand total to *total.
__device__ __forceinline__ int block_rank(int flag, unsigned long long* state_words, unsigned epoch, int* total) {
  __shared__ int warp_sums[32];
  __shared__ int s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
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
    const int block_total = __shfl_sync(0xffffffffu, w, 31);
    volatile unsigned long long* state = state_words;
    if (lane == 0) {
      state[blockIdx.x] = ((unsigned long long)epoch << 32) | (unsigned)block_total;
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
      if (blockIdx.x == gridDim.x - 1) *total = base + block_total;
    }
  }
  __syncthreads();
  return s_base + (wid > 0 ? warp_sums[wid - 1] : 0) + v - flag;
}

// A fresh epoch for the look-back state of a block_rank launch of `blocks` blocks on `st`: the array is cleared when it is newly
// allocated (no stale epoch may match) and when the epoch wraps (it restarts at 1).  Each user owns its own state array: two launches
// sharing one on different streams could overwrite each other's words and spin forever.  The epoch is a kernel argument advanced
// here on the host, so a block_rank launch must not be captured into a graph: a replay would wait for a stale epoch.
inline cudaError_t lookback_next(DevBuf<unsigned long long>& state, unsigned& epoch, int blocks, cudaStream_t st) {
  const unsigned long long* before = state.p;
  cudaError_t e = state.reserve((size_t)blocks);
  if (e != cudaSuccess) return e;
  if (state.p != before) {
    e = cudaMemsetAsync(state.p, 0, state.cap * sizeof(unsigned long long), st);
    epoch = 0;
  }
  if (e == cudaSuccess && ++epoch == 0) {
    e = cudaMemsetAsync(state.p, 0, state.cap * sizeof(unsigned long long), st);
    epoch = 1;
  }
  return e;
}

__host__ __device__ inline unsigned cell_enc(int c) { return (unsigned)c ^ 0x80000000u; }  // order-preserving int -> unsigned
__host__ __device__ inline int cell_dec(unsigned u) { return (int)(u ^ 0x80000000u); }

// Cell c = floorf(p * inv) of a point.  0: dropped (a non-finite coordinate, or near the origin when `filter`: (x x + y y) + z z <
// 1e-3, align.cpp's filter), 1: kept with its cell in c, 2: kept but a cell outside the int range
__device__ __forceinline__ int cell_of(float x, float y, float z, float inv, int filter, int c[3]) {
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) return 0;
  if (filter && __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)) < 1e-3f) return 0;
  const float f[3] = {floorf(__fmul_rn(x, inv)), floorf(__fmul_rn(y, inv)), floorf(__fmul_rn(z, inv))};
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (!(f[a] >= -2147483648.0f && f[a] < 2147483648.0f)) return 2;
    c[a] = (int)f[a];
  }
  return 1;
}

// Box of cells: words [0..2] ~enc(min c), [3..5] enc(max c) (unsigned max reductions, zero = empty), [6] a sum, [7] an or; the
// caller zeroes the words before the launch.  Each thread folds its cells into mx with box_add, then the whole block calls box_flush.
constexpr int kBoxWords = 8;

__device__ __forceinline__ void box_add(unsigned (&mx)[6], const int c[3]) {
#pragma unroll
  for (int a = 0; a < 3; a++) {
    mx[a] = max(mx[a], ~cell_enc(c[a]));
    mx[3 + a] = max(mx[3 + a], cell_enc(c[a]));
  }
}

__device__ __forceinline__ void box_flush(unsigned (&mx)[6], unsigned sum, unsigned bits, unsigned* __restrict__ st) {
  __shared__ unsigned sh[kBoxWords];
  if (threadIdx.x < kBoxWords) sh[threadIdx.x] = 0;
  __syncthreads();
  const unsigned full = 0xffffffffu;
#pragma unroll
  for (int a = 0; a < 6; a++) mx[a] = __reduce_max_sync(full, mx[a]);
  sum = __reduce_add_sync(full, sum);
  bits = __reduce_or_sync(full, bits);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 6; a++) atomicMax(&sh[a], mx[a]);
    atomicAdd(&sh[6], sum);
    atomicOr(&sh[7], bits);
  }
  __syncthreads();
  if (threadIdx.x < 6) atomicMax(&st[threadIdx.x], sh[threadIdx.x]);
  else if (threadIdx.x == 6) atomicAdd(&st[6], sh[6]);
  else if (threadIdx.x == 7) atomicOr(&st[7], sh[7]);
}

}  // namespace vgicp
