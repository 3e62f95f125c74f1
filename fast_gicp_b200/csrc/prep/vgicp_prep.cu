// vgicp_prep.cu -- device-side input preparation (include/vgicp_prep_b200.h): near-origin filter + pcl::ApproximateVoxelGrid,
// bit-identical to the serial filter (points and order).  Reference call sites: src/align.cpp:128-147, src/kitti.cpp:80-82,
// src/python/main.cpp:46-62,81-91.  Parity: tests/test_input_prep.py.
//
// Why one block: the filter's 512 history entries are 512 independent sequential chains; thread h of the walk block owns entry h
// and sees the points that hash to it in input order.  Per tile of 2048 staged points every point announces itself to its entry
// (shared-memory atomic append, then the entry sorts its <= 16 tile-local indices: arrival order of the atomics is arbitrary,
// input order is what the filter defines); an entry with more matches in one tile falls back to scanning the staged hashes.
// A flushed centroid is stored at the index of the point that flushed it; a scan over those flags (one block per 1024 points,
// decoupled look-back) gives it the rank the serial filter would have emitted it at, and the entries still holding a voxel at the
// end follow in entry order.
//
// The exact grid (vgicp_prep_voxel_grid, pcl::VoxelGrid) is data-parallel throughout: see "exact grid" below.
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>
#include <new>
#include <string>

#include "../vgicp_scan.cuh"
#include "../vgicp_sort.cuh"
#include "vgicp_prep_b200.h"

using namespace vgicp;

namespace {

constexpr int kHist = 512;   // pcl::ApproximateVoxelGrid histsize_ (default; the reference never changes it)
constexpr int kTile = 2048;  // points staged per round of the walk
constexpr int kCap = 16;     // tile-local matches per entry kept in the fast list
constexpr unsigned short kNoEntry = 0xFFFF;

// x y z -> float4 copy + history entry (kNoEntry for a point the near-origin filter drops)
__global__ void k_prep_keys(const float* __restrict__ xyz, size_t stride_f, int n, float inv_leaf, int filter, float4* __restrict__ pts4, unsigned short* __restrict__ entry) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = xyz + (size_t)i * stride_f;
  const float x = p[0], y = p[1], z = p[2];
  // align.cpp:131: squaredNorm() < 1e-3, evaluated as (x*x + y*y) + z*z without contraction (Eigen's unrolled redux order)
  const float sq = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
  const bool keep = !(filter && sq < 1e-3f);
  const int ix = (int)floorf(__fmul_rn(x, inv_leaf)), iy = (int)floorf(__fmul_rn(y, inv_leaf)), iz = (int)floorf(__fmul_rn(z, inv_leaf));
  const long long hl = (long long)ix * 7171 + (long long)iy * 3079 + (long long)iz * 4231;
  pts4[i] = make_float4(x, y, z, 0.f);
  entry[i] = keep ? (unsigned short)(hl & (long long)(kHist - 1)) : kNoEntry;
}

// Per-point float fields averaged next to x y z (vgicp_prep_approximate_voxel_grid_fields); the kernels below are templates on the
// field count F, and F = 0 is vgicp_prep_approximate_voxel_grid.  A flushed field centroid goes to flushed[F * i + j], i the index of
// the flushing point (beside the float4 of its xyz), a held one to tail[F * h + j]; both are read only where the float4 flag is set.
constexpr int kMaxFields = 8;
struct FieldArgs {
  const float* in;  // the input records (device), stride_f floats apart
  size_t stride_f;
  int off[kMaxFields];  // offset of field j in floats
  float* flushed;       // [n][F]
  float* tail;          // [kHist][F]
};

template <int F>
struct FieldSums {
  float s[F];
};
template <>
struct FieldSums<0> {};

template <int F>
struct Entry {  // one history entry, in the registers of its thread
  int ix, iy, iz, count;
  float sx, sy, sz;
  FieldSums<F> f;
};

template <int F>
__device__ __forceinline__ void entry_step(Entry<F>& e, int i, const float4* __restrict__ pts4, float inv_leaf, float4* __restrict__ flushed, const FieldArgs& fa) {
  const float4 p = pts4[i];
  const int ix = (int)floorf(__fmul_rn(p.x, inv_leaf)), iy = (int)floorf(__fmul_rn(p.y, inv_leaf)), iz = (int)floorf(__fmul_rn(p.z, inv_leaf));
  if (e.count && (e.ix != ix || e.iy != iy || e.iz != iz)) {  // another voxel lands on this entry: emit the centroid held so far
    const float c = (float)e.count;
    flushed[i] = make_float4(__fdiv_rn(e.sx, c), __fdiv_rn(e.sy, c), __fdiv_rn(e.sz, c), 1.f);
    e.count = 0;
    e.sx = e.sy = e.sz = 0.f;
    if constexpr (F > 0) {
#pragma unroll
      for (int j = 0; j < F; j++) {
        fa.flushed[(size_t)F * i + j] = __fdiv_rn(e.f.s[j], c);
        e.f.s[j] = 0.f;
      }
    }
  }
  e.ix = ix; e.iy = iy; e.iz = iz;
  e.count++;
  e.sx = __fadd_rn(e.sx, p.x); e.sy = __fadd_rn(e.sy, p.y); e.sz = __fadd_rn(e.sz, p.z);
  if constexpr (F > 0) {
    const float* r = fa.in + (size_t)i * fa.stride_f;
#pragma unroll
    for (int j = 0; j < F; j++) e.f.s[j] = __fadd_rn(e.f.s[j], r[fa.off[j]]);
  }
}

template <int F>
__global__ void __launch_bounds__(kHist) k_prep_walk(const float4* __restrict__ pts4, const unsigned short* __restrict__ entry, int n, float inv_leaf, float4* __restrict__ flushed,
                                                     float4* __restrict__ tail, const FieldArgs fa) {
  __shared__ unsigned short sh_entry[kTile];
  __shared__ int cnt[kHist];
  __shared__ unsigned short list[kHist * kCap];
  const int h = threadIdx.x;
  Entry<F> e;
  e.ix = e.iy = e.iz = e.count = 0;
  e.sx = e.sy = e.sz = 0.f;
  if constexpr (F > 0) {
#pragma unroll
    for (int j = 0; j < F; j++) e.f.s[j] = 0.f;
  }
  for (int base = 0; base < n; base += kTile) {
    cnt[h] = 0;
    __syncthreads();
    for (int j = h; j < kTile; j += kHist) {
      const int i = base + j;
      const unsigned short t = i < n ? entry[i] : kNoEntry;
      sh_entry[j] = t;
      if (t != kNoEntry) {
        const int p = atomicAdd(&cnt[t], 1);
        if (p < kCap) list[(int)t * kCap + p] = (unsigned short)j;
      }
    }
    __syncthreads();
    const int c = cnt[h];
    if (c > 0 && c <= kCap) {
      unsigned short* mine = &list[h * kCap];  // this thread's segment: sort the tile-local indices ascending (= input order)
      for (int a = 1; a < c; a++) {
        const unsigned short v = mine[a];
        int b = a - 1;
        while (b >= 0 && mine[b] > v) { mine[b + 1] = mine[b]; b--; }
        mine[b + 1] = v;
      }
      for (int q = 0; q < c; q++) entry_step(e, base + (int)mine[q], pts4, inv_leaf, flushed, fa);
    } else if (c > kCap) {  // a run of points on one entry (e.g. the invalid returns at the origin): walk the staged tile
      for (int j = 0; j < kTile; j++)
        if (sh_entry[j] == (unsigned short)h) entry_step(e, base + j, pts4, inv_leaf, flushed, fa);
    }
    __syncthreads();  // the tile's lists are consumed before the next tile overwrites them
  }
  if (e.count) {
    const float c = (float)e.count;
    tail[h] = make_float4(__fdiv_rn(e.sx, c), __fdiv_rn(e.sy, c), __fdiv_rn(e.sz, c), 1.f);
    if constexpr (F > 0) {
#pragma unroll
      for (int j = 0; j < F; j++) fa.tail[F * h + j] = __fdiv_rn(e.f.s[j], c);
    }
  } else {
    tail[h] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// rank of every flushed centroid = number of flushes at smaller point indices (block_rank, one block per kRankThreads points);
// output records of 3 + F floats: x y z, then the F fields
template <int F>
__global__ void __launch_bounds__(kRankThreads) k_prep_scatter(const float4* __restrict__ flushed, int n, float* __restrict__ out, size_t cap, unsigned long long* chunk_state,
                                                               unsigned epoch, int* __restrict__ total, const float* __restrict__ fflushed) {
  const int i = blockIdx.x * kRankThreads + threadIdx.x;
  float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n) f = flushed[i];
  const int flag = f.w != 0.f ? 1 : 0;
  const int r = block_rank(flag, chunk_state, epoch, total);
  if (flag) {
    const size_t pos = (size_t)r;
    if (pos < cap) {
      float* o = out + (3 + F) * pos;
      o[0] = f.x; o[1] = f.y; o[2] = f.z;
      if constexpr (F > 0) {
#pragma unroll
        for (int j = 0; j < F; j++) o[3 + j] = fflushed[(size_t)F * i + j];
      }
    }
  }
}

// the entries still holding a voxel, in entry order, behind the flushed centroids
template <int F>
__global__ void __launch_bounds__(kHist) k_prep_tail(const float4* __restrict__ tail, const int* __restrict__ total, float* __restrict__ out, size_t cap, int* __restrict__ n_out,
                                                     const float* __restrict__ ftail) {
  __shared__ int warp_sums[kHist / 32];
  const int h = threadIdx.x, lane = h & 31, wid = h >> 5;
  const float4 f = tail[h];
  const int flag = f.w != 0.f ? 1 : 0;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_sums[wid] = __popc(m);
  __syncthreads();
  int before = 0, all = 0;
  for (int w = 0; w < kHist / 32; w++) {
    const int s = warp_sums[w];
    if (w < wid) before += s;
    all += s;
  }
  const int first = *total;
  if (flag) {
    const size_t pos = (size_t)(first + before + __popc(m & ((1u << lane) - 1u)));
    if (pos < cap) {
      float* o = out + (3 + F) * pos;
      o[0] = f.x; o[1] = f.y; o[2] = f.z;
      if constexpr (F > 0) {
#pragma unroll
        for (int j = 0; j < F; j++) o[3 + j] = ftail[F * h + j];
      }
    }
  }
  if (h == 0) *n_out = first + all;
}

// ---------------------------------------------------------------------------------------------------- exact grid (pcl::VoxelGrid)
// vgicp_prep_voxel_grid: box of the kept points' cells (k_grid_box), one sync to read it back, voxel index keys with their digit
// histograms (k_grid_keys), the library's stable LSD radix sort carrying x y z and the input index (vgicp_sort.cuh), the voxels that
// reach the minimum ranked in key order (k_grid_heads), one warp per voxel summing its points in sorted = input order
// (k_grid_centroids).  Dropped points get the key V = div_x * div_y * div_z, past every voxel, so they sort behind the kept ones.
constexpr int kGridBoxThreads = 256;
constexpr int kGridWarps = 4;                  // warps per centroid block
constexpr int kGridItems = 4;                  // points per lane per round of a centroid warp
constexpr int kGridChunk = 32 * kGridItems;    // points staged per round
// state words: [0..7] the box of the kept points' cells (kBoxWords) with the kept count in [6] and a kept cell outside the int
// range in [7], [8] surviving voxels m
constexpr int kGridState = 9;

__global__ void __launch_bounds__(kGridBoxThreads) k_grid_box(const float* __restrict__ in, size_t stride_f, int n, float inv, int filter, float4* __restrict__ pts4,
                                                              unsigned* __restrict__ st) {
  unsigned mx[6] = {0, 0, 0, 0, 0, 0}, kept = 0, bad = 0;
  for (int i = blockIdx.x * kGridBoxThreads + threadIdx.x; i < n; i += gridDim.x * kGridBoxThreads) {
    const float* p = in + (size_t)i * stride_f;
    const float x = p[0], y = p[1], z = p[2];
    pts4[i] = make_float4(x, y, z, 0.f);
    int g[3];
    const int s = cell_of(x, y, z, inv, filter, g);
    kept += s != 0;
    bad |= s == 2;
    if (s == 1) box_add(mx, g);
  }
  box_flush(mx, kept, bad, st);
}

// key of every point (voxel index, or V for a dropped one) and the digit counts of all sort passes
__global__ void __launch_bounds__(vgicp::kSortThreads) k_grid_keys(const float4* __restrict__ pts4, int n, float inv, int filter, int3 min_b, unsigned div_x, unsigned div_xy,
                                                                   unsigned dropped_key, int passes, unsigned* __restrict__ keys, unsigned* __restrict__ hist) {
  __shared__ unsigned sh[kSortMaxPasses * kSortBins];
  sort_hist_zero(sh, passes);
  const int n_round = (n + 31) & ~31;
  for (int i = blockIdx.x * kSortThreads + threadIdx.x; i < n_round; i += gridDim.x * kSortThreads) {  // warp-uniform trip count
    const bool valid = i < n;
    unsigned key = dropped_key;
    if (valid) {
      const float4 p = pts4[i];
      int g[3];
      if (cell_of(p.x, p.y, p.z, inv, filter, g) == 1)
        key = ((unsigned)g[0] - (unsigned)min_b.x) + ((unsigned)g[1] - (unsigned)min_b.y) * div_x + ((unsigned)g[2] - (unsigned)min_b.z) * div_xy;
      keys[i] = key;
    }
    sort_hist_add(sh, passes, valid, key);
  }
  sort_hist_flush(sh, passes, hist);
}

// the sorted positions that start a voxel reaching the minimum (the run of equal keys starting at p is at least min_points long iff
// key[p + min_points - 1] is still p's key), ranked in key order by block_rank: vstart[rank] = p, st[8] = their number.  One block
// per kRankThreads of the kept points' positions.
__global__ void __launch_bounds__(kRankThreads) k_grid_heads(const unsigned* __restrict__ keys, int kept, unsigned min_points, unsigned long long* chunk_state, unsigned epoch,
                                                             int* __restrict__ vstart, unsigned* __restrict__ st) {
  const int p = blockIdx.x * kRankThreads + threadIdx.x;
  int flag = 0;
  if (p < kept) {
    const unsigned k = keys[p];
    flag = p == 0 || keys[p - 1] != k;
    if (flag && min_points > 1) {
      const long long q = (long long)p + min_points - 1;
      flag = q < kept && keys[q] == k;
    }
  }
  const int r = block_rank(flag, chunk_state, epoch, reinterpret_cast<int*>(st + 8));
  if (flag) vstart[r] = p;
}

// One round of a centroid warp: the run's points among sorted positions base ... base + kGridChunk - 1, x y z and the F fields of
// position base + it * 32 + lane into v[it]; returns how many belong to the run (they are a prefix of the round).
template <int F>
__device__ __forceinline__ int grid_round(const unsigned* __restrict__ keys, const float4* __restrict__ sorted4, int kept, unsigned key, int base, const FieldArgs fa,
                                          float (&v)[kGridItems][3 + F]) {
  const int lane = threadIdx.x & 31;
  int cnt = 0;
#pragma unroll
  for (int it = 0; it < kGridItems; it++) {
    const int p = base + it * 32 + lane;
    const bool in = p < kept && keys[p] == key;
    cnt += __popc(__ballot_sync(0xffffffffu, in));
    const float4 q = in ? sorted4[p] : make_float4(0.f, 0.f, 0.f, 0.f);
    v[it][0] = q.x; v[it][1] = q.y; v[it][2] = q.z;
    if constexpr (F > 0) {
      const float* rec = fa.in + (size_t)__float_as_uint(q.w) * fa.stride_f;
#pragma unroll
      for (int j = 0; j < F; j++) v[it][3 + j] = in ? rec[fa.off[j]] : 0.f;
    }
  }
  return cnt;
}

// One warp per surviving voxel (grid-stride over the ranks), in rounds of kGridChunk sorted positions staged point-major in shared
// memory; lane c < 3 + F adds channel c of the staged points in order while the next round's loads are in flight (a long run is
// bound by its chain of adds, not by load latency).  The run ends at the first position with another key.  Nothing is written
// when m > cap.
template <int F>
__global__ void __launch_bounds__(kGridWarps * 32, 1) k_grid_centroids(const unsigned* __restrict__ keys, const float4* __restrict__ sorted4, int kept,
                                                                    const int* __restrict__ vstart, const unsigned* __restrict__ st, const FieldArgs fa,
                                                                    float* __restrict__ out, size_t cap) {
  constexpr int R = 3 + F, Row = R | 1;  // odd row length: the lanes' staging stores fall in distinct banks
  __shared__ float buf[kGridWarps][kGridChunk * Row];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float* b = buf[w];
  const int m = (int)st[8];
  if ((size_t)m > cap) return;
  for (int r = blockIdx.x * kGridWarps + w; r < m; r += gridDim.x * kGridWarps) {
    const int start = vstart[r];
    const unsigned key = keys[start];
    float v[kGridItems][R];
    int cnt = grid_round<F>(keys, sorted4, kept, key, start, fa, v);
    float s = 0.f;
    int count = 0;
    for (int base = start;; base += kGridChunk) {
#pragma unroll
      for (int it = 0; it < kGridItems; it++) {
        if (it * 32 + lane < cnt) {
#pragma unroll
          for (int c = 0; c < R; c++) b[(it * 32 + lane) * Row + c] = v[it][c];
        }
      }
      __syncwarp();
      const int cur = cnt;
      if (cur == kGridChunk) cnt = grid_round<F>(keys, sorted4, kept, key, base + kGridChunk, fa, v);
      if (lane < R) {
        if (cur == kGridChunk) {
#pragma unroll 32
          for (int q = 0; q < kGridChunk; q++) s = __fadd_rn(s, b[q * Row + lane]);
        } else {
          for (int q = 0; q < cur; q++) s = __fadd_rn(s, b[q * Row + lane]);
        }
      }
      count += cur;
      __syncwarp();
      if (cur < kGridChunk) break;
    }
    if (lane < R) out[(size_t)r * R + lane] = __fdiv_rn(s, (float)count);
  }
}

}  // namespace

struct vgicp_prep_context {
  int device = 0;
  Stream stream;
  std::string err;
  DevBuf<unsigned char> staging;  // host input copied here
  DevBuf<float4> pts4;
  DevBuf<unsigned short> entry;
  DevBuf<float4> flushed;
  DevBuf<float> out;
  DevBuf<unsigned long long> chunk_state;
  unsigned chunk_epoch = 0;
  DevPtr<float4[]> tail;    // [kHist]
  DevPtr<int[]> d_counts;   // [0] flushed total, [1] n_out
  HostPtr<int[]> h_counts;  // pinned
  DevBuf<float> fflushed;  // per-point fields: flushed field centroids [n][F]
  DevBuf<float> ftail;     // ... and those of the entries still holding a voxel [kHist][F]
  // exact grid: sort keys and values (two buffers each), the sorted float4 payload, the sort scratch, the voxel starts
  DevBuf<unsigned> gkeys[2], gvals[2];
  DevBuf<float4> gsorted4;
  DevBuf<unsigned char> gscratch;
  DevBuf<int> gvstart;
  DevPtr<unsigned[]> d_grid;   // [kGridState]
  HostPtr<unsigned[]> h_grid;  // pinned
};

namespace {
int fail(vgicp_prep_handle h, int code, const std::string& msg) {
  if (h) h->err = msg;
  return code;
}
#define PREP_TRY(h, expr)                                                                                   \
  do {                                                                                                      \
    cudaError_t e__ = (expr);                                                                               \
    if (e__ != cudaSuccess) return fail(h, 3, std::string(#expr) + ": " + cudaGetErrorString(e__));         \
  } while (0)
}  // namespace

extern "C" {

int vgicp_prep_create(int device, vgicp_prep_handle* out) {
  if (!out) return 1;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return 5;
  if (device < 0 || device >= ndev) return 1;
  vgicp_prep_context* h = new (std::nothrow) vgicp_prep_context();
  if (!h) return 3;
  h->device = device;
  bool ok = cudaSetDevice(device) == cudaSuccess;
  ok = ok && stream_create(h->stream, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && device_alloc(h->tail, kHist * sizeof(float4)) == cudaSuccess;
  ok = ok && device_alloc(h->d_counts, 2 * sizeof(int)) == cudaSuccess;
  ok = ok && host_alloc(h->h_counts, 2 * sizeof(int), cudaHostAllocDefault) == cudaSuccess;
  ok = ok && device_alloc(h->d_grid, kGridState * sizeof(unsigned)) == cudaSuccess;
  ok = ok && host_alloc(h->h_grid, kGridState * sizeof(unsigned), cudaHostAllocDefault) == cudaSuccess;
  if (!ok) {
    delete h;
    return 3;
  }
  *out = h;
  return 0;
}

void vgicp_prep_destroy(vgicp_prep_handle h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream.get());
  delete h;
}

const char* vgicp_prep_last_error(vgicp_prep_handle h) { return h ? h->err.c_str() : "null handle"; }

}  // extern "C"

namespace {

template <int F>
cudaError_t launch_filter(vgicp_prep_handle h, const float* d_in, size_t stride_f, const int* off, int ni, float inv_leaf, int filter, float* d_out, size_t out_cap, int chunks) {
  FieldArgs fa{};
  fa.in = d_in;
  fa.stride_f = stride_f;
  for (int j = 0; j < F; j++) fa.off[j] = off[j];
  fa.flushed = h->fflushed.p;
  fa.tail = h->ftail.p;
  k_prep_keys<<<(ni + 255) / 256, 256, 0, h->stream.get()>>>(d_in, stride_f, ni, inv_leaf, filter, h->pts4.p, h->entry.p);
  const cudaError_t e = cudaMemsetAsync(h->flushed.p, 0, (size_t)ni * sizeof(float4), h->stream.get());
  if (e != cudaSuccess) return e;
  k_prep_walk<F><<<1, kHist, 0, h->stream.get()>>>(h->pts4.p, h->entry.p, ni, inv_leaf, h->flushed.p, h->tail.get(), fa);
  k_prep_scatter<F><<<chunks, kRankThreads, 0, h->stream.get()>>>(h->flushed.p, ni, d_out, out_cap, h->chunk_state.p, h->chunk_epoch, h->d_counts.get(), h->fflushed.p);
  k_prep_tail<F><<<1, kHist, 0, h->stream.get()>>>(h->tail.get(), h->d_counts.get(), d_out, out_cap, h->d_counts.get() + 1, h->ftail.p);
  return cudaGetLastError();
}

// the device copy of the input: a host input is copied up to the last byte of the last record the filter reads
cudaError_t stage_input(vgicp_prep_handle h, const float* points, size_t n, size_t stride_bytes, int on_device, const int* off, int F, const float** d_in) {
  size_t span = 12;
  for (int j = 0; j < F; j++) span = span > (size_t)off[j] * 4 + 4 ? span : (size_t)off[j] * 4 + 4;
  *d_in = points;
  if (on_device) return cudaSuccess;
  cudaError_t e = h->staging.reserve(n * stride_bytes);
  if (e == cudaSuccess) e = cudaMemcpyAsync(h->staging.p, points, (n - 1) * stride_bytes + span, cudaMemcpyHostToDevice, h->stream.get());
  *d_in = reinterpret_cast<const float*>(h->staging.p);
  return e;
}

// both entry points: F = n_fields per-point fields at float offsets off[] (F = 0: x y z only)
int run_filter(vgicp_prep_handle h, const char* who, const float* points, size_t n, size_t stride_bytes, int on_device, float leaf, int remove_near_origin, const int* off, int F,
               float* out, size_t cap, int out_on_device, size_t* n_out) {
  const std::string w(who);
  const size_t rec = 3 + (size_t)F;  // output floats per point
  PREP_TRY(h, cudaSetDevice(h->device));
  const int ni = (int)n;
  const float* d_in = nullptr;
  PREP_TRY(h, stage_input(h, points, n, stride_bytes, on_device, off, F, &d_in));
  PREP_TRY(h, h->pts4.reserve(n));
  PREP_TRY(h, h->entry.reserve(n));
  PREP_TRY(h, h->flushed.reserve(n));
  if (F > 0) {
    PREP_TRY(h, h->fflushed.reserve(n * F));
    PREP_TRY(h, h->ftail.reserve((size_t)kHist * F));
  }
  float* d_out = out;
  const size_t out_cap = out_on_device ? cap : n;  // the filter never emits more points than it reads
  if (!out_on_device) {
    PREP_TRY(h, h->out.reserve(rec * n));
    d_out = h->out.p;
  }
  const int chunks = (ni + kRankThreads - 1) / kRankThreads;
  PREP_TRY(h, lookback_next(h->chunk_state, h->chunk_epoch, chunks, h->stream.get()));
  const float inv_leaf = 1.0f / leaf;
  const size_t sf = stride_bytes / 4;
  const int flt = remove_near_origin ? 1 : 0;
  switch (F) {
    case 0: PREP_TRY(h, (launch_filter<0>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    case 1: PREP_TRY(h, (launch_filter<1>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    case 2: PREP_TRY(h, (launch_filter<2>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    case 3: PREP_TRY(h, (launch_filter<3>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    case 4: PREP_TRY(h, (launch_filter<4>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    case 5: PREP_TRY(h, (launch_filter<5>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    case 6: PREP_TRY(h, (launch_filter<6>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    case 7: PREP_TRY(h, (launch_filter<7>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    case 8: PREP_TRY(h, (launch_filter<8>(h, d_in, sf, off, ni, inv_leaf, flt, d_out, out_cap, chunks))); break;
    default: return fail(h, 1, w + ": unsupported field count");
  }
  PREP_TRY(h, cudaMemcpyAsync(h->h_counts.get(), h->d_counts.get(), 2 * sizeof(int), cudaMemcpyDeviceToHost, h->stream.get()));
  PREP_TRY(h, cudaStreamSynchronize(h->stream.get()));
  const size_t m = (size_t)h->h_counts[1];
  *n_out = m;
  if (m > cap) return fail(h, 1, w + ": output capacity too small (n points always suffice)");
  if (!out_on_device && m > 0) {
    PREP_TRY(h, cudaMemcpyAsync(out, d_out, m * rec * sizeof(float), cudaMemcpyDeviceToHost, h->stream.get()));
    PREP_TRY(h, cudaStreamSynchronize(h->stream.get()));
  }
  return 0;
}

template <int F>
cudaError_t launch_centroids(vgicp_prep_handle h, const float* d_in, size_t stride_f, const int* off, const unsigned* keys, int kept, int blocks, float* d_out, size_t out_cap) {
  FieldArgs fa{};
  fa.in = d_in;
  fa.stride_f = stride_f;
  for (int j = 0; j < F; j++) fa.off[j] = off[j];
  k_grid_centroids<F><<<blocks, kGridWarps * 32, 0, h->stream.get()>>>(keys, h->gsorted4.p, kept, h->gvstart.p, h->d_grid.get(), fa, d_out, out_cap);
  return cudaGetLastError();
}

int run_voxel_grid(vgicp_prep_handle h, const float* points, size_t n, size_t stride_bytes, int on_device, float leaf, int remove_near_origin, const int* off, int F,
                   unsigned min_points, float* out, size_t cap, int out_on_device, size_t* n_out) {
  const size_t rec = 3 + (size_t)F;
  PREP_TRY(h, cudaSetDevice(h->device));
  const int ni = (int)n;
  const float* d_in = nullptr;
  PREP_TRY(h, stage_input(h, points, n, stride_bytes, on_device, off, F, &d_in));
  PREP_TRY(h, h->pts4.reserve(n));
  for (int k = 0; k < 2; k++) {
    PREP_TRY(h, h->gkeys[k].reserve(n));
    PREP_TRY(h, h->gvals[k].reserve(n));
  }
  PREP_TRY(h, h->gsorted4.reserve(n));
  const float inv = 1.0f / leaf;
  const size_t sf = stride_bytes / 4;
  const int flt = remove_near_origin ? 1 : 0;
  // 1. the box of the kept points' cells, read back: the one host decision (refusals, key width) before the sort
  PREP_TRY(h, cudaMemsetAsync(h->d_grid.get(), 0, kGridState * sizeof(unsigned), h->stream.get()));
  const int bb = (ni + kGridBoxThreads - 1) / kGridBoxThreads;
  k_grid_box<<<bb < 4 * kNumSMs ? bb : 4 * kNumSMs, kGridBoxThreads, 0, h->stream.get()>>>(d_in, sf, ni, inv, flt, h->pts4.p, h->d_grid.get());
  PREP_TRY(h, cudaGetLastError());
  PREP_TRY(h, cudaMemcpyAsync(h->h_grid.get(), h->d_grid.get(), kGridState * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream.get()));
  PREP_TRY(h, cudaStreamSynchronize(h->stream.get()));
  if (h->h_grid[7]) return fail(h, 1, "voxel_grid: a kept point's cell floor(x / leaf) lies outside the int range");
  const int kept = (int)h->h_grid[6];
  if (kept == 0) return 0;
  int lo[3];
  long long div[3];
  for (int a = 0; a < 3; a++) {
    lo[a] = cell_dec(~h->h_grid[a]);
    div[a] = (long long)cell_dec(h->h_grid[3 + a]) - lo[a] + 1;
  }
  const long long lim = 0x7fffffff;
  if (div[0] > lim || div[1] > lim / div[0] || div[2] > lim / (div[0] * div[1]))
    return fail(h, 1, "voxel_grid: the leaf is too small for the extent of the cloud (more than INT32_MAX cells in the box)");
  const unsigned V = (unsigned)(div[0] * div[1] * div[2]);  // the voxel count, and the key of a dropped point
  const int key_bits = 32 - __builtin_clz(V);
  const int passes = sort_num_passes(key_bits);
  // 2. keys + digit histograms, the sort carrying x y z and the input index
  const size_t sb = sort_scratch_bytes(ni, passes);
  PREP_TRY(h, h->gscratch.reserve(sb));
  PREP_TRY(h, cudaMemsetAsync(h->gscratch.p, 0, sb, h->stream.get()));
  const int hb = (ni + kSortThreads * 8 - 1) / (kSortThreads * 8);
  k_grid_keys<<<hb < 4 * kNumSMs ? hb : 4 * kNumSMs, kSortThreads, 0, h->stream.get()>>>(h->pts4.p, ni, inv, flt, make_int3(lo[0], lo[1], lo[2]), (unsigned)div[0],
                                                                                   (unsigned)(div[0] * div[1]), V, passes, h->gkeys[0].p,
                                                                                   reinterpret_cast<unsigned*>(h->gscratch.p));
  PREP_TRY(h, cudaGetLastError());
  PREP_TRY(h, launch_sort_pairs<unsigned>(h->gkeys[0].p, h->gvals[0].p, h->gkeys[1].p, h->gvals[1].p, ni, key_bits, h->gscratch.p, true, h->pts4.p, h->gsorted4.p, nullptr,
                                          h->stream.get()));
  const unsigned* keys = h->gkeys[passes & 1].p;
  // 3. the voxels that reach the minimum, ranked; 4. their centroids
  const int chunks = (kept + kRankThreads - 1) / kRankThreads;
  PREP_TRY(h, lookback_next(h->chunk_state, h->chunk_epoch, chunks, h->stream.get()));
  PREP_TRY(h, h->gvstart.reserve((size_t)kept));
  k_grid_heads<<<chunks, kRankThreads, 0, h->stream.get()>>>(keys, kept, min_points, h->chunk_state.p, h->chunk_epoch, h->gvstart.p, h->d_grid.get());
  PREP_TRY(h, cudaGetLastError());
  float* d_out = out;
  size_t out_cap = cap;
  if (!out_on_device) {
    PREP_TRY(h, h->out.reserve(rec * kept));
    d_out = h->out.p;
    out_cap = (size_t)kept;  // m <= kept; the cap itself is checked on the host before anything is copied back
  }
  const long long most = (long long)kept / (min_points > 1 ? min_points : 1);  // voxels that can reach the minimum
  const long long cb = (most < (long long)V ? most : (long long)V) + kGridWarps - 1;
  const int cblocks = (int)(cb / kGridWarps < 16 * kNumSMs ? (cb / kGridWarps > 0 ? cb / kGridWarps : 1) : 16 * kNumSMs);
  switch (F) {
    case 0: PREP_TRY(h, (launch_centroids<0>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    case 1: PREP_TRY(h, (launch_centroids<1>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    case 2: PREP_TRY(h, (launch_centroids<2>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    case 3: PREP_TRY(h, (launch_centroids<3>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    case 4: PREP_TRY(h, (launch_centroids<4>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    case 5: PREP_TRY(h, (launch_centroids<5>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    case 6: PREP_TRY(h, (launch_centroids<6>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    case 7: PREP_TRY(h, (launch_centroids<7>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    case 8: PREP_TRY(h, (launch_centroids<8>(h, d_in, sf, off, keys, kept, cblocks, d_out, out_cap))); break;
    default: return fail(h, 1, "voxel_grid: unsupported field count");
  }
  PREP_TRY(h, cudaMemcpyAsync(h->h_grid.get() + 8, h->d_grid.get() + 8, sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream.get()));
  PREP_TRY(h, cudaStreamSynchronize(h->stream.get()));
  const size_t m = h->h_grid[8];
  *n_out = m;
  if (m > cap) return fail(h, 1, "voxel_grid: output capacity too small (n points always suffice)");
  if (!out_on_device && m > 0) {
    PREP_TRY(h, cudaMemcpyAsync(out, d_out, m * rec * sizeof(float), cudaMemcpyDeviceToHost, h->stream.get()));
    PREP_TRY(h, cudaStreamSynchronize(h->stream.get()));
  }
  return 0;
}

}  // namespace

extern "C" {

int vgicp_prep_approximate_voxel_grid(vgicp_prep_handle h, const float* xyz, size_t n, size_t stride_bytes, int on_device, float leaf, int remove_near_origin, float* out_xyz,
                                      size_t cap, int out_on_device, size_t* n_out) {
  if (!h) return 1;
  if (!n_out) return fail(h, 1, "approximate_voxel_grid: n_out is null");
  *n_out = 0;
  if (n == 0) return 0;
  if (!xyz || !out_xyz) return fail(h, 1, "approximate_voxel_grid: null buffer");
  if (stride_bytes < 12 || stride_bytes % 4) return fail(h, 1, "approximate_voxel_grid: stride must be >= 12 and a multiple of 4");
  if (!(leaf > 0.f)) return fail(h, 1, "approximate_voxel_grid: leaf size must be positive");
  if (n > (size_t)0x7fffffff - 4096) return fail(h, 1, "approximate_voxel_grid: too many points");
  return run_filter(h, "approximate_voxel_grid", xyz, n, stride_bytes, on_device, leaf, remove_near_origin, nullptr, 0, out_xyz, cap, out_on_device, n_out);
}

int vgicp_prep_approximate_voxel_grid_fields(vgicp_prep_handle h, const float* points, size_t n, size_t stride_bytes, int on_device, float leaf, int remove_near_origin,
                                             const size_t* field_offsets, int n_fields, float* out, size_t cap, int out_on_device, size_t* n_out) {
  if (!h) return 1;
  if (!n_out) return fail(h, 1, "approximate_voxel_grid_fields: n_out is null");
  *n_out = 0;
  if (n_fields < 1 || n_fields > kMaxFields) return fail(h, 1, "approximate_voxel_grid_fields: n_fields must be 1 ... 8");
  if (!field_offsets) return fail(h, 1, "approximate_voxel_grid_fields: null field_offsets");
  if (stride_bytes < 12 || stride_bytes % 4) return fail(h, 1, "approximate_voxel_grid_fields: stride must be >= 12 and a multiple of 4");
  int off[kMaxFields];
  for (int j = 0; j < n_fields; j++) {
    const size_t o = field_offsets[j];
    if (o % 4 || o < 12 || o > stride_bytes - 4)
      return fail(h, 1, "approximate_voxel_grid_fields: a field offset must be a multiple of 4, >= 12 and leave 4 bytes within the stride");
    off[j] = (int)(o / 4);
  }
  if (n == 0) return 0;
  if (!points || !out) return fail(h, 1, "approximate_voxel_grid_fields: null buffer");
  if (!(leaf > 0.f)) return fail(h, 1, "approximate_voxel_grid_fields: leaf size must be positive");
  if (n > (size_t)0x7fffffff - 4096) return fail(h, 1, "approximate_voxel_grid_fields: too many points");
  return run_filter(h, "approximate_voxel_grid_fields", points, n, stride_bytes, on_device, leaf, remove_near_origin, off, n_fields, out, cap, out_on_device, n_out);
}

int vgicp_prep_voxel_grid(vgicp_prep_handle h, const float* points, size_t n, size_t stride_bytes, int on_device, float leaf, int remove_near_origin, const size_t* field_offsets,
                          int n_fields, unsigned min_points_per_voxel, float* out, size_t cap, int out_on_device, size_t* n_out) {
  if (!h) return 1;
  if (!n_out) return fail(h, 1, "voxel_grid: n_out is null");
  *n_out = 0;
  if (n_fields < 0 || n_fields > kMaxFields) return fail(h, 1, "voxel_grid: n_fields must be 0 ... 8");
  if (n_fields > 0 && !field_offsets) return fail(h, 1, "voxel_grid: null field_offsets");
  if (stride_bytes < 12 || stride_bytes % 4) return fail(h, 1, "voxel_grid: stride must be >= 12 and a multiple of 4");
  int off[kMaxFields];
  for (int j = 0; j < n_fields; j++) {
    const size_t o = field_offsets[j];
    if (o % 4 || o < 12 || o > stride_bytes - 4)
      return fail(h, 1, "voxel_grid: a field offset must be a multiple of 4, >= 12 and leave 4 bytes within the stride");
    off[j] = (int)(o / 4);
  }
  if (!(leaf > 0.f) || !std::isfinite(leaf)) return fail(h, 1, "voxel_grid: leaf size must be finite and positive");
  if (n == 0) return 0;
  if (!points || !out) return fail(h, 1, "voxel_grid: null buffer");
  if (n > (size_t)0x7fffffff - 4096) return fail(h, 1, "voxel_grid: too many points");
  return run_voxel_grid(h, points, n, stride_bytes, on_device, leaf, remove_near_origin, off, n_fields, min_points_per_voxel, out, cap, out_on_device, n_out);
}

}  // extern "C"
