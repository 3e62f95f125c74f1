// vgicp_kernels.cuh -- hand-written sm_90a (H100) kernels of the VGICP hot path.
//
// Stage 1  k-NN + covariance + regularisation   (reference: brute_force_knn.cu, covariance_estimation.cu,
//                                                covariance_estimation_rbf.cu, covariance_regularization.cu)
// Stage 2  Gaussian voxel map build              (reference: gaussian_voxelmap.cu, vector3_hash.cuh)
// Stage 3  fused voxel lookup + Mahalanobis residual/Jacobian reduction
//                                                (reference: find_voxel_correspondences.cu + compute_derivatives.cu)
//
// Device data layout (all arrays 16-byte aligned, one element per point / voxel / bucket):
//   points      float4 {x,y,z,0}                          16 B/pt   coalesced LDG.128
//   covariance  float4 {xx,xy,xz,yy} + float2 {yz,zz}     24 B/pt   symmetric-packed (reference: 36 B Matrix3f)
//   neighbours  int32  [n][k]
//   buckets     int4   {cx,cy,cz,voxel id | -1}           16 B/bucket  == thrust::pair<Vector3i,int>
//   voxels      3 x float4: {mx,my,mz,n(int bits)} {cxx,cxy,cxz,cyy} {cyz,czz,-,-}   48 B/voxel
//
// Arithmetic that the parity contract makes order-defined (voxel coordinate, hash, transformed point, k-NN distance,
// raw covariance) is written with explicit __f*_rn / __fmaf_rn so nvcc cannot re-associate or contract it differently
// from the CPU checker used by the tests (which spells the same operations).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lsq_math.hpp"
#include "vgicp_sort.cuh"
#include "vgicp_stage1.cuh"

namespace vgicp {

constexpr int kLinThreads = 128;     // block size of the linearize kernel
constexpr int kLinMaxBlocks = 4 * kNumSMs;  // 4 blocks per SM: upper bound on partial sums the last block has to fold (more resident warps only thrash L1: measured)
constexpr int kLinValues = 28;       // 21 unique H + 6 b + 1 err
constexpr int kLinStride = 32;       // row length of the partial-sum arrays (the speculative evaluation carries 29 values)
constexpr int kLinOutCommError = 44; // out[44]: 1.0 when a sharded evaluation timed out waiting for a peer (the sums are then incomplete)

struct Pose {      // float image of an Eigen::Isometry3f: R row-major here, t
  float r[9];
  float t[3];
};

constexpr int kCommMaxRanks = 8;
// Stage-1 sharding: per rank one IPC-exported arena holding the covariance arrays of both clouds (so that peers can store the
// covariances of their slice straight into it) and the "slice delivered" flags.
struct CommArenaHeader {
  volatile unsigned long long delivered[2][kCommMaxRanks];  // [cloud slot][sender rank] = sequence number of the last delivered slice
  volatile int error;
};
constexpr size_t kCommArenaHeaderBytes = 256;
// one per rank, in that rank's device memory, mapped into every peer with CUDA IPC
struct CommMailbox {
  double vals[2][kCommMaxRanks][32];                 // [seq & 1][sender][28 sums]
  volatile unsigned long long flags[2][kCommMaxRanks];  // [seq & 1][sender] = seq + 1 once the sender's values are visible
  volatile int error;                                // set when a wait times out
};


// ---------------------------------------------------------------------------------------------------------------
// vector3_hash.cuh:8-38
// ---------------------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t hash_mix(uint64_t k) {
  const uint64_t m = 0xc6a4a7935bd1e995ULL;
  k *= m;
  k ^= k >> 47;
  k *= m;
  return k;
}
__host__ __device__ __forceinline__ uint64_t hash_fold(uint64_t h, uint64_t kmixed) {
  const uint64_t m = 0xc6a4a7935bd1e995ULL;
  h ^= kmixed;
  h *= m;
  h += 0xe6546b64ULL;
  return h;
}
// vector3i_hash: the int -> uint64_t conversion sign-extends (vector3_hash.cuh:29-31)
__host__ __device__ __forceinline__ uint64_t vector3i_hash(int x, int y, int z) {
  uint64_t h = 0;
  h = hash_fold(h, hash_mix((uint64_t)(int64_t)x));
  h = hash_fold(h, hash_mix((uint64_t)(int64_t)y));
  h = hash_fold(h, hash_mix((uint64_t)(int64_t)z));
  return h;
}

// calc_voxel_coord (vector3_hash.cuh:35-38): floor(x / res - 0.5) in float
__device__ __forceinline__ int voxel_coord1(float x, float res) { return (int)floorf(__fsub_rn(__fdiv_rn(x, res), 0.5f)); }

// R*a + t the way nvcc contracts Eigen's expression: fma(r2,a2, fma(r1,a1, r0*a0)) + t
__device__ __forceinline__ float3 transform_point(const Pose& T, float ax, float ay, float az) {
  float3 o;
  o.x = __fadd_rn(__fmaf_rn(T.r[2], az, __fmaf_rn(T.r[1], ay, __fmul_rn(T.r[0], ax))), T.t[0]);
  o.y = __fadd_rn(__fmaf_rn(T.r[5], az, __fmaf_rn(T.r[4], ay, __fmul_rn(T.r[3], ax))), T.t[1]);
  o.z = __fadd_rn(__fmaf_rn(T.r[8], az, __fmaf_rn(T.r[7], ay, __fmul_rn(T.r[6], ax))), T.t[2]);
  return o;
}

// ---------------------------------------------------------------------------------------------------------------
// cloud upload: strided host xyz image -> float4
// ---------------------------------------------------------------------------------------------------------------
__global__ void k_unpack_points(const unsigned char* __restrict__ raw, size_t stride, int n, float4* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = reinterpret_cast<const float*>(raw + (size_t)i * stride);
  out[i] = make_float4(p[0], p[1], p[2], 0.0f);
}

// ---------------------------------------------------------------------------------------------------------------
// Stage 2: voxel map build (gaussian_voxelmap.cu:21-58, 61-73, 76-120, 158-176, 258-289)
//
// The reference resolves slot ownership by atomicCAS arrival order.  Here a contended slot goes to the voxel with
// the lexicographically smaller coordinate and the loser keeps probing (priority linear probing): the final table
// is exactly what serial first-come-first-served insertion of the distinct voxels in lexicographic order produces,
// independent of thread timing -- the order the oracle uses.  slots[] holds a representative point index per voxel.
// ---------------------------------------------------------------------------------------------------------------
// bbox[0..2] / bbox[3..5]: running min / max of the voxel coordinates (sizes the direct-mapped index of the evaluation kernels)
__global__ void k_voxel_coords(const float4* __restrict__ pts, int n, float res, int4* __restrict__ coords, int* __restrict__ bbox) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int4 c = make_int4(0, 0, 0, 0);
  const bool in = i < n;
  if (in) {
    float4 p = pts[i];
    c = make_int4(voxel_coord1(p.x, res), voxel_coord1(p.y, res), voxel_coord1(p.z, res), 0);
    coords[i] = c;
  }
  const int lo_x = __reduce_min_sync(0xffffffffu, in ? c.x : INT_MAX), lo_y = __reduce_min_sync(0xffffffffu, in ? c.y : INT_MAX), lo_z = __reduce_min_sync(0xffffffffu, in ? c.z : INT_MAX);
  const int hi_x = __reduce_max_sync(0xffffffffu, in ? c.x : INT_MIN), hi_y = __reduce_max_sync(0xffffffffu, in ? c.y : INT_MIN), hi_z = __reduce_max_sync(0xffffffffu, in ? c.z : INT_MIN);
  if ((threadIdx.x & 31) == 0 && lo_x != INT_MAX) {
    atomicMin(&bbox[0], lo_x); atomicMin(&bbox[1], lo_y); atomicMin(&bbox[2], lo_z);
    atomicMax(&bbox[3], hi_x); atomicMax(&bbox[4], hi_y); atomicMax(&bbox[5], hi_z);
  }
}

// Direct-mapped voxel index: cells[((x - x0) * ny + (y - y0)) * nz + (z - z0)] = voxel id or -1 over the bounding box of the map's
// voxel coordinates.  A lookup in the reference's table answers "is this coordinate one of the map's voxels, and which" (every stored
// voxel sits within the probe window of its home bucket and nothing is ever deleted), so any exact index returns the same ids; this
// one needs no hashing (vector3i_hash is nine 64-bit multiplies per cell) and no probe chain (3.8 probes per miss at 60 % load).
struct DenseIndex {
  int* cells;  // nullptr: not in use
  int x0, y0, z0;
  unsigned nx, ny, nz;
};
__device__ __forceinline__ int dense_offset(const DenseIndex& d, int x, int y, int z) {
  const unsigned ux = (unsigned)(x - d.x0), uy = (unsigned)(y - d.y0), uz = (unsigned)(z - d.z0);
  return (ux < d.nx && uy < d.ny && uz < d.nz) ? (int)((ux * d.ny + uy) * d.nz + uz) : -1;
}

// `skip` (may be null): the table attempts of a growth sequence are enqueued back to back; once one of them has met the reference's
// acceptance rule (*skip != 0, set by k_table_verdict) the kernels of the later, larger attempts return at once
__global__ void k_fill_i32(int* __restrict__ p, int v, size_t n, const int* __restrict__ skip) {
  if (skip && *skip) return;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
// gaussian_voxelmap.cu:280: the table is accepted when fewer than 1 % of the points failed to find their voxel
__global__ void k_table_verdict(int* __restrict__ counters /* [0] failures, [9] accepted table size */, int n, int num_buckets) {
  if (counters[9] == 0 && (double)counters[0] / (double)n < 0.01) counters[9] = num_buckets;
}

// after a sharded covariance kernel (stream order): make this rank's peer stores visible, tell every rank that the slice of cloud
// slot `slot` number `seq` has been delivered, and wait until every rank's slice of it has arrived here
struct ArenaPeers {
  CommArenaHeader* hdr[kCommMaxRanks];
};
__global__ void k_comm_deliver_and_wait(ArenaPeers peers, int rank, int nranks, int slot, unsigned long long seq) {
  __threadfence_system();
  if ((int)threadIdx.x < nranks) {
    peers.hdr[threadIdx.x]->delivered[slot][rank] = seq;
    __threadfence_system();
    CommArenaHeader* me = peers.hdr[rank];
    long long spins = 0;
    while (me->delivered[slot][threadIdx.x] < seq) {
      if (++spins > (1LL << 31)) { me->error = 1; break; }
    }
  }
  __threadfence_system();
}

// set_{source,target}_neighbors: flag any caller-supplied neighbour index outside [0, n)
__global__ void k_validate_indices(const int* __restrict__ idx, size_t count, int n, int* __restrict__ bad) {
  bool any = false;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) any |= (unsigned)idx[i] >= (unsigned)n;
  if (__any_sync(0xffffffffu, any) && (threadIdx.x & 31) == 0) atomicOr(bad, 1);
}

__device__ __forceinline__ bool coord_eq(int4 a, int4 b) { return a.x == b.x && a.y == b.y && a.z == b.z; }
__device__ __forceinline__ bool coord_less(int4 a, int4 b) {
  if (a.x != b.x) return a.x < b.x;
  if (a.y != b.y) return a.y < b.y;
  return a.z < b.z;
}

__global__ void k_table_insert(const int4* __restrict__ coords, int n, int* slots, unsigned mask, int max_scan, const int* __restrict__ skip) {
  if (skip && *skip) return;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int cur = i;
  int4 cc = coords[i];
  unsigned pos = (unsigned)(vector3i_hash(cc.x, cc.y, cc.z) & mask);
  int dist = 0;
  while (dist < max_scan) {
    int r = *reinterpret_cast<volatile int*>(&slots[pos]);
    if (r < 0) {
      int old = atomicCAS(&slots[pos], -1, cur);
      if (old < 0) return;  // claimed an empty slot
      r = old;
    }
    int4 cr = coords[r];
    if (coord_eq(cr, cc)) return;  // voxel already present
    if (coord_less(cc, cr)) {      // we outrank the resident: take the slot, carry the resident onward
      int old = atomicCAS(&slots[pos], r, cur);
      if (old != r) continue;      // slot changed under us: look again
      cur = r;
      cc = cr;
      unsigned home = (unsigned)(vector3i_hash(cc.x, cc.y, cc.z) & mask);
      dist = (int)((pos - home) & mask);
    }
    pos = (pos + 1) & mask;
    dist++;
  }
  // fell off the 10-probe window: this voxel is dropped from the map (gaussian_voxelmap.cu:57, SURVEY Q5)
}

// per point: find the slot of its voxel (stop at first empty like find_voxel_correspondences.cu:43-45) and count failures
__global__ void k_table_lookup_points(const int4* __restrict__ coords, int n, const int* __restrict__ slots, unsigned mask, int max_scan, int* __restrict__ slot_of_point,
                                      int* __restrict__ fail_counter, const int* __restrict__ skip) {
  if (skip && *skip) return;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int4 c = coords[i];
  unsigned pos = (unsigned)(vector3i_hash(c.x, c.y, c.z) & mask);
  int found = -1;
  for (int s = 0; s < max_scan; s++) {
    int r = slots[pos];
    if (r < 0) break;
    if (coord_eq(coords[r], c)) { found = (int)pos; break; }
    pos = (pos + 1) & mask;
  }
  slot_of_point[i] = found;
  if (found < 0) atomicAdd(fail_counter, 1);
}

// voxel id = rank of the slot among occupied slots; buckets = {coord, id} or {0,0,0,-1} (voxel_coord_select_kernel :61-73).
// One block per 1024 buckets: block scan, then a decoupled look-back over the totals the preceding blocks publish in
// chunk_state (epoch << 32 | total; the epoch changes every launch, so the array never needs clearing).  A block only ever
// waits for blocks with a smaller index, which the hardware scheduled before it.
__global__ void __launch_bounds__(1024) k_table_assign_ids(const int4* __restrict__ coords, const int* __restrict__ slots, int num_buckets, int4* __restrict__ buckets,
                                                          int* __restrict__ num_voxels, const DenseIndex dense, unsigned long long* chunk_state, unsigned epoch) {
  __shared__ int warp_sums[32];
  __shared__ int s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int b = blockIdx.x * 1024 + tid;
  const int r = b < num_buckets ? slots[b] : -1;
  const int flag = r >= 0 ? 1 : 0;
  int v = flag;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) warp_sums[wid] = v;
  __syncthreads();
  if (wid == 0) {
    int w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    warp_sums[lane] = w;
    const int total = __shfl_sync(0xffffffffu, w, 31);
    volatile unsigned long long* state = chunk_state;
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
      if (blockIdx.x == gridDim.x - 1) *num_voxels = base + total;
    }
  }
  __syncthreads();
  const int prefix = s_base + (wid > 0 ? warp_sums[wid - 1] : 0) + v - flag;  // exclusive
  if (b < num_buckets) {
    if (flag) {
      int4 c = coords[r];
      buckets[b] = make_int4(c.x, c.y, c.z, prefix);
      if (dense.cells) dense.cells[dense_offset(dense, c.x, c.y, c.z)] = prefix;  // (inside the box by construction)
    } else {
      buckets[b] = make_int4(0, 0, 0, -1);
    }
  }
}

// Voxel Gaussians: accumulate_points_kernel :76-120 + finalize_voxels_kernel :158-176 (VGICP: per-point covariances) and
// accumulate / ndt_finalize_voxels_kernel :122-148,178-198 (NDT: the points alone).  The reference adds floats with atomicAdd in
// arrival order (thread-timing dependent).  Here the points are stably sorted by voxel id (vgicp_sort.cuh: index ascending inside
// a voxel), and one warp per voxel adds its points IN POINT ORDER in double, each of ten lanes one component, and rounds once:
// exactly the sums of the CPU checker, bit for bit, and no atomics (hot voxels hold thousands of points at 1 M points).
// k_voxel_sort_keys: sort key of point i = its voxel id, or `invalid` (sorts last) for the points of dropped voxels; also counts
// the sort's digits.
__global__ void __launch_bounds__(kSortThreads) k_voxel_sort_keys(const int* __restrict__ slot_of_point, const int4* __restrict__ buckets, int n, unsigned invalid, int passes,
                                                                  unsigned* __restrict__ keys, unsigned* __restrict__ hist) {
  __shared__ unsigned sh[kSortMaxPasses * kSortBins];
  for (int i = threadIdx.x; i < passes * kSortBins; i += kSortThreads) sh[i] = 0;
  __syncthreads();
  const int n_round = (n + 31) & ~31;
  for (int i = blockIdx.x * kSortThreads + threadIdx.x; i < n_round; i += gridDim.x * kSortThreads) {
    const bool valid = i < n;
    unsigned key = invalid;
    if (valid) {
      const int s = slot_of_point[i];
      if (s >= 0) key = (unsigned)buckets[s].w;
      keys[i] = key;
    }
    sort_hist_add(sh, passes, valid, (unsigned long long)key);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < passes * kSortBins; i += kSortThreads)
    if (sh[i]) atomicAdd(&hist[i], sh[i]);
}

// [start, end) of every voxel in the sorted list
__global__ void k_voxel_segments(const unsigned* __restrict__ keys, int n, unsigned invalid, int2* __restrict__ seg) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const unsigned key = keys[j];
  if (key == invalid) return;
  if (j == 0 || keys[j - 1] != key) seg[key].x = j;
  if (j == n - 1 || keys[j + 1] != key) seg[key].y = j + 1;
}

// one warp per voxel.  Lane c < 10 carries one sum: 0..2 the point, 3..8 the covariance terms (xx xy xz yy yz zz; VGICP: the
// point's packed covariance, NDT: p p^T formed in double), 9 nothing (the count is the segment length).
template <bool NDT>
__global__ void __launch_bounds__(128) k_voxel_reduce(const float4* __restrict__ pts, const float4* __restrict__ covA, const float2* __restrict__ covB, const unsigned* __restrict__ order,
                                                      const int2* __restrict__ seg, const int* __restrict__ nv_ptr, VoxelRec* __restrict__ vox) {
  const int v = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (v >= *nv_ptr) return;
  const int2 se = seg[v];
  const int c = lane < 9 ? lane : 0;
  // component c of point i as a double
  auto term = [&](unsigned i) -> double {
    const float* p = reinterpret_cast<const float*>(pts + i);
    if (c < 3) return (double)p[c];
    if (NDT) {  // xx xy xz yy yz zz
      const int t = c - 3;
      const int r0 = t < 3 ? 0 : (t < 5 ? 1 : 2), c0 = t < 3 ? t : (t < 5 ? t - 2 : 2);
      return (double)p[r0] * (double)p[c0];
    }
    if (c < 7) return (double)reinterpret_cast<const float*>(covA + i)[c - 3];
    return (double)reinterpret_cast<const float*>(covB + i)[c - 7];
  };
  // 32 points per round: one coalesced load of their indices, then the gathers sixteen at a time in flight, added in point order
  // (a dependent index -> gather -> add chain per point made the largest voxel -- 158 points at 17 k -- a long tail)
  double sum = 0.0;
  for (int j0 = se.x; j0 < se.y; j0 += 32) {
    const int nb = min(32, se.y - j0);
    const unsigned mine = lane < nb ? order[j0 + lane] : 0u;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      double t[16];
#pragma unroll
      for (int u = 0; u < 16; u++) {
        const unsigned i = __shfl_sync(0xffffffffu, mine, h * 16 + u);
        t[u] = h * 16 + u < nb ? term(i) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 16; u++)
        if (h * 16 + u < nb) sum += t[u];
    }
  }
  const int cnt = se.y - se.x;
  const double nn = (double)cnt;
  float out;
  if (NDT) {  // mean = sum / n ; cov(r, c) = (S_rc - mean_r * S_c) / n, lower triangle in the packed record
    const double sx = __shfl_sync(0xffffffffu, sum, 0), sy = __shfl_sync(0xffffffffu, sum, 1), sz = __shfl_sync(0xffffffffu, sum, 2);
    const double mx = sx / nn, my = sy / nn, mz = sz / nn;
    // (spelled with intrinsics: a contracted fma would round differently from the checker's multiply-then-subtract)
    double val = sum / nn;
    if (c >= 3) {
      const double m_r = c == 3 ? mx : (c == 4 || c == 6 ? my : mz);
      const double s_c = c <= 5 ? sx : (c <= 7 ? sy : sz);
      val = __ddiv_rn(__dsub_rn(sum, __dmul_rn(m_r, s_c)), nn);
    }
    out = (float)val;
  } else {
    out = (float)(sum / nn);
  }
  // record layout: {mx my mz n} {cxx cxy cxz cyy} {cyz czz 0 0}: lane c < 3 -> float c, lanes 3..8 -> floats 4..9, lane 9 -> n, lanes 10, 11 -> 0
  float* rec = reinterpret_cast<float*>(vox + v);
  if (lane < 3) rec[lane] = out;
  else if (lane < 9) rec[lane + 1] = out;
  else if (lane == 9) rec[3] = __int_as_float(cnt);
  else if (lane < 12) rec[lane] = 0.f;
}

// D2D: the source voxel means / covariances become the "source cloud" of the evaluation kernel
__global__ void k_vox_to_cloud(const VoxelRec* __restrict__ vox, const int* __restrict__ nv_ptr, float4* __restrict__ pts, float4* __restrict__ covA, float2* __restrict__ covB) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= *nv_ptr) return;
  VoxelRec r = vox[v];
  pts[v] = make_float4(r.mean_n.x, r.mean_n.y, r.mean_n.z, 0.f);
  covA[v] = r.c0;
  covB[v] = make_float2(r.c1.x, r.c1.y);
}

// ---------------------------------------------------------------------------------------------------------------
// Stage 2b + 3 fused: per source point, transform by the linearisation pose, probe the neighbour voxels
// (find_voxel_correspondences.cu:32-60), and accumulate the Mahalanobis residual and Jacobian terms
// (compute_derivatives.cu:50-92 / :105-135) without materialising the correspondence list.
//   J = [skew(p') | -I] depends on the point only, so  sum_c w J^T M_c J = J^T (sum_c w M_c) J : the 3x3 sums
//   Msum = sum w M_c and v = sum w M_c e_c are formed per point and J is applied once.
// Per-block partials (double) are folded by the last block in a fixed order -> bitwise reproducible H, b, err.
// ---------------------------------------------------------------------------------------------------------------
struct LinArgs {
  const float4* pts;
  const float4* covA;
  const float2* covB;
  int n;
  const int4* buckets;
  unsigned mask;
  int max_scan;
  const VoxelRec* vox;
  DenseIndex dense;     // direct-mapped index over the map's bounding box (cells == nullptr: probe the hash table)
  const int4* offsets;  // generic mode
  int n_off;
  float res;
  int ndt;  // 0: VGICP weights (sqrt(n), compute_derivatives.cu:78); 1: NDT (Cauchy weight, voxels with <= 6 points skipped, ndt_compute_derivatives.cu)
  Pose Tlin, Teval;
  double* partials;       // [gridDim.x][kLinStride]
  unsigned int* ticket;   // zero before first launch; reset by the last block
  double* out;            // [43]: err, H (36, column-major), b (6); may be mapped pinned host memory
  volatile unsigned long long* done_flag;  // optional (mapped host memory): set to done_seq once `out` is complete
  unsigned long long done_seq;
  // source sharded over several GPUs (SURVEY 8e): the folded sums of this rank are exchanged with the peers by the last
  // block itself, through mailboxes in peer memory (NVLink P2P stores), and summed in rank order
  int comm_ranks;         // 0/1 = single GPU
  int comm_rank;
  unsigned long long comm_seq;   // evaluation number (same on every rank), selects the mailbox half
  CommMailbox* comm_peers[kCommMaxRanks];  // peers' mailboxes (index = rank; own mailbox included)
};

__device__ __forceinline__ int lookup_voxel(const int4* __restrict__ buckets, unsigned mask, int max_scan, uint64_t h, int cx, int cy, int cz) {
  unsigned pos = (unsigned)(h & mask);
  for (int s = 0; s < max_scan; s++) {
    int4 b = __ldg(&buckets[pos]);
    if (b.w < 0) return -1;
    if (b.x == cx && b.y == cy && b.z == cz) return b.w;
    pos = (pos + 1) & mask;
  }
  return -1;
}

template <bool WANT_H>
struct PointAcc {
  float m[6];  // sum w*M  (xx xy xz yy yz zz)
  float v[3];  // sum w*M*e
  float err;
};

// one correspondence: S = C_B + R C_A R^T (symmetric), M = S^-1 by cofactors (Eigen Matrix3f::inverse), w = sqrt(n);
// `hit` = false contributes exactly zero (the voxel record read for a miss is voxel 0, only there to keep the load
// unconditional so that all loads of a lane can be in flight together).
template <bool WANT_H>
__device__ __forceinline__ void accumulate_voxel(float4 mn, float4 c0, float4 c1, bool hit, const float* rcr, float3 pe, PointAcc<WANT_H>& acc, int ndt, float res) {
  int np = __float_as_int(mn.w);
  if (ndt ? (np <= 6) : (WANT_H && np <= 0)) hit = false;  // ndt_compute_derivatives.cu:61,132 / compute_derivatives.cu:62-64
  float a = c0.x + rcr[0], b = c0.y + rcr[1], c = c0.z + rcr[2], d = c0.w + rcr[3], e = c1.x + rcr[4], f = c1.y + rcr[5];
  float k00 = d * f - e * e, k01 = c * e - b * f, k02 = b * e - c * d;
  float det = (a * k00 + b * k01) + c * k02;
  float id_ = 1.0f / det;
  float m00 = k00 * id_, m01 = k01 * id_, m02 = k02 * id_;
  float m11 = (a * f - c * c) * id_, m12 = (b * c - a * e) * id_, m22 = (a * d - b * b) * id_;
  float ex = mn.x - pe.x, ey = mn.y - pe.y, ez = mn.z - pe.z;
  float w;
  if (ndt) {  // cauchy(resolution, |e|) = k^2 / (k^2 + x^2), ndt_compute_derivatives.cu:15-18,78,150
    float x = sqrtf((ex * ex + ey * ey) + ez * ez);
    float k_sq = res * res;
    w = k_sq / (k_sq + x * x);
  } else {
    w = sqrtf((float)np);
  }
  if (!hit) w = 0.0f;
  float mex = (m00 * ex + m01 * ey) + m02 * ez;
  float mey = (m01 * ex + m11 * ey) + m12 * ez;
  float mez = (m02 * ex + m12 * ey) + m22 * ez;
  if (hit) {
    acc.err += w * ((ex * mex + ey * mey) + ez * mez);
    if (WANT_H) {
      acc.m[0] += w * m00; acc.m[1] += w * m01; acc.m[2] += w * m02; acc.m[3] += w * m11; acc.m[4] += w * m12; acc.m[5] += w * m22;
      acc.v[0] += w * mex; acc.v[1] += w * mey; acc.v[2] += w * mez;
    }
  }
}

// neighbour offset number o of the reference's fixed tables (fast_vgicp_cuda.cu:57-74)
template <int MODE>
__device__ __forceinline__ int3 fixed_offset(int o) {
  if (MODE == 27) return make_int3(o / 9 - 1, (o / 3) % 3 - 1, o % 3 - 1);  // i-major
  if (MODE == 7) {
    // {0,0,0},{1,0,0},{-1,0,0},{0,1,0},{0,-1,0},{0,0,1},{0,0,-1}
    int axis = (o - 1) >> 1, sgn = (o & 1) ? 1 : -1;
    return make_int3(o > 0 && axis == 0 ? sgn : 0, o > 0 && axis == 1 ? sgn : 0, o > 0 && axis == 2 ? sgn : 0);
  }
  return make_int3(0, 0, 0);
}

// J = [skew(pe) | -I] applied to one correspondence's  wM (symmetric-packed), wMe and w e^T M e, added to the lane's 28 running sums:
//   B = S*wM (3x3), A = -B*S, with S = skew(pe);  H = [[A, B],[B^T, wM]],  b = [-(pe x wMe); -wMe]
template <bool WANT_H>
__device__ __forceinline__ void apply_jacobian(float3 pe, const PointAcc<WANT_H>& acc, float* sum) {
  sum[0] += acc.err;
  if (WANT_H) {
    const float* M = acc.m;  // xx xy xz yy yz zz
    float Mf[9] = {M[0], M[1], M[2], M[1], M[3], M[4], M[2], M[4], M[5]};
    float B[9];
#pragma unroll
    for (int j = 0; j < 3; j++) {
      B[0 * 3 + j] = pe.y * Mf[2 * 3 + j] - pe.z * Mf[1 * 3 + j];
      B[1 * 3 + j] = pe.z * Mf[0 * 3 + j] - pe.x * Mf[2 * 3 + j];
      B[2 * 3 + j] = pe.x * Mf[1 * 3 + j] - pe.y * Mf[0 * 3 + j];
    }
    // (B*S)[i][0] = B[i][1]*pz - B[i][2]*py ; [i][1] = -B[i][0]*pz + B[i][2]*px ; [i][2] = B[i][0]*py - B[i][1]*px
    sum[1] += -(B[1] * pe.z - B[2] * pe.y);
    sum[2] += -(-B[0] * pe.z + B[2] * pe.x);
    sum[3] += -(B[0] * pe.y - B[1] * pe.x);
    sum[4] += -(-B[3] * pe.z + B[5] * pe.x);
    sum[5] += -(B[3] * pe.y - B[4] * pe.x);
    sum[6] += -(B[6] * pe.y - B[7] * pe.x);
#pragma unroll
    for (int j = 0; j < 9; j++) sum[7 + j] += B[j];
#pragma unroll
    for (int j = 0; j < 6; j++) sum[16 + j] += M[j];
    sum[22] += -(pe.y * acc.v[2] - pe.z * acc.v[1]);
    sum[23] += -(pe.z * acc.v[0] - pe.x * acc.v[2]);
    sum[24] += -(pe.x * acc.v[1] - pe.y * acc.v[0]);
    sum[25] += -acc.v[0]; sum[26] += -acc.v[1]; sum[27] += -acc.v[2];
  }
}

// per-warp staging for the compacted evaluation (below)
constexpr int kLinQueue = 256;  // ring of pending (slot, voxel) hits: a pass adds at most 4*32, a batch of 32 is drained whenever one is full
struct LinWarpStage {
  float pe[3][32];    // evaluation-pose point of the warp's current points (slot-major inside each component: conflict-free)
  float rcr[6][32];   // R C_A R^T, symmetric-packed
  int queue[kLinQueue];
};

// one correspondence from the queue: entry = slot << 27 | voxel id
template <bool WANT_H>
__device__ __forceinline__ void lin_process_hit(const LinArgs& a, const LinWarpStage& st, int entry, float* sum) {
  const int slot = (int)((unsigned)entry >> 27), id = entry & 0x7ffffff;
  const float4* vr = reinterpret_cast<const float4*>(a.vox + id);
  const float4 mn = __ldg(vr), c0 = __ldg(vr + 1), c1 = __ldg(vr + 2);
  const float3 pe = make_float3(st.pe[0][slot], st.pe[1][slot], st.pe[2][slot]);
  float rcr[6];
#pragma unroll
  for (int q = 0; q < 6; q++) rcr[q] = st.rcr[q][slot];
  PointAcc<WANT_H> acc;
#pragma unroll
  for (int q = 0; q < 6; q++) acc.m[q] = 0.f;
  acc.v[0] = acc.v[1] = acc.v[2] = 0.f;
  acc.err = 0.f;
  accumulate_voxel<WANT_H>(mn, c0, c1, true, rcr, pe, acc, a.ndt, a.res);
  apply_jacobian<WANT_H>(pe, acc, sum);
}

// MODE: 0 = offsets from memory (DIRECT_RADIUS or anything), 1 / 7 / 27 = the reference's fixed tables.
// Two phases per warp and set of 32/G source points, so that both run at full lane efficiency:
//  (1) lookup: G lanes share one point and split its neighbour cells (lane s takes offsets s, s+G, ...), the bucket probes
//      of a lane (<= 4 per pass) are in flight together; only ~28 % of the probed cells hold a voxel, so nothing but the
//      lookup itself happens here -- every hit is appended (ballot + prefix) to a per-warp queue in shared memory;
//  (2) accumulate: whenever 32 hits are queued each lane takes ONE (point, voxel) correspondence: voxel record loads, the
//      3x3 inversion and the Jacobian products run with all lanes busy instead of ~9 of 32.
// The per-point terms (evaluation-pose point, R C_A R^T) are computed once per point and staged in shared memory.
// The running sums are per lane over whatever correspondences the lane drew: the total is a sum over all of them anyway,
// and the assignment depends only on the data, so the result is reproducible run to run.
__device__ __forceinline__ LinWarpStage& lin_stage() {
  __shared__ LinWarpStage stage[kLinThreads / 32];
  return stage[threadIdx.x >> 5];
}

// COUNT: sum[NV] also counts the (source point, voxel) hits under Tl -- the length of the reference's correspondence list
template <int MODE, bool WANT_H, int G, bool DENSE, bool COUNT = false>
__device__ __forceinline__ void lin_accumulate_impl(const LinArgs& a, const Pose& Tl, const Pose& Te, float* sum) {
  constexpr int NV = WANT_H ? kLinValues : 1;
  constexpr int NOFF = MODE == 0 ? 0 : MODE;
  // MODE 27: a lane walks whole z-columns (3 cells sharing the x,y hash prefix) of a contiguous run of 27/G cells, G in {1, 3, 9}
  constexpr bool COLUMNS = (MODE == 27);
  static_assert(MODE != 27 || G == 1 || G == 3 || G == 9, "DIRECT27 splits its 9 z-columns over 1, 3 or 9 lanes");
  constexpr int CELLS = COLUMNS ? 3 : (MODE == 0 ? 4 : ((NOFF + G - 1) / G < 4 ? (NOFF + G - 1) / G : 4));  // cells per lane per pass (loads in flight)
  constexpr int TPW = (32 / G) * G;  // (point, lane) tasks per warp: whole points only (30 of 32 lanes at G = 3, 27 at G = 9)
  LinWarpStage& st = lin_stage();
  const int lane = threadIdx.x & 31;
  const unsigned lt_mask = (1u << lane) - 1u;
#pragma unroll
  for (int i = 0; i < NV + (COUNT ? 1 : 0); i++) sum[i] = 0.f;
  const int n_off = MODE == 0 ? a.n_off : NOFF;
  const int n_pass = COLUMNS ? 9 / G : (n_off + G * CELLS - 1) / (G * CELLS);
  const long long n_tasks = (long long)a.n * G;
  constexpr int kWarps = kLinThreads / 32;
  // warp-uniform trip count (the body uses warp votes): lanes past the end are clamped onto the last task and masked out
  for (long long base = ((long long)blockIdx.x * kWarps + (threadIdx.x >> 5)) * TPW; base < n_tasks; base += (long long)gridDim.x * kWarps * TPW) {
    const long long task_raw = base + lane;
    const bool active = lane < TPW && task_raw < n_tasks;
    const long long task = active ? task_raw : n_tasks - 1;
    const int i = (int)(task / G);
    const int sub = (int)(task % G);
    const int slot = (lane / G) & 31;
    const float4 p = a.pts[i];
    const float3 pl = transform_point(Tl, p.x, p.y, p.z);
    __syncwarp();  // the previous set's hits are all consumed before its staging is overwritten
    if (sub == 0) {
      const float4 ca = a.covA[i];
      const float2 cb = a.covB[i];
      const float3 pe = transform_point(Te, p.x, p.y, p.z);
      st.pe[0][slot] = pe.x; st.pe[1][slot] = pe.y; st.pe[2][slot] = pe.z;
      // RCR = R_lin C_A R_lin^T  (compute_derivatives.cu:75), symmetric-packed
      const float* R = Tl.r;
      float t[9];  // T = R*C
#pragma unroll
      for (int r = 0; r < 3; r++) {
        t[r * 3 + 0] = (R[r * 3] * ca.x + R[r * 3 + 1] * ca.y) + R[r * 3 + 2] * ca.z;
        t[r * 3 + 1] = (R[r * 3] * ca.y + R[r * 3 + 1] * ca.w) + R[r * 3 + 2] * cb.x;
        t[r * 3 + 2] = (R[r * 3] * ca.z + R[r * 3 + 1] * cb.x) + R[r * 3 + 2] * cb.y;
      }
      st.rcr[0][slot] = (t[0] * R[0] + t[1] * R[1]) + t[2] * R[2];
      st.rcr[1][slot] = (t[0] * R[3] + t[1] * R[4]) + t[2] * R[5];
      st.rcr[2][slot] = (t[0] * R[6] + t[1] * R[7]) + t[2] * R[8];
      st.rcr[3][slot] = (t[3] * R[3] + t[4] * R[4]) + t[5] * R[5];
      st.rcr[4][slot] = (t[3] * R[6] + t[4] * R[7]) + t[5] * R[8];
      st.rcr[5][slot] = (t[6] * R[6] + t[7] * R[7]) + t[8] * R[8];
    }
    const int bx = voxel_coord1(pl.x, a.res), by = voxel_coord1(pl.y, a.res), bz = voxel_coord1(pl.z, a.res);
    unsigned head = 0, tail = 0;  // warp-uniform ring indices

    // the 27 neighbours share hash prefixes (vector3i_hash folds x, then y, then z): 9 + 9 + 27 folds instead of 81
    uint64_t kzm[3] = {0, 0, 0};
    if (COLUMNS && !DENSE) {
#pragma unroll
      for (int d = 0; d < 3; d++) kzm[d] = hash_mix((uint64_t)(int64_t)(bz + d - 1));
    }
    for (int pass = 0; pass < n_pass; pass++) {  // same trip count in every lane (warp votes below)
      const int o0 = COLUMNS ? sub * (27 / G) + pass * 3 : pass * (G * CELLS) + sub;
      int cx[CELLS], cy[CELLS], cz[CELLS], found[CELLS];
      bool valid[CELLS];
#pragma unroll
      for (int j = 0; j < CELLS; j++) {
        const int o = COLUMNS ? o0 + j : o0 + j * G;
        valid[j] = active && o < n_off;
        int3 off;
        if (MODE == 0) {
          int4 t4 = __ldg(&a.offsets[valid[j] ? o : 0]);
          off = make_int3(t4.x, t4.y, t4.z);
        } else {
          off = fixed_offset<MODE>(valid[j] ? o : 0);
        }
        cx[j] = bx + off.x; cy[j] = by + off.y; cz[j] = bz + off.z;
      }
      if (DENSE) {  // one 4-byte load per cell (the three cells of a z-column are adjacent)
#pragma unroll
        for (int j = 0; j < CELLS; j++) {
          const int off = dense_offset(a.dense, cx[j], cy[j], cz[j]);
          found[j] = (valid[j] && off >= 0) ? __ldg(&a.dense.cells[off]) : -1;
        }
      } else {
        // all first-probe bucket loads of this lane in flight together
        unsigned pos[CELLS];
        int4 bk[CELLS];
        uint64_t hxy = 0;
        if (COLUMNS) {  // o0 = 9*ix + 3*iy (i-major order of fast_vgicp_cuda.cu:68-74), cells o0, o0+1, o0+2 = iz 0..2
          const int ix = o0 / 9, iy = (o0 / 3) % 3;
          hxy = hash_fold(hash_fold(0, hash_mix((uint64_t)(int64_t)(bx + ix - 1))), hash_mix((uint64_t)(int64_t)(by + iy - 1)));
        }
#pragma unroll
        for (int j = 0; j < CELLS; j++) {
          const uint64_t hsh = COLUMNS ? hash_fold(hxy, kzm[j]) : vector3i_hash(cx[j], cy[j], cz[j]);
          pos[j] = (unsigned)(hsh & a.mask);
          bk[j] = __ldg(&a.buckets[pos[j]]);
        }
        // resolve (find_voxel_correspondences.cu:39-51)
#pragma unroll
        for (int j = 0; j < CELLS; j++) {
          int4 b = bk[j];
          found[j] = -1;
          for (int s = 0; s < a.max_scan; s++) {
            if (b.w < 0) break;
            if (b.x == cx[j] && b.y == cy[j] && b.z == cz[j]) { found[j] = b.w; break; }
            pos[j] = (pos[j] + 1) & a.mask;
            if (s + 1 < a.max_scan) b = __ldg(&a.buckets[pos[j]]);
          }
        }
      }
      // queue the hits
#pragma unroll
      for (int j = 0; j < CELLS; j++) {
        const bool hit = valid[j] && found[j] >= 0;
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (hit) st.queue[(tail + __popc(m & lt_mask)) & (kLinQueue - 1)] = (slot << 27) | found[j];
        tail += __popc(m);
        if (COUNT && hit) sum[NV] += 1.f;  // (exact: a lane sees far fewer than 2^24 hits)
      }
      __syncwarp();
      while (tail - head >= 32u) {  // full batches: one correspondence per lane
        lin_process_hit<WANT_H>(a, st, st.queue[(head + lane) & (kLinQueue - 1)], sum);
        head += 32u;
      }
    }
    if (tail != head) {  // the set's last, partial batch
      if (lane < (int)(tail - head)) lin_process_hit<WANT_H>(a, st, st.queue[(head + lane) & (kLinQueue - 1)], sum);
    }
  }
}

template <int MODE, bool WANT_H, int G, bool COUNT = false>
__device__ __forceinline__ void lin_accumulate(const LinArgs& a, const Pose& Tl, const Pose& Te, float* sum) {
  if (a.dense.cells) lin_accumulate_impl<MODE, WANT_H, G, true, COUNT>(a, Tl, Te, sum);  // (grid-uniform branch)
  else lin_accumulate_impl<MODE, WANT_H, G, false, COUNT>(a, Tl, Te, sum);
}

// block reduction (warp shuffles in float -> shared in double -> per-block partial), ticket, fixed-order fold by the last
// block.  Returns true in every thread of the last block; the folded sums are then in fin[0][0..NV).
// (Tried and dropped: a first-level reduction over distributed shared memory inside 8-block clusters, so that the last block folds
// grid/8 partials.  It gained little at 17 k points and lost at 1 M points, where the cluster placement constraint left SMs idle
// at the tail of the single wave.)
// `partials` ([gridDim.x][kLinStride]) and `ticket` belong to one evaluation: a.partials / a.ticket, or one hypothesis's slice of a
// multi-pose launch
template <int NV>
__device__ __forceinline__ bool lin_reduce(const LinArgs& a, const float* sum, double (*fin)[kLinStride], double* partials, unsigned int* ticket) {
  // ---- block reduction: warp shuffles (float) -> shared (double) -> per-block partial ----
  __shared__ double sh[kLinThreads / 32][kLinStride];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    float v = sum[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sh[wid][i] = (double)v;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kLinThreads / 32; w++) s += sh[w][threadIdx.x];
    partials[(size_t)blockIdx.x * kLinStride + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return false;
  __threadfence();
  // ---- last block: fold the per-block partials in block order (4 interleaved chains per value) ----
  {
    const int v = threadIdx.x & 31, chain = threadIdx.x >> 5;  // kLinThreads == 128 -> 4 chains
    if (v < NV) {
      // ld.global.cg: coherent at L2 (the partials were written by other SMs), 16 independent loads in flight per
      // round -- a dependent load->add chain over hundreds of blocks serialises on L2 latency
      double s = 0.0;
      const double* part = partials + v;
      unsigned b = chain;
      for (; b + 4 * 15 < gridDim.x; b += 4 * 16) {
        double t[16];
#pragma unroll
        for (int u = 0; u < 16; u++) t[u] = __ldcg(part + (size_t)(b + 4 * u) * kLinStride);
#pragma unroll
        for (int u = 0; u < 16; u++) s += t[u];
      }
      for (; b < gridDim.x; b += 4) s += __ldcg(part + (size_t)b * kLinStride);
      fin[chain][v] = s;
    }
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double s = ((fin[0][threadIdx.x] + fin[1][threadIdx.x]) + fin[2][threadIdx.x]) + fin[3][threadIdx.x];
    fin[0][threadIdx.x] = s;
  }
  __syncthreads();
  if (a.comm_ranks > 1) {
    // ---- fused exchange: store this rank's sums into every peer's mailbox over NVLink, publish, wait for the peers,
    // add in rank order (identical doubles in identical order on every rank -> identical LM decisions everywhere) ----
    const int half = (int)(a.comm_seq & 1ULL);
    const unsigned long long tag = a.comm_seq + 1ULL;
    if (threadIdx.x < NV) {
      const double mine = fin[0][threadIdx.x];
      for (int p = 0; p < a.comm_ranks; p++) a.comm_peers[p]->vals[half][a.comm_rank][threadIdx.x] = mine;
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < a.comm_ranks) {
      a.comm_peers[threadIdx.x]->flags[half][a.comm_rank] = tag;  // one publisher thread per peer
      __threadfence_system();
      CommMailbox* me = a.comm_peers[a.comm_rank];
      long long spins = 0;
      while (me->flags[half][threadIdx.x] != tag) {  // thread q waits for rank q
        if (++spins > (1LL << 31)) { me->error = 1; break; }
      }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < NV) {
      const CommMailbox* me = a.comm_peers[a.comm_rank];
      double s = 0.0;
      for (int q = 0; q < a.comm_ranks; q++) s += *reinterpret_cast<const volatile double*>(&me->vals[half][q][threadIdx.x]);
      fin[0][threadIdx.x] = s;
    }
    if (threadIdx.x == 0) a.out[kLinOutCommError] = (double)a.comm_peers[a.comm_rank]->error;  // sticky; the host turns it into VGICP_ERR_COMM
    __syncthreads();
  }
  return true;
}
template <int NV>
__device__ __forceinline__ bool lin_reduce(const LinArgs& a, const float* sum, double (*fin)[kLinStride]) {
  return lin_reduce<NV>(a, sum, fin, a.partials, a.ticket);
}

// unpack the folded sums into err, H (36, column-major), b (6)
template <bool WANT_H>
__device__ __forceinline__ void lin_unpack(const double* s, double* out) {
  out[0] = s[0];
  if (WANT_H) {
    double H[36];
    // A (rows/cols 0..2)
    H[0 * 6 + 0] = s[1]; H[1 * 6 + 0] = H[0 * 6 + 1] = s[2]; H[2 * 6 + 0] = H[0 * 6 + 2] = s[3];
    H[1 * 6 + 1] = s[4]; H[2 * 6 + 1] = H[1 * 6 + 2] = s[5]; H[2 * 6 + 2] = s[6];
    // B: H(r, 3+c) = B[r][c] (column-major index (3+c)*6 + r) and its transpose
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        H[(3 + c) * 6 + r] = s[7 + r * 3 + c];
        H[r * 6 + (3 + c)] = s[7 + r * 3 + c];
      }
    // M (rows/cols 3..5)
    H[3 * 6 + 3] = s[16]; H[4 * 6 + 3] = H[3 * 6 + 4] = s[17]; H[5 * 6 + 3] = H[3 * 6 + 5] = s[18];
    H[4 * 6 + 4] = s[19]; H[5 * 6 + 4] = H[4 * 6 + 5] = s[20]; H[5 * 6 + 5] = s[21];
    for (int j = 0; j < 36; j++) out[1 + j] = H[j];
    for (int j = 0; j < 6; j++) out[37 + j] = s[22 + j];
  }
}

// One evaluation (update_correspondences + compute_error fused).  MODE: 0 = offsets from memory (DIRECT_RADIUS or anything),
// 1 / 7 / 27 = the reference's fixed tables; G = lanes per source point in the lookup phase (see lin_accumulate_impl): at 17k points
// a one-thread-per-point mapping would leave one warp per scheduler with 27 serial dependent lookups per thread.
template <int MODE, bool WANT_H, int G>
__global__ void __launch_bounds__(kLinThreads) k_linearize(const LinArgs a) {
  constexpr int NV = WANT_H ? kLinValues : 1;
  __shared__ double fin[4][kLinStride];
  float sum[NV];
  lin_accumulate<MODE, WANT_H, G>(a, a.Tlin, a.Teval, sum);
  if (!lin_reduce<NV>(a, sum, fin)) return;
  if (threadIdx.x == 0) {
    lin_unpack<WANT_H>(fin[0], a.out);
    *a.ticket = 0u;
    if (a.done_flag) {  // the host spins on this word instead of waiting for the stream (saves the copy + wake-up latency)
      __threadfence_system();
      *a.done_flag = a.done_seq;
    }
  }
}

// Speculative LM evaluation (lsq_registration_impl.hpp:141-160): one launch returns what the optimiser needs to judge a trial
// pose xi = a.Teval -- the error at xi over the correspondences of the current linearisation point a.Tlin (compute_error) -- and
// what it needs next if the step is accepted: the full linearisation AT xi (update_correspondences + compute_error(H, b) with
// Tlin = Teval = xi).  Both are the sums the two separate launches would produce, bit for bit (same grid, same per-lane order);
// an accepted step saves a launch and a host round trip, a rejected one discards the second half.
//   out[0..42] = err, H, b at xi (linearised at xi);  out[43] = err at xi over the old correspondences
template <int MODE, int G>
__device__ __forceinline__ void lin_spec_accumulate(const LinArgs& a, const Pose& Tl, const Pose& Te, float* sum) {  // sum[kLinValues + 1]
  {
    float e_old[1];
    lin_accumulate<MODE, false, G>(a, Tl, Te, e_old);
    sum[kLinValues] = e_old[0];
  }
  {
    float lin[kLinValues];
    lin_accumulate<MODE, true, G>(a, Te, Te, lin);
#pragma unroll
    for (int i = 0; i < kLinValues; i++) sum[i] = lin[i];
  }
}
template <int MODE, int G>
__global__ void __launch_bounds__(kLinThreads) k_linearize_spec(const LinArgs a) {
  constexpr int NV = kLinValues + 1;
  __shared__ double fin[4][kLinStride];
  float sum[NV];
  lin_spec_accumulate<MODE, G>(a, a.Tlin, a.Teval, sum);
  if (!lin_reduce<NV>(a, sum, fin)) return;
  if (threadIdx.x == 0) {
    lin_unpack<true>(fin[0], a.out);
    a.out[43] = fin[0][kLinValues];
    *a.ticket = 0u;
    if (a.done_flag) {
      __threadfence_system();
      *a.done_flag = a.done_seq;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// DIRECT1 on large clouds: the bandwidth-bound shape of the evaluation (one lookup and at most one correspondence per point: about
// 150 instructions against 40 bytes of point + covariance).  The source is streamed through shared memory with the bulk-copy engine:
// an elected thread issues cp.async.bulk (global -> shared, completion counted on an mbarrier) for the point, covA and covB slices
// of the tile kLinStreamStages - 1 tiles ahead, so that the HBM reads of later tiles are in flight while the warps chase the
// dependent loads of the current one (cell index -> voxel record).  No hit compaction: a lane keeps its own point.
// SPEC: error over the correspondences of Tlin at Teval (sum[28]) and the full linearisation at Teval (sums 0..27) from one pass
// over the staged points, like k_linearize_spec.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kLinStreamTile = 128;     // points per tile (1 per thread)
constexpr int kLinStreamStages = 4;
constexpr int kLinStreamMaxBlocks = 8 * kNumSMs;

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

struct LinStreamSmem {
  float4 pts[kLinStreamStages][kLinStreamTile];
  float4 covA[kLinStreamStages][kLinStreamTile];
  float2 covB[kLinStreamStages][kLinStreamTile];
  unsigned long long full[kLinStreamStages];
};

// one point against the voxel of its cell under the linearisation pose Tl, residual at the evaluation pose Te
// (COUNT: the slot after the sums counts the hits, as in lin_accumulate_impl)
template <bool WANT_H, bool COUNT = false>
__device__ __forceinline__ void lin_stream_point(const LinArgs& a, const Pose& Tl, const Pose& Te, float4 p, float4 ca, float2 cb, float* sum) {
  const float3 pl = transform_point(Tl, p.x, p.y, p.z);
  const int off = dense_offset(a.dense, voxel_coord1(pl.x, a.res), voxel_coord1(pl.y, a.res), voxel_coord1(pl.z, a.res));
  const int id = off >= 0 ? __ldg(&a.dense.cells[off]) : -1;
  if (id < 0) return;
  if (COUNT) sum[WANT_H ? kLinValues : 1] += 1.f;
  const float4* vr = reinterpret_cast<const float4*>(a.vox + id);
  const float4 mn = __ldg(vr), c0 = __ldg(vr + 1), c1 = __ldg(vr + 2);
  const float3 pe = transform_point(Te, p.x, p.y, p.z);
  const float* R = Tl.r;
  float t[9], rcr[6];
#pragma unroll
  for (int r = 0; r < 3; r++) {
    t[r * 3 + 0] = (R[r * 3] * ca.x + R[r * 3 + 1] * ca.y) + R[r * 3 + 2] * ca.z;
    t[r * 3 + 1] = (R[r * 3] * ca.y + R[r * 3 + 1] * ca.w) + R[r * 3 + 2] * cb.x;
    t[r * 3 + 2] = (R[r * 3] * ca.z + R[r * 3 + 1] * cb.x) + R[r * 3 + 2] * cb.y;
  }
  rcr[0] = (t[0] * R[0] + t[1] * R[1]) + t[2] * R[2];
  rcr[1] = (t[0] * R[3] + t[1] * R[4]) + t[2] * R[5];
  rcr[2] = (t[0] * R[6] + t[1] * R[7]) + t[2] * R[8];
  rcr[3] = (t[3] * R[3] + t[4] * R[4]) + t[5] * R[5];
  rcr[4] = (t[3] * R[6] + t[4] * R[7]) + t[5] * R[8];
  rcr[5] = (t[6] * R[6] + t[7] * R[7]) + t[8] * R[8];
  PointAcc<WANT_H> acc;
#pragma unroll
  for (int q = 0; q < 6; q++) acc.m[q] = 0.f;
  acc.v[0] = acc.v[1] = acc.v[2] = 0.f;
  acc.err = 0.f;
  accumulate_voxel<WANT_H>(mn, c0, c1, true, rcr, pe, acc, a.ndt, a.res);
  apply_jacobian<WANT_H>(pe, acc, sum);
}

// WHAT: 0 = error only, 1 = linearisation (H, b, err), 2 = speculative (both).  COUNT (WHAT 0 / 1): one more slot counts the hits.
template <int WHAT, bool COUNT = false>
__device__ __forceinline__ void lin_stream_accumulate(const LinArgs& a, const Pose& Tl, const Pose& Te, float* sum) {
  constexpr int NV = (WHAT == 0 ? 1 : (WHAT == 1 ? kLinValues : kLinValues + 1)) + (COUNT ? 1 : 0);
  static_assert(!COUNT || WHAT != 2, "the speculative evaluation does not count hits");
  extern __shared__ __align__(128) unsigned char stream_smem_raw[];
  LinStreamSmem& sm = *reinterpret_cast<LinStreamSmem*>(stream_smem_raw);
  const int tid = threadIdx.x;
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kLinStreamStages; s++) mbar_init(&sm.full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int n_tiles = (a.n + kLinStreamTile - 1) / kLinStreamTile;
  auto issue = [&](int it) {  // tile number it of this block -> stage it % kLinStreamStages
    const long long tile = (long long)blockIdx.x + (long long)it * gridDim.x;
    if (tile >= n_tiles) return;
    const int s = it % kLinStreamStages;
    const int first = (int)tile * kLinStreamTile;
    const int cnt = min(kLinStreamTile, a.n - first);
    const int cnt2 = (cnt + 1) & ~1;  // covB is 8 bytes per point: whole 16-byte units (the arrays are padded by at least one element)
    mbar_expect_tx(&sm.full[s], (unsigned)(cnt * 32 + cnt2 * 8));
    bulk_copy_g2s(sm.pts[s], a.pts + first, (unsigned)cnt * 16u, &sm.full[s]);
    bulk_copy_g2s(sm.covA[s], a.covA + first, (unsigned)cnt * 16u, &sm.full[s]);
    bulk_copy_g2s(sm.covB[s], a.covB + first, (unsigned)cnt2 * 8u, &sm.full[s]);
  };
  if (tid == 0)
    for (int it = 0; it < kLinStreamStages - 1; it++) issue(it);
#pragma unroll
  for (int i = 0; i < NV; i++) sum[i] = 0.f;
  for (int it = 0;; it++) {
    const long long tile = (long long)blockIdx.x + (long long)it * gridDim.x;
    if (tile >= n_tiles) break;
    const int s = it % kLinStreamStages;
    if (tid == 0) issue(it + kLinStreamStages - 1);  // refills the stage read in iteration it - 1 (all threads are past its barrier)
    mbar_wait(&sm.full[s], (unsigned)((it / kLinStreamStages) & 1));
    const int first = (int)tile * kLinStreamTile;
#pragma unroll
    for (int u = 0; u < kLinStreamTile / kLinThreads; u++) {
      const int j = u * kLinThreads + tid;
      if (first + j < a.n) {
        const float4 p = sm.pts[s][j], ca = sm.covA[s][j];
        const float2 cb = sm.covB[s][j];
        if (WHAT == 0) {
          lin_stream_point<false, COUNT>(a, Tl, Te, p, ca, cb, sum);
        } else if (WHAT == 1) {
          lin_stream_point<true, COUNT>(a, Tl, Te, p, ca, cb, sum);
        } else {
          lin_stream_point<false>(a, Tl, Te, p, ca, cb, sum + kLinValues);
          lin_stream_point<true>(a, Te, Te, p, ca, cb, sum);
        }
      }
    }
    __syncthreads();  // the stage may be overwritten by the copy issued in the next iteration
  }
}
template <int WHAT>
__global__ void __launch_bounds__(kLinThreads) k_linearize_stream(const LinArgs a) {
  constexpr int NV = WHAT == 0 ? 1 : (WHAT == 1 ? kLinValues : kLinValues + 1);
  __shared__ double fin[4][kLinStride];
  const int tid = threadIdx.x;
  float sum[NV];
  lin_stream_accumulate<WHAT>(a, a.Tlin, a.Teval, sum);
  if (!lin_reduce<NV>(a, sum, fin)) return;
  if (tid == 0) {
    if (WHAT == 0) {
      lin_unpack<false>(fin[0], a.out);
    } else {
      lin_unpack<true>(fin[0], a.out);
      if (WHAT == 2) a.out[43] = fin[0][kLinValues];
    }
    *a.ticket = 0u;
    if (a.done_flag) {
      __threadfence_system();
      *a.done_flag = a.done_seq;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Multi-pose evaluation (vgicp_align_multi / vgicp_evaluate_poses): one launch evaluates many hypotheses -- poses of the same
// source against the same map.  blockIdx.y is a row of the launch; row y evaluates hypothesis hyp[y] with the poses the host
// wrote to the device array for this launch.  Every row has exactly the single-pose launch's gridDim.x, lane assignment and
// fixed-order fold (the same accumulate functions, lin_reduce over the row's own partial slice and ticket), so each row's sums
// are the single-pose evaluation's sums bit for bit.
// ---------------------------------------------------------------------------------------------------------------
// (The multi-pose kernels declare a minimum of one block per SM: without it ptxas capped some of them at 64 / 72 registers and spilled.)
constexpr int kMultiMaxHyp = 4096;
constexpr int kMultiOut = 48;        // per-row record: [0..42] err, H, b;  [43] speculative: err over the old correspondences;
constexpr int kMultiOutCount = 44;   //                 [44] hit count (the length of the reference's correspondence list)

struct MultiArgs {
  const int* hyp;            // [gridDim.y]: hypothesis evaluated by each row
  const Pose* poses;         // [hypothesis][2] = Tlin, Teval
  double* partials;          // [gridDim.y][gridDim.x][kLinStride]
  unsigned int* tickets;     // [gridDim.y]: zero before the first launch; reset by each row's last block
  double* out;               // [gridDim.y][kMultiOut]; may be mapped pinned host memory
  volatile unsigned long long* done;  // optional [gridDim.y] (mapped host memory): set to done_seq once the row's record is complete
  unsigned long long done_seq;
};

// the row's Tlin, Teval staged in shared memory (sp[0], sp[1]): read like the single-pose kernels' parameter-space poses, without
// holding 24 more registers (which made ptxas spill in the error-only kernels)
__device__ __forceinline__ int multi_row(const MultiArgs& m, Pose* sp) {
  const int y = blockIdx.y;
  constexpr int kWords = 2 * (int)(sizeof(Pose) / sizeof(float));
  if (threadIdx.x < kWords) reinterpret_cast<float*>(sp)[threadIdx.x] = __ldg(reinterpret_cast<const float*>(m.poses + 2 * m.hyp[y]) + threadIdx.x);
  __syncthreads();
  return y;
}
template <int NV>
__device__ __forceinline__ bool multi_reduce(const LinArgs& a, const MultiArgs& m, int y, const float* sum, double (*fin)[kLinStride]) {
  return lin_reduce<NV>(a, sum, fin, m.partials + (size_t)y * gridDim.x * kLinStride, m.tickets + y);
}
// thread 0 of a row's last block, after its record is written
__device__ __forceinline__ void multi_publish(const MultiArgs& m, int y) {
  m.tickets[y] = 0u;
  if (m.done) {
    __threadfence_system();
    m.done[y] = m.done_seq;
  }
}

template <int MODE, bool WANT_H, int G, bool COUNT>
__global__ void __launch_bounds__(kLinThreads, 1) k_linearize_multi(const LinArgs a, const MultiArgs m) {
  constexpr int NV = (WANT_H ? kLinValues : 1) + (COUNT ? 1 : 0);
  __shared__ double fin[4][kLinStride];
  __shared__ Pose sp[2];
  const int y = multi_row(m, sp);
  float sum[NV];
  lin_accumulate<MODE, WANT_H, G, COUNT>(a, sp[0], sp[1], sum);
  if (!multi_reduce<NV>(a, m, y, sum, fin)) return;
  if (threadIdx.x == 0) {
    double* rec = m.out + (size_t)y * kMultiOut;
    lin_unpack<WANT_H>(fin[0], rec);
    if (COUNT) rec[kMultiOutCount] = fin[0][NV - 1];
    multi_publish(m, y);
  }
}

template <int MODE, int G>
__global__ void __launch_bounds__(kLinThreads, 1) k_linearize_spec_multi(const LinArgs a, const MultiArgs m) {
  constexpr int NV = kLinValues + 1;
  __shared__ double fin[4][kLinStride];
  __shared__ Pose sp[2];
  const int y = multi_row(m, sp);
  float sum[NV];
  lin_spec_accumulate<MODE, G>(a, sp[0], sp[1], sum);
  if (!multi_reduce<NV>(a, m, y, sum, fin)) return;
  if (threadIdx.x == 0) {
    double* rec = m.out + (size_t)y * kMultiOut;
    lin_unpack<true>(fin[0], rec);
    rec[43] = fin[0][kLinValues];
    multi_publish(m, y);
  }
}

template <int WHAT, bool COUNT>
__global__ void __launch_bounds__(kLinThreads, 1) k_linearize_stream_multi(const LinArgs a, const MultiArgs m) {
  constexpr int NB = WHAT == 0 ? 1 : (WHAT == 1 ? kLinValues : kLinValues + 1);
  constexpr int NV = NB + (COUNT ? 1 : 0);
  __shared__ double fin[4][kLinStride];
  __shared__ Pose sp[2];
  const int y = multi_row(m, sp);
  float sum[NV];
  lin_stream_accumulate<WHAT, COUNT>(a, sp[0], sp[1], sum);
  if (!multi_reduce<NV>(a, m, y, sum, fin)) return;
  if (threadIdx.x == 0) {
    double* rec = m.out + (size_t)y * kMultiOut;
    if (WHAT == 0) {
      lin_unpack<false>(fin[0], rec);
    } else {
      lin_unpack<true>(fin[0], rec);
      if (WHAT == 2) rec[43] = fin[0][kLinValues];
    }
    if (COUNT) rec[kMultiOutCount] = fin[0][NB];
    multi_publish(m, y);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Device-resident optimiser: LsqRegistration::computeTransformation (lsq_registration_impl.hpp:53-79) with step_gn
// (:106-120) / step_lm (:123-168) as a chain of evaluation kernels.  Each launch reads the phase and the two poses from
// the state block, evaluates (linearize = lookup at x0 + H,b,err ; or error only at the candidate xi with the
// correspondences of x0), and thread 0 of its last block advances the state machine in double -- exactly the host
// logic, same arithmetic (lsq_math.hpp is shared).  A launch that finds phase == DONE returns at once, so the host
// can enqueue a fixed number of launches and read the state back once.
// The state machine is host+device: vgicp_align_multi runs one per hypothesis on the host (host libm, like vgicp_align's loop).
// ---------------------------------------------------------------------------------------------------------------
struct LmState {
  double x0[16], xi[16], delta[16];
  double H[36], b[6], d[6], final_H[36];
  double y0, lambda, nu;
  // parameters
  double rotation_epsilon, transformation_epsilon, lm_init_lambda_factor;
  int max_iterations, lm_max_iterations, use_gauss_newton;
  // progress
  int phase;  // 0 = linearize at x0, 1 = error at xi, 2 = done
  int it, lm_j, converged, lm_failed, n_linearize, n_error, nr_iterations;
  Pose lin_pose, eval_pose;
};
enum { kLmLinearize = 0, kLmError = 1, kLmDone = 2 };

VGICP_HD Pose pose_from_iso(const double* T) {
  Pose p;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) p.r[r * 3 + c] = (float)T[c * 4 + r];
    p.t[r] = (float)T[12 + r];
  }
  return p;
}

VGICP_HD void lm_propose(LmState* st) {  // solve (H + lambda I) d = -b, delta = exp(d), xi = delta * x0   (:134-139)
  double Hl[36], nb[6];
  for (int j = 0; j < 36; j++) Hl[j] = st->H[j];
  for (int q = 0; q < 6; q++) { Hl[q * 7] += st->lambda; nb[q] = -st->b[q]; }
  ldlt_solve6(Hl, nb, st->d);
  Iso3d delta = se3_exp(st->d);
  Iso3d x0;
  for (int j = 0; j < 16; j++) x0.m[j] = st->x0[j];
  Iso3d xi = iso_mul(delta, x0);
  for (int j = 0; j < 16; j++) { st->delta[j] = delta.m[j]; st->xi[j] = xi.m[j]; }
  st->eval_pose = pose_from_iso(st->xi);
  st->phase = kLmError;
}

VGICP_HD void lm_finish_outer(LmState* st) {  // end of step_optimize: converged_ = is_converged(delta), next outer iteration (:65-75)
  Iso3d delta;
  for (int j = 0; j < 16; j++) delta.m[j] = st->delta[j];
  st->converged = is_converged(delta, st->rotation_epsilon, st->transformation_epsilon) ? 1 : 0;
  st->it++;
  if (st->converged || st->it >= st->max_iterations) { st->phase = kLmDone; return; }
  st->nr_iterations = st->it;
  st->lin_pose = pose_from_iso(st->x0);
  st->eval_pose = st->lin_pose;
  st->phase = kLmLinearize;
}

VGICP_HD void lm_advance(LmState* st, const double* out /*err, H, b*/) {
  if (st->phase == kLmLinearize) {
    st->y0 = out[0];
    for (int j = 0; j < 36; j++) st->H[j] = out[1 + j];
    for (int j = 0; j < 6; j++) st->b[j] = out[37 + j];
    st->n_linearize++;
    if (st->use_gauss_newton) {  // step_gn
      double nb[6];
      for (int q = 0; q < 6; q++) nb[q] = -st->b[q];
      ldlt_solve6(st->H, nb, st->d);
      Iso3d delta = se3_exp(st->d), x0;
      for (int j = 0; j < 16; j++) x0.m[j] = st->x0[j];
      x0 = iso_mul(delta, x0);
      for (int j = 0; j < 16; j++) { st->x0[j] = x0.m[j]; st->delta[j] = delta.m[j]; }
      for (int j = 0; j < 36; j++) st->final_H[j] = st->H[j];
      lm_finish_outer(st);
      return;
    }
    if (st->lambda < 0.0) {  // :128-130
      double mx = 0.0;
      for (int j = 0; j < 6; j++) mx = fmax(mx, fabs(st->H[j * 7]));
      st->lambda = st->lm_init_lambda_factor * mx;
    }
    st->nu = 2.0;
    st->lm_j = 0;
    lm_propose(st);
    return;
  }
  // phase == kLmError  (:140-164)
  const double yi = out[0];
  st->n_error++;
  double den = 0.0;
  for (int q = 0; q < 6; q++) den += st->d[q] * (st->lambda * st->d[q] - st->b[q]);
  const double rho = (st->y0 - yi) / den;
  if (rho < 0) {
    Iso3d delta;
    for (int j = 0; j < 16; j++) delta.m[j] = st->delta[j];
    if (is_converged(delta, st->rotation_epsilon, st->transformation_epsilon)) { lm_finish_outer(st); return; }  // :151-154
    st->lambda = st->nu * st->lambda;
    st->nu = 2 * st->nu;
    st->lm_j++;
    if (st->lm_j >= st->lm_max_iterations) {  // step_lm returns false -> "lm not converged!!" (:69-72)
      st->lm_failed = 1;
      st->phase = kLmDone;
      return;
    }
    lm_propose(st);
    return;
  }
  for (int j = 0; j < 16; j++) st->x0[j] = st->xi[j];  // :161-164
  const double f = 1.0 - pow(2.0 * rho - 1.0, 3);
  st->lambda = st->lambda * fmax(1.0 / 3.0, f);
  for (int j = 0; j < 36; j++) st->final_H[j] = st->H[j];
  lm_finish_outer(st);
}

template <int MODE, int G>
__global__ void __launch_bounds__(kLinThreads) k_lm_step(const LinArgs a, LmState* st) {
  __shared__ double fin[4][kLinStride];
  __shared__ double out[44];
  const int phase = st->phase;
  if (phase == kLmDone) return;
  const Pose Tl = st->lin_pose, Te = st->eval_pose;
  bool last;
  if (phase == kLmLinearize) {
    float sum[kLinValues];
    lin_accumulate<MODE, true, G>(a, Tl, Te, sum);
    last = lin_reduce<kLinValues>(a, sum, fin);
  } else {
    float sum[1];
    lin_accumulate<MODE, false, G>(a, Tl, Te, sum);
    last = lin_reduce<1>(a, sum, fin);
  }
  if (!last) return;
  if (threadIdx.x == 0) {
    if (phase == kLmLinearize) lin_unpack<true>(fin[0], out);
    else lin_unpack<false>(fin[0], out);
    lm_advance(st, out);
    __threadfence();
    *a.ticket = 0u;
  }
}

// Materialise the reference's correspondence list for the getter (fast_vgicp_cuda.cu:221-225): dense [n_off][n] voxel ids,
// compacted on the host in offset-major / point-minor order.
__global__ void k_correspondence_ids(const float4* __restrict__ pts, int n, const int4* __restrict__ buckets, unsigned mask, int max_scan, const int4* __restrict__ offsets, int n_off,
                                     float res, const Pose Tlin, int* __restrict__ ids) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = pts[i];
  float3 pl = transform_point(Tlin, p.x, p.y, p.z);
  int bx = voxel_coord1(pl.x, res), by = voxel_coord1(pl.y, res), bz = voxel_coord1(pl.z, res);
  for (int o = 0; o < n_off; o++) {
    int4 off = offsets[o];
    int cx = bx + off.x, cy = by + off.y, cz = bz + off.z;
    ids[(size_t)o * n + i] = lookup_voxel(buckets, mask, max_scan, vector3i_hash(cx, cy, cz), cx, cy, cz);
  }
}

// pcl::Registration::getFitnessScore support: squared distance from every transformed source point to its nearest target
// point (tiled scan of the target through shared memory, one source point per thread).
__global__ void __launch_bounds__(256) k_nn1_sqdist(const float4* __restrict__ src, int n_src, const float4* __restrict__ tgt, int n_tgt, const Pose T, float* __restrict__ out) {
  __shared__ float4 tile[1024];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float3 q = make_float3(0.f, 0.f, 0.f);
  if (i < n_src) {
    float4 p = src[i];
    q = transform_point(T, p.x, p.y, p.z);
  }
  float best = __int_as_float(0x7f800000);
  for (int base = 0; base < n_tgt; base += 1024) {
    __syncthreads();
    for (int j = threadIdx.x; j < 1024; j += blockDim.x) tile[j] = (base + j < n_tgt) ? tgt[base + j] : make_float4(1e30f, 1e30f, 1e30f, 0.f);
    __syncthreads();
    const int lim = min(1024, n_tgt - base);
#pragma unroll 8
    for (int j = 0; j < lim; j++) {
      float4 t = tile[j];
      float dx = t.x - q.x, dy = t.y - q.y, dz = t.z - q.z;
      best = fminf(best, (dx * dx + dy * dy) + dz * dz);
    }
  }
  if (i < n_src) out[i] = best;
}

// pcl::transformPointCloud (lsq_registration_impl.hpp:78): out = T * p, written back in the caller's stride
__global__ void k_transform_points(const float4* __restrict__ pts, int n, const Pose T, unsigned char* __restrict__ out, size_t stride) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = pts[i];
  float3 o = transform_point(T, p.x, p.y, p.z);
  float* dst = reinterpret_cast<float*>(out + (size_t)i * stride);
  dst[0] = o.x; dst[1] = o.y; dst[2] = o.z;
}

}  // namespace vgicp
