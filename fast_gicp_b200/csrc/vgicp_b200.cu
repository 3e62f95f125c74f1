// vgicp_b200.cu -- C-ABI implementation (include/vgicp_b200.h) on top of the kernels in vgicp_kernels.cuh.
// Replaces fast_gicp::cuda::FastVGICPCudaCore (reference src/fast_gicp/cuda/fast_vgicp_cuda.cu:18-284).
// Design: one stream per handle, grow-only device buffers (no allocation in steady state), poses passed as kernel
// arguments (the reference cudaMallocs a device_vector per call, fast_vgicp_cuda.cu:266-267,277-281), one pinned
// 43-double mailbox for the result of an evaluation.
#include "../../include/vgicp_b200.h"

#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <limits>
#include <new>
#include <string>
#include <vector>

#include "lsq_math.hpp"
#include "vgicp_kernels.cuh"

using namespace vgicp;

namespace {

template <typename T>
struct DevBuf {  // grow-only device array
  T* p = nullptr;
  size_t cap = 0;
  bool external = false;  // points into memory owned elsewhere (the multi-GPU exchange arena): fixed capacity, never freed here
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (external) return cudaErrorMemoryAllocation;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 4 + 16;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (p && !external) cudaFree(p);
    p = nullptr;
    cap = 0;
    external = false;
  }
  void attach(T* q, size_t capacity) {  // switch to external storage
    release();
    p = q;
    cap = capacity;
    external = true;
  }
};

struct Cloud {
  DevBuf<float4> pts;
  DevBuf<int> nbr;
  DevBuf<float4> covA;
  DevBuf<float2> covB;
  int n = 0;
  int k = 0;           // neighbours per point currently stored (0 = none)
  bool has_pts = false;
  bool has_cov = false;
  // each cloud has its own stream: the stage-1 work of target and source overlaps on the GPU; `ready` marks the end of the
  // last operation enqueued for this cloud
  cudaStream_t st = nullptr;
  cudaEvent_t ready = nullptr;
  DevBuf<unsigned char> staging;
  DevBuf<unsigned char> knn_scratch;
  const float4* knn_sorted = nullptr;  // the cloud in the k-NN grid's Morton order (inside knn_scratch), original index in .w
  int knn_q_begin = 0, knn_q_end = 0;  // sorted positions whose neighbour rows the last find_neighbors computed
  int arena_slot = 0;                  // which half of the exchange arena holds this cloud's covariances (stage-1 sharding)
  unsigned long long arena_seq = 0;    // slices delivered for this cloud so far
  void release() { pts.release(); nbr.release(); covA.release(); covB.release(); staging.release(); knn_scratch.release(); }
};

constexpr long long kDenseMaxCells = 16ll << 20;  // 64 MB of cell ids per map at most

struct VoxelMap {
  bool created = false;  // GaussianVoxelMap object exists (keeps its first resolution, SURVEY Q3)
  bool built = false;
  bool pending = false;    // first insertion attempt enqueued, outcome not yet read (voxelmap_finish completes the build)
  int pending_B = 0;
  bool v_pending = false;  // num_voxels still in flight
  cudaEvent_t ev_attempt = nullptr, ev_done = nullptr;
  int ndt = 0;             // 1: built from the points alone + MIN_EIG (NDT), 0: from points + covariances (VGICP)
  int* d_counters = nullptr;  // [0] fail count, [1] num_voxels, [2..4] / [5..7] min / max voxel coordinate, [8] set_neighbors verdict
  int* h_counters = nullptr;  // pinned
  DevBuf<unsigned long long> chunk_state;  // k_table_assign_ids look-back (epoch-tagged block totals)
  unsigned chunk_epoch = 0;
  DevBuf<int> dense_cells;    // direct-mapped voxel index over the bounding box (evaluation kernels), when it fits
  DenseIndex dense{nullptr, 0, 0, 0, 0u, 0u, 0u};
  float res = 1.0f;
  int init_num_buckets = 8192;  // gaussian_voxelmap.cuh:20
  int max_scan = 10;            // gaussian_voxelmap.cuh:20
  int num_buckets = 0;
  int num_voxels = 0;
  DevBuf<int4> buckets;
  DevBuf<VoxelRec> vox;
  // build scratch
  DevBuf<int4> coords;
  DevBuf<int> slots;
  DevBuf<int> slot_of_point;
  // points stably sorted by voxel id for the ordered per-voxel sums (vgicp_sort.cuh)
  DevBuf<unsigned> sort_keys[2], sort_vals[2];
  DevBuf<unsigned char> sort_scratch;
  DevBuf<int2> segments;
  void release() {
    buckets.release(); vox.release(); coords.release(); slots.release(); slot_of_point.release(); dense_cells.release(); chunk_state.release();
    for (int j = 0; j < 2; j++) { sort_keys[j].release(); sort_vals[j].release(); }
    sort_scratch.release(); segments.release();
  }
};

}  // namespace

struct vgicp_context {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  uint64_t launches = 0;

  double resolution = 1.0;
  double kernel_width = 0.25;
  double kernel_max_dist = 3.0;
  int offset_mode = 1;  // 1 / 7 / 27 = fixed tables, 0 = generic list
  int voxel_index_mode = 0;  // 0: direct-mapped index when the map's bounding box fits (else the hash table), 1: hash table only
  std::vector<int4> h_offsets;
  DevBuf<int4> d_offsets;

  Cloud source, target;
  VoxelMap map;

  bool has_lin = false;
  Pose lin;  // linearized_x (float)

  DevBuf<unsigned char> staging;    // main-stream scratch (transform_source, fitness score)
  cudaStream_t stream_b = nullptr;  // second cloud stream
  cudaEvent_t ev_copy = nullptr;    // "host buffer consumed" marker of set_cloud
  // multi-GPU source sharding
  CommMailbox* comm_box = nullptr;               // this rank's mailbox (device memory, IPC-exported)
  CommMailbox* comm_peers[kCommMaxRanks] = {};   // mapped peer mailboxes (own included)
  int comm_rank = 0, comm_ranks = 0;
  unsigned long long comm_seq = 0;
  int shard_begin = 0, shard_end = -1;           // evaluations cover source points [begin, end)
  // stage-1 sharding: exchange arena (covariances of both clouds + delivery flags), own and peers' (IPC-mapped)
  unsigned char* arena = nullptr;
  unsigned char* arena_peers[kCommMaxRanks] = {};
  size_t arena_points = 0;
  int stage1_sharding = 0;
  int speculate = 1;  // LM trial evaluations also linearise at the trial pose (vgicp_set_speculation)
  int exec_hint = 0;  // 0 = latency (one registration should finish as soon as possible), 1 = throughput (many concurrent handles)
  int align_mode = 1;  // 1 = host-driven loop over the evaluation kernels (default: faster today), 0 = device-resident LM chain
  LmState* d_lm = nullptr;
  LmState* h_lm = nullptr;  // pinned
  int lin_stream = 1;   // VGICP_LIN_STREAM=0 disables the bulk-copy streaming kernel of DIRECT1 (A/B measurements)
  int force_lin_g = 0;  // VGICP_LIN_G override of the lanes-per-point split (experiments)
  int knn_mode = 0;  // 0 = hash grid (default), 1 = warp-cooperative scan of the whole cloud, 2 = legacy per-thread scan
  DevBuf<double> partials;
  DevBuf<int> corr_ids;
  unsigned int* d_ticket = nullptr;
  double* d_out = nullptr;    // 43 doubles
  double* h_out = nullptr;    // pinned + mapped: in latency mode the kernel's last block writes the result straight here
  unsigned long long* h_flag = nullptr;  // pinned + mapped completion word
  unsigned long long eval_seq = 0;

  // NDT (NDTCudaCore, ndt_cuda.cu): 0 = VGICP problem, 1 = NDT point-to-distribution, 2 = NDT distribution-to-distribution
  int problem = 0;
  VoxelMap ndt_t, ndt_s;        // target / source NDT voxel maps
  DevBuf<float4> ndt_src_pts;   // D2D: source voxel means as the evaluation's source cloud
  DevBuf<float4> ndt_src_covA;  // D2D: source voxel covariances; P2D: zeros
  DevBuf<float2> ndt_src_covB;
  int ndt_src_n = 0;
  bool ndt_ready = false;

  // optional per-kernel timing (vgicp_set_profiling): CUDA events on the handle's stream around every launch
  bool prof_on = false;
  struct ProfRec { int cat; cudaEvent_t a, b; };
  std::vector<ProfRec> prof_pending;
  std::vector<cudaEvent_t> prof_pool;
  double prof_ms[VGICP_PROF_NUM_CATEGORIES] = {0};
  uint64_t prof_launches[VGICP_PROF_NUM_CATEGORIES] = {0};
};

namespace {

int fail(vgicp_handle h, int code, const std::string& msg) {
  if (h) h->err = msg;
  return code;
}

cudaEvent_t prof_event(vgicp_handle h) {
  if (!h->prof_pool.empty()) {
    cudaEvent_t e = h->prof_pool.back();
    h->prof_pool.pop_back();
    return e;
  }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
inline void prof_begin(vgicp_handle h, int cat, cudaStream_t st) {
  h->prof_launches[cat]++;
  if (!h->prof_on) return;
  vgicp_context::ProfRec r{cat, prof_event(h), prof_event(h)};
  cudaEventRecord(r.a, st);
  h->prof_pending.push_back(r);
}
inline void prof_end(vgicp_handle h, cudaStream_t st) {
  if (!h->prof_on) return;
  cudaEventRecord(h->prof_pending.back().b, st);
}
// every kernel launch of the library goes through here: counts it, optionally brackets it with events on its stream
#define KLAUNCH_ST(h, st, cat, ...) \
  do {                              \
    prof_begin(h, cat, st);         \
    __VA_ARGS__;                    \
    prof_end(h, st);                \
    (h)->launches++;                \
  } while (0)
#define KLAUNCH(h, cat, ...) KLAUNCH_ST(h, (h)->stream, cat, __VA_ARGS__)

#define CU_TRY(h, expr)                                                                                       \
  do {                                                                                                        \
    cudaError_t _e = (expr);                                                                                  \
    if (_e != cudaSuccess) return fail(h, VGICP_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

#define CHECK_HANDLE(h) \
  if (!(h)) return VGICP_ERR_INVALID_ARGUMENT

struct DeviceGuard {  // every call runs on the handle's device (the reference uses the current device)
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

inline int blocks_for(size_t n, int threads) { return (int)((n + threads - 1) / threads); }

Pose to_pose(const double* T) {  // Eigen::Isometry3d (column-major) -> float image, like trans.cast<float>()
  Pose p;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) p.r[r * 3 + c] = (float)T[c * 4 + r];
    p.t[r] = (float)T[12 + r];
  }
  return p;
}

int set_cloud(vgicp_handle h, Cloud& c, const float* xyz, size_t n, size_t stride, bool on_device = false) {
  // NDT: set_{source,target}_cloud resets that cloud's voxel map only (ndt_cuda.cu:104,114); it is rebuilt by the next create_voxelmaps
  h->ndt_ready = false;
  {
    VoxelMap& nm = (&c == &h->target) ? h->ndt_t : h->ndt_s;
    nm.built = false;
    nm.pending = false;
  }
  if (n > 0 && !xyz) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_cloud: null points");
  if (stride < 12 || (stride % 4) != 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_cloud: stride_bytes must be a multiple of 4 and >= 12");
  if (n > (size_t)0x7fffffff / 64) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_cloud: too many points");
  CU_TRY(h, c.pts.reserve(n));
  c.n = (int)n;
  c.has_pts = true;
  if (n == 0) return VGICP_OK;
  if (on_device) {  // caller's buffer already lives in this GPU's memory: read it in place (stream-ordered)
    KLAUNCH_ST(h, c.st, VGICP_PROF_UNPACK, k_unpack_points<<<blocks_for(n, 256), 256, 0, c.st>>>(reinterpret_cast<const unsigned char*>(xyz), stride, (int)n, c.pts.p));
    CU_TRY(h, cudaGetLastError());
    CU_TRY(h, cudaEventRecord(c.ready, c.st));
    return VGICP_OK;
  }
  CU_TRY(h, c.staging.reserve(n * stride));
  CU_TRY(h, cudaMemcpyAsync(c.staging.p, xyz, n * stride, cudaMemcpyHostToDevice, c.st));
  // the caller may free/modify xyz after return: pageable copies are staged synchronously by the driver, pinned ones are
  // not -> wait for the copy itself (an event right behind it), not for the kernels that follow
  CU_TRY(h, cudaEventRecord(h->ev_copy, c.st));
  KLAUNCH_ST(h, c.st, VGICP_PROF_UNPACK, k_unpack_points<<<blocks_for(n, 256), 256, 0, c.st>>>(c.staging.p, stride, (int)n, c.pts.p));
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaEventRecord(c.ready, c.st));
  CU_TRY(h, cudaEventSynchronize(h->ev_copy));
  return VGICP_OK;
}

int set_neighbors(vgicp_handle h, Cloud& c, int k, const int* idx, size_t nk) {
  if (!c.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "set_neighbors: cloud not set");
  if (k <= 0 || !idx || nk != (size_t)k * (size_t)c.n) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_neighbors: k * num_points != neighbors.size()");
  CU_TRY(h, c.nbr.reserve(nk));
  CU_TRY(h, cudaMemcpyAsync(c.nbr.p, idx, nk * sizeof(int), cudaMemcpyHostToDevice, c.st));
  // an index outside [0, n) would be an illegal address in k_covariance_knn and poison the context of every handle of the process:
  // one pass over the table, the verdict comes back with the synchronisation the copy needs anyway
  int* bad = h->map.d_counters + 8;
  CU_TRY(h, cudaMemsetAsync(bad, 0, sizeof(int), c.st));
  KLAUNCH_ST(h, c.st, VGICP_PROF_OTHER, k_validate_indices<<<blocks_for(nk, 256) < 8 * kNumSMs ? blocks_for(nk, 256) : 8 * kNumSMs, 256, 0, c.st>>>(c.nbr.p, nk, c.n, bad));
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(h->map.h_counters + 8, bad, sizeof(int), cudaMemcpyDeviceToHost, c.st));
  CU_TRY(h, cudaStreamSynchronize(c.st));
  if (h->map.h_counters[8] != 0) {
    c.k = 0;
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_neighbors: neighbour index outside [0, num_points)");
  }
  c.k = k;
  return VGICP_OK;
}

int find_neighbors(vgicp_handle h, Cloud& c, int k) {
  if (!c.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "find_neighbors: cloud not set");
  if (k <= 0 || k > kMaxK || k > c.n) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "find_neighbors: need 1 <= k <= min(num_points, 64)");
  CU_TRY(h, c.nbr.reserve((size_t)c.n * k));
  cudaError_t ke = cudaSuccess;
  if (h->knn_mode == 2) {  // legacy one-thread-per-query scan, kept for A/B measurements
    c.knn_sorted = nullptr;
    c.knn_q_begin = 0;
    c.knn_q_end = c.n;
    KLAUNCH_ST(h, c.st, VGICP_PROF_KNN, ke = launch_knn_bruteforce(c.pts.p, c.n, k, c.nbr.p, c.st));
  } else {
    const size_t need = knn_grid_scratch_bytes(c.n, nullptr, nullptr);
    CU_TRY(h, c.knn_scratch.reserve(need));
    int nl = 0;
    c.knn_q_begin = 0;
    c.knn_q_end = c.n;
    if (h->stage1_sharding && h->comm_ranks > 1 && h->arena_peers[h->comm_rank]) {  // this rank's slice of the queries (sorted positions)
      const long long base = c.n / h->comm_ranks, rem = c.n % h->comm_ranks, r = h->comm_rank;
      c.knn_q_begin = (int)(r * base + (r < rem ? r : rem));
      c.knn_q_end = c.knn_q_begin + (int)base + (r < rem ? 1 : 0);
    }
    KLAUNCH_ST(h, c.st, VGICP_PROF_KNN, ke = launch_knn_grid(c.pts.p, c.n, k, c.nbr.p, c.knn_scratch.p, c.knn_scratch.cap, (h->knn_mode == 1 || c.n < 256) ? 1 : 0, c.knn_q_begin,
                                                            c.knn_q_end, &nl, &c.knn_sorted, c.st));
    h->launches += nl > 0 ? nl - 1 : 0;
  }
  CU_TRY(h, ke);
  CU_TRY(h, cudaEventRecord(c.ready, c.st));
  c.k = k;
  return VGICP_OK;
}

int calc_covariances(vgicp_handle h, Cloud& c, int method) {
  if (!c.has_pts || c.k <= 0) return fail(h, VGICP_ERR_BAD_STATE, "calculate_covariances: cloud and neighbours must be set first");
  if (method < 0 || method > 4) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "calculate_covariances: bad regularization method");
  CU_TRY(h, c.covA.reserve(c.n));
  CU_TRY(h, c.covB.reserve(c.n));
  const bool sharded = h->stage1_sharding && h->comm_ranks > 1 && h->arena_peers[h->comm_rank] && c.knn_sorted && (c.knn_q_begin > 0 || c.knn_q_end < c.n);
  if (c.n > 0 && sharded) {
    // this rank computed the neighbour rows of a slice only: covariances of that slice go straight into every rank's arena
    // (peer stores), then the ranks tell each other and wait -- all in stream order, the host does not block
    if ((size_t)c.n > h->arena_points) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "calculate_covariances: cloud larger than the exchange arena (vgicp_comm_export_arena max_points)");
    float4* pa[kCommMaxRanks];
    float2* pb[kCommMaxRanks];
    ArenaPeers ap;
    for (int r = 0; r < kCommMaxRanks; r++) {
      unsigned char* base = r < h->comm_ranks ? h->arena_peers[r] : nullptr;
      ap.hdr[r] = reinterpret_cast<CommArenaHeader*>(base);
      pa[r] = base ? reinterpret_cast<float4*>(base + kCommArenaHeaderBytes + (size_t)c.arena_slot * h->arena_points * 24) : nullptr;
      pb[r] = base ? reinterpret_cast<float2*>(reinterpret_cast<unsigned char*>(pa[r]) + h->arena_points * 16) : nullptr;
    }
    cudaError_t ke = cudaSuccess;
    KLAUNCH_ST(h, c.st, VGICP_PROF_COVARIANCE, ke = launch_covariance_knn_sharded(c.pts.p, c.nbr.p, c.knn_sorted, c.knn_q_begin, c.knn_q_end, c.k, method, pa, pb, h->comm_ranks, c.st));
    CU_TRY(h, ke);
    c.arena_seq++;
    KLAUNCH_ST(h, c.st, VGICP_PROF_COVARIANCE, k_comm_deliver_and_wait<<<1, 32, 0, c.st>>>(ap, h->comm_rank, h->comm_ranks, c.arena_slot, c.arena_seq));
    CU_TRY(h, cudaGetLastError());
  } else if (c.n > 0) {
    cudaError_t ke = cudaSuccess;
    KLAUNCH_ST(h, c.st, VGICP_PROF_COVARIANCE, ke = launch_covariance_knn(c.pts.p, c.nbr.p, c.n, c.k, method, c.covA.p, c.covB.p, c.st));
    CU_TRY(h, ke);
  }
  c.has_cov = true;
  CU_TRY(h, cudaEventRecord(c.ready, c.st));
  if (method == VGICP_REG_NORMALIZED_MIN_EIG)
    return fail(h, VGICP_ERR_UNSUPPORTED, "unimplemented covariance regularization method was selected (NORMALIZED_MIN_EIG has no GPU path in the reference either); raw covariances kept");
  return VGICP_OK;
}

int calc_covariances_rbf(vgicp_handle h, Cloud& c, int method) {
  if (!c.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "calculate_covariances_rbf: cloud not set");
  if (method < 0 || method > 4) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "calculate_covariances_rbf: bad regularization method");
  CU_TRY(h, c.covA.reserve(c.n));
  CU_TRY(h, c.covB.reserve(c.n));
  if (c.n > 0) {
    cudaError_t ke = cudaSuccess;
    const size_t box_bytes = sizeof(float) * 6 * (size_t)((c.n + kRbfBlock - 1) / kRbfBlock);
    CU_TRY(h, c.knn_scratch.reserve(box_bytes));  // (the k-NN scratch is idle here: RBF covariances use no neighbour table)
    KLAUNCH_ST(h, c.st, VGICP_PROF_COVARIANCE,
               ke = launch_covariance_rbf(c.pts.p, c.n, (float)h->kernel_width, (float)h->kernel_max_dist, method, reinterpret_cast<float*>(c.knn_scratch.p), c.covA.p, c.covB.p, c.st));
    h->launches++;
    CU_TRY(h, ke);
  }
  c.has_cov = true;
  CU_TRY(h, cudaEventRecord(c.ready, c.st));
  if (method == VGICP_REG_NORMALIZED_MIN_EIG) return fail(h, VGICP_ERR_UNSUPPORTED, "unimplemented covariance regularization method was selected; raw covariances kept");
  return VGICP_OK;
}

int get_covariances(vgicp_handle h, Cloud& c, float* out9, size_t cap) {
  if (!c.has_cov) return fail(h, VGICP_ERR_BAD_STATE, "get_covariances: covariances not computed");
  if (!out9 || cap < (size_t)c.n) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_covariances: buffer too small");
  std::vector<float4> a(c.n);
  std::vector<float2> b(c.n);
  if (c.n) {
    CU_TRY(h, cudaMemcpyAsync(a.data(), c.covA.p, sizeof(float4) * c.n, cudaMemcpyDeviceToHost, c.st));
    CU_TRY(h, cudaMemcpyAsync(b.data(), c.covB.p, sizeof(float2) * c.n, cudaMemcpyDeviceToHost, c.st));
    CU_TRY(h, cudaStreamSynchronize(c.st));
  }
  for (int i = 0; i < c.n; i++) {
    float* o = out9 + (size_t)i * 9;
    o[0] = a[i].x; o[1] = a[i].y; o[2] = a[i].z;
    o[3] = a[i].y; o[4] = a[i].w; o[5] = b[i].x;
    o[6] = a[i].z; o[7] = b[i].x; o[8] = b[i].y;
  }
  return VGICP_OK;
}

int set_covariances(vgicp_handle h, Cloud& c, const float* in9, size_t n) {
  if (!c.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "set_covariances: cloud not set");
  if (!in9 || n != (size_t)c.n) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_covariances: need one 3x3 per point of the cloud");
  CU_TRY(h, c.covA.reserve(c.n));
  CU_TRY(h, c.covB.reserve(c.n));
  std::vector<float4> a(c.n);
  std::vector<float2> b(c.n);
  for (int i = 0; i < c.n; i++) {  // column-major in, symmetric-packed out (the mean of the two triangles, like the kernels)
    const float* m = in9 + (size_t)i * 9;
    a[i] = make_float4(m[0], 0.5f * (m[1] + m[3]), 0.5f * (m[2] + m[6]), m[4]);
    b[i] = make_float2(0.5f * (m[5] + m[7]), m[8]);
  }
  if (c.n) {
    CU_TRY(h, cudaMemcpyAsync(c.covA.p, a.data(), sizeof(float4) * c.n, cudaMemcpyHostToDevice, c.st));
    CU_TRY(h, cudaMemcpyAsync(c.covB.p, b.data(), sizeof(float2) * c.n, cudaMemcpyHostToDevice, c.st));
    CU_TRY(h, cudaStreamSynchronize(c.st));
  }
  c.has_cov = true;
  CU_TRY(h, cudaEventRecord(c.ready, c.st));
  return VGICP_OK;
}

int get_neighbors(vgicp_handle h, Cloud& c, int* out, size_t cap, int* k_out) {
  if (c.k <= 0) return fail(h, VGICP_ERR_BAD_STATE, "get_neighbors: neighbours not set");
  if (k_out) *k_out = c.k;
  size_t need = (size_t)c.n * c.k;
  if (!out || cap < need) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_neighbors: buffer too small");
  if (need) {
    CU_TRY(h, cudaMemcpyAsync(out, c.nbr.p, need * sizeof(int), cudaMemcpyDeviceToHost, c.st));
    CU_TRY(h, cudaStreamSynchronize(c.st));
  }
  return VGICP_OK;
}

// GaussianVoxelMap::create_voxelmap(points, covs): gaussian_voxelmap.cu:233-289, split in two so that the host does not block
// on the table-growth decision while the other cloud's work could be enqueued:
//   voxelmap_begin  enqueues coordinates + the first insertion attempt (8192 buckets) + the read-back of its failure count
//   voxelmap_finish (called by whoever needs the map) waits for that count, grows the table if the reference would
//                   (:265-285), then ids / accumulate / finalize.  num_voxels itself is fetched lazily.
// One or more table attempts (B, 2B, 4B, ...) enqueued back to back; k_table_verdict records the first size that meets the
// reference's rule and the kernels of the later attempts see it and return, so the outcome is that of the reference's sequential
// doubling with one host synchronisation instead of one per attempt (large clouds need 3: 8192 -> 32768 buckets at 1 M points).
int voxelmap_attempt(vgicp_handle h, Cloud& t, VoxelMap& m, int B, int count) {
  const int n = t.n;
  int B_last = B;
  for (int j = 1; j < count && B_last < (1 << 28); j++) B_last *= 2;
  CU_TRY(h, m.slots.reserve(B_last));
  int* skip = m.d_counters + 9;
  CU_TRY(h, cudaMemsetAsync(skip, 0, sizeof(int), t.st));
  int Bj = B;
  for (int j = 0; j < count && Bj <= B_last; j++, Bj *= 2) {
    CU_TRY(h, cudaMemsetAsync(m.d_counters, 0, sizeof(int), t.st));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_fill_i32<<<blocks_for(Bj, 256), 256, 0, t.st>>>(m.slots.p, -1, (size_t)Bj, skip));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_table_insert<<<blocks_for(n, 256), 256, 0, t.st>>>(m.coords.p, n, m.slots.p, (unsigned)(Bj - 1), m.max_scan, skip));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP,
               k_table_lookup_points<<<blocks_for(n, 256), 256, 0, t.st>>>(m.coords.p, n, m.slots.p, (unsigned)(Bj - 1), m.max_scan, m.slot_of_point.p, m.d_counters, skip));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_table_verdict<<<1, 1, 0, t.st>>>(m.d_counters, n, Bj));
  }
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(m.h_counters + 9, m.d_counters + 9, sizeof(int), cudaMemcpyDeviceToHost, t.st));
  CU_TRY(h, cudaEventRecord(m.ev_attempt, t.st));
  m.pending_B = B_last;
  return VGICP_OK;
}

int voxelmap_begin(vgicp_handle h, Cloud& t, VoxelMap& m) {
  if (!t.has_pts || (!m.ndt && !t.has_cov)) return fail(h, VGICP_ERR_BAD_STATE, "create_target_voxelmap: target points and covariances required");
  if (t.n <= 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "create_target_voxelmap: empty target cloud");
  if (!m.created) {  // fast_vgicp_cuda.cu:259-261: created once with the resolution current at that time
    m.created = true;
    m.res = (float)h->resolution;
  }
  m.built = false;
  m.pending = false;
  const int n = t.n;
  CU_TRY(h, m.coords.reserve(n));
  CU_TRY(h, m.slot_of_point.reserve(n));
  CU_TRY(h, cudaMemsetAsync(m.d_counters + 2, 0x7f, 3 * sizeof(int), t.st));  // running minimum: starts at 0x7f7f7f7f
  CU_TRY(h, cudaMemsetAsync(m.d_counters + 5, 0x80, 3 * sizeof(int), t.st));  // running maximum: starts at 0x80808080
  KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_voxel_coords<<<blocks_for(n, 256), 256, 0, t.st>>>(t.pts.p, n, m.res, m.coords.p, m.d_counters + 2));
  CU_TRY(h, cudaMemcpyAsync(m.h_counters + 2, m.d_counters + 2, 6 * sizeof(int), cudaMemcpyDeviceToHost, t.st));
  // small clouds pass with the initial 8192 buckets (1082 voxels at 17 k points); large ones are given three sizes to try at once
  int rc = voxelmap_attempt(h, t, m, m.init_num_buckets, n > 200000 ? 3 : 1);
  if (rc) return rc;
  m.pending = true;
  return VGICP_OK;
}

int voxelmap_finish(vgicp_handle h, Cloud& t, VoxelMap& m) {
  if (!m.pending) return m.built ? VGICP_OK : fail(h, VGICP_ERR_BAD_STATE, "target voxel map not built");
  const int n = t.n;
  int B = 0;
  for (;;) {  // :265 (no upper bound in the reference; bounded here)
    CU_TRY(h, cudaEventSynchronize(m.ev_attempt));
    if (m.h_counters[9] != 0) { B = m.h_counters[9]; break; }  // :280, decided on the device
    B = m.pending_B * 2;
    if (B > (1 << 28)) { m.pending = false; return fail(h, VGICP_ERR_INVALID_ARGUMENT, "create_target_voxelmap: hash table would exceed 2^28 buckets"); }
    int rc = voxelmap_attempt(h, t, m, B, 2);
    if (rc) return rc;
  }
  m.pending = false;
  m.num_buckets = B;
  const int vmax = n < B ? n : B;  // upper bound on the number of voxels: buffers are sized for it, the exact count arrives later
  if (vmax > (1 << 27)) { m.pending = false; return fail(h, VGICP_ERR_INVALID_ARGUMENT, "create_target_voxelmap: more than 2^27 voxels (the evaluation kernels pack a voxel id in 27 bits)"); }
  CU_TRY(h, m.buckets.reserve(B));
  CU_TRY(h, m.vox.reserve(vmax));
  // direct-mapped index for the evaluation kernels, when the bounding box of the voxel coordinates is small enough (LiDAR scans
  // are: 84 x 84 x 10 cells for the 17k fixture, 300 x 300 x 40 at 1M points / 0.5 m); otherwise they probe the hash table
  m.dense.cells = nullptr;
  if (h->voxel_index_mode == 0) {
    const int* hc = m.h_counters;
    const long long nx = (long long)hc[5] - hc[2] + 1, ny = (long long)hc[6] - hc[3] + 1, nz = (long long)hc[7] - hc[4] + 1;
    if (nx > 0 && ny > 0 && nz > 0 && nx <= kDenseMaxCells && ny <= kDenseMaxCells && nz <= kDenseMaxCells && nx * ny <= kDenseMaxCells && nx * ny * nz <= kDenseMaxCells) {
      const size_t cells = (size_t)(nx * ny * nz);
      CU_TRY(h, m.dense_cells.reserve(cells));
      CU_TRY(h, cudaMemsetAsync(m.dense_cells.p, 0xff, cells * sizeof(int), t.st));
      m.dense = DenseIndex{m.dense_cells.p, hc[2], hc[3], hc[4], (unsigned)nx, (unsigned)ny, (unsigned)nz};
    }
  }
  {
    const int chunks = (B + 1023) / 1024;
    const unsigned long long* before = m.chunk_state.p;
    CU_TRY(h, m.chunk_state.reserve(chunks));
    if (m.chunk_state.p != before) {  // fresh allocation: no stale epoch may match
      CU_TRY(h, cudaMemsetAsync(m.chunk_state.p, 0, m.chunk_state.cap * sizeof(unsigned long long), t.st));
      m.chunk_epoch = 0;
    }
    if (++m.chunk_epoch == 0) {  // wrapped: clear once and restart
      CU_TRY(h, cudaMemsetAsync(m.chunk_state.p, 0, m.chunk_state.cap * sizeof(unsigned long long), t.st));
      m.chunk_epoch = 1;
    }
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP,
               k_table_assign_ids<<<chunks, 1024, 0, t.st>>>(m.coords.p, m.slots.p, B, m.buckets.p, m.d_counters + 1, m.dense, m.chunk_state.p, m.chunk_epoch));
  }
  // voxel Gaussians: stable sort of the points by voxel id, then one warp per voxel adds its points in index order
  {
    int key_bits = 1;
    while ((1 << key_bits) < B) key_bits++;
    key_bits += 1;  // ids < B; the all-ones key marks the points of dropped voxels (sorts last)
    const unsigned invalid = (1u << key_bits) - 1u;
    const int passes = sort_num_passes(key_bits);
    const size_t sbytes = sort_scratch_bytes(n, passes);
    for (int j = 0; j < 2; j++) {
      CU_TRY(h, m.sort_keys[j].reserve(n));
      CU_TRY(h, m.sort_vals[j].reserve(n));
    }
    CU_TRY(h, m.sort_scratch.reserve(sbytes));
    CU_TRY(h, m.segments.reserve(vmax));
    CU_TRY(h, cudaMemsetAsync(m.sort_scratch.p, 0, sbytes, t.st));
    const int kb = blocks_for(n, kSortThreads);
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP,
               k_voxel_sort_keys<<<kb < 8 * kNumSMs ? kb : 8 * kNumSMs, kSortThreads, 0, t.st>>>(m.slot_of_point.p, m.buckets.p, n, invalid, passes, m.sort_keys[0].p, reinterpret_cast<unsigned*>(m.sort_scratch.p)));
    int nl = 0;
    cudaError_t se = cudaSuccess;
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP,
               se = launch_sort_pairs<unsigned>(m.sort_keys[0].p, m.sort_vals[0].p, m.sort_keys[1].p, m.sort_vals[1].p, n, key_bits, m.sort_scratch.p, true, nullptr, nullptr, &nl, t.st));
    CU_TRY(h, se);
    h->launches += nl > 0 ? nl - 1 : 0;
    const unsigned* skeys = m.sort_keys[passes & 1].p;
    const unsigned* order = m.sort_vals[passes & 1].p;
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_voxel_segments<<<blocks_for(n, 256), 256, 0, t.st>>>(skeys, n, invalid, m.segments.p));
    if (m.ndt) {
      KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_voxel_reduce<true><<<blocks_for(vmax, 4), 128, 0, t.st>>>(t.pts.p, nullptr, nullptr, order, m.segments.p, m.d_counters + 1, m.vox.p));
      cudaError_t ke = cudaSuccess;
      KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, ke = launch_regularize_voxels(m.vox.p, m.d_counters + 1, vmax, VGICP_REG_MIN_EIG, t.st));  // ndt_cuda.cu:129,140
      CU_TRY(h, ke);
    } else {
      KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_voxel_reduce<false><<<blocks_for(vmax, 4), 128, 0, t.st>>>(t.pts.p, t.covA.p, t.covB.p, order, m.segments.p, m.d_counters + 1, m.vox.p));
    }
  }
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(m.h_counters + 1, m.d_counters + 1, sizeof(int), cudaMemcpyDeviceToHost, t.st));
  CU_TRY(h, cudaEventRecord(m.ev_done, t.st));
  CU_TRY(h, cudaEventRecord(t.ready, t.st));
  m.v_pending = true;
  m.built = true;
  return VGICP_OK;
}

int voxelmap_num_voxels(vgicp_handle h, Cloud& t, VoxelMap& m, int* nv) {
  int rc = voxelmap_finish(h, t, m);
  if (rc) return rc;
  if (m.v_pending) {
    CU_TRY(h, cudaEventSynchronize(m.ev_done));
    m.num_voxels = m.h_counters[1];
    m.v_pending = false;
  }
  *nv = m.num_voxels;
  return VGICP_OK;
}

int build_voxelmap(vgicp_handle h) { return voxelmap_begin(h, h->target, h->map); }

// everything an evaluation on the main stream depends on: the finished voxel map and the last operations enqueued on the two
// cloud streams
int ndt_prepare(vgicp_handle h);

int sync_inputs(vgicp_handle h) {
  int rc = h->problem == 0 ? voxelmap_finish(h, h->target, h->map) : ndt_prepare(h);
  if (rc) return rc;
  if (h->target.st != h->stream && h->target.ready) CU_TRY(h, cudaStreamWaitEvent(h->stream, h->target.ready, 0));
  if (h->source.st != h->stream && h->source.ready) CU_TRY(h, cudaStreamWaitEvent(h->stream, h->source.ready, 0));
  return VGICP_OK;
}

// arguments + launch geometry of an evaluation kernel
struct LinLaunch {
  LinArgs a;
  int grid;
  int G;
};
LinLaunch make_lin_launch(vgicp_handle h) {
  Cloud& s = h->source;
  VoxelMap& m = h->problem != 0 ? h->ndt_t : h->map;
  LinLaunch L;
  LinArgs& a = L.a;
  a.ndt = h->problem != 0 ? 1 : 0;
  if (h->problem != 0) {  // NDT: target map = ndt_t; source = points + zero covariances (P2D) or source voxel Gaussians (D2D)
    a.pts = h->problem == 2 ? h->ndt_src_pts.p : s.pts.p;
    a.covA = h->ndt_src_covA.p; a.covB = h->ndt_src_covB.p; a.n = h->ndt_src_n;
  } else {
    const int sb = h->shard_end >= 0 ? h->shard_begin : 0;
    const int se = h->shard_end >= 0 ? (h->shard_end < s.n ? h->shard_end : s.n) : s.n;
    a.pts = s.pts.p + sb; a.covA = s.covA.p + sb; a.covB = s.covB.p + sb; a.n = se > sb ? se - sb : 0;
  }
  a.comm_ranks = h->comm_ranks; a.comm_rank = h->comm_rank; a.comm_seq = 0;
  for (int r = 0; r < kCommMaxRanks; r++) a.comm_peers[r] = h->comm_peers[r];
  a.buckets = m.buckets.p; a.mask = (unsigned)(m.num_buckets - 1); a.max_scan = m.max_scan; a.vox = m.vox.p;
  a.dense = m.dense;
  if (h->voxel_index_mode != 0) a.dense.cells = nullptr;
  a.offsets = h->d_offsets.p; a.n_off = (int)h->h_offsets.size(); a.res = m.res;
  a.Tlin = h->lin; a.Teval = h->lin;
  a.partials = h->partials.p; a.ticket = h->d_ticket; a.out = h->d_out;
  a.done_flag = nullptr; a.done_seq = 0;
  // lanes per source point in the lookup phase: split the neighbour cells of a point over G lanes while the cloud is too small to
  // fill the GPU with one thread per point (latency-bound regime); one lane per point once it is large
  const int n_off = a.n_off;
  const bool wide = a.n < 400000 && n_off > 1;
  // small clouds: split a point's cells over 3 (DIRECT27: whole z-columns), 4 (<= 7 offsets) or 8 lanes.  With the hits compacted
  // before the arithmetic the split costs no lane efficiency, so it is used under both execution hints
  const bool cols = h->offset_mode == 27;
  L.G = !wide ? 1 : (cols ? 3 : (n_off <= 7 ? 4 : 8));
  {
    const int force_g = h->force_lin_g;  // VGICP_LIN_G, read once in vgicp_create (A/B measurements)
    if (cols ? (force_g == 1 || force_g == 3) : (force_g == 1 || force_g == 4 || force_g == 8)) L.G = force_g;
  }
  const int tasks_per_block = (kLinThreads / 32) * ((32 / L.G) * L.G);
  long long tasks = (long long)(a.n > 0 ? a.n : 1) * L.G;
  long long grid = (tasks + tasks_per_block - 1) / tasks_per_block;
  L.grid = (int)(grid > kLinMaxBlocks ? kLinMaxBlocks : grid);
  return L;
}

// one evaluation: launches the fused lookup+derivative kernel; result lands in h->h_out after the stream sync
int launch_linearize(vgicp_handle h, const Pose& Teval, bool want_H, bool direct_to_host = false, bool spec = false) {
  LinLaunch L = make_lin_launch(h);
  LinArgs& a = L.a;
  a.Teval = Teval;
  a.comm_seq = h->comm_seq++;
  if (direct_to_host) {  // UVA: the mapped pinned pointers are valid on the device
    a.out = h->h_out;
    a.done_flag = h->h_flag;
    a.done_seq = ++h->eval_seq;
  }
  const int grid = L.grid, G = L.G;
#define LAUNCH_LIN_G(MODE, GG)                                                           \
  do {                                                                                   \
    if (spec) k_linearize_spec<MODE, GG><<<grid, kLinThreads, 0, h->stream>>>(a);        \
    else if (want_H) k_linearize<MODE, true, GG><<<grid, kLinThreads, 0, h->stream>>>(a); \
    else k_linearize<MODE, false, GG><<<grid, kLinThreads, 0, h->stream>>>(a);           \
  } while (0)
#define LAUNCH_LIN(MODE)                 \
  do {                                   \
    if (G == 8) LAUNCH_LIN_G(MODE, 8);   \
    else if (G == 4) LAUNCH_LIN_G(MODE, 4); \
    else LAUNCH_LIN_G(MODE, 1);          \
  } while (0)
  prof_begin(h, want_H ? VGICP_PROF_LINEARIZE : VGICP_PROF_ERROR, h->stream);
  // DIRECT1 on a large cloud with the direct-mapped index: the bandwidth-bound shape, streamed through shared memory by bulk copies
  const bool stream_kernel = h->offset_mode == 1 && a.dense.cells != nullptr && a.n >= 65536 && h->lin_stream != 0 && (reinterpret_cast<uintptr_t>(a.covB) & 15) == 0;
  if (stream_kernel) {
    const int tiles = (a.n + kLinStreamTile - 1) / kLinStreamTile;
    const int sgrid = tiles < kLinStreamMaxBlocks ? tiles : kLinStreamMaxBlocks;
    const size_t smem = sizeof(LinStreamSmem);
    if (spec) k_linearize_stream<2><<<sgrid, kLinThreads, smem, h->stream>>>(a);
    else if (want_H) k_linearize_stream<1><<<sgrid, kLinThreads, smem, h->stream>>>(a);
    else k_linearize_stream<0><<<sgrid, kLinThreads, smem, h->stream>>>(a);
  } else
  switch (h->offset_mode) {
    case 1: LAUNCH_LIN_G(1, 1); break;
    case 7: LAUNCH_LIN(7); break;
    case 27:
      if (G == 3) LAUNCH_LIN_G(27, 3);
      else LAUNCH_LIN_G(27, 1);
      break;
    default: LAUNCH_LIN(0); break;
  }
#undef LAUNCH_LIN_G
#undef LAUNCH_LIN
  prof_end(h, h->stream);
  h->launches++;
  CU_TRY(h, cudaGetLastError());
  return VGICP_OK;
}

// one link of the device-resident optimiser chain
int launch_lm_step(vgicp_handle h, const LinLaunch& L) {
  LinArgs a = L.a;
  a.comm_seq = h->comm_seq++;  // (links that find the chain finished return before the exchange, on every rank alike)
  const int grid = L.grid, G = L.G;
#define LAUNCH_LM_G(MODE, GG) k_lm_step<MODE, GG><<<grid, kLinThreads, 0, h->stream>>>(a, h->d_lm)
#define LAUNCH_LM(MODE)                 \
  do {                                  \
    if (G == 8) LAUNCH_LM_G(MODE, 8);   \
    else if (G == 4) LAUNCH_LM_G(MODE, 4); \
    else LAUNCH_LM_G(MODE, 1);          \
  } while (0)
  prof_begin(h, VGICP_PROF_LINEARIZE, h->stream);
  switch (h->offset_mode) {
    case 1: LAUNCH_LM_G(1, 1); break;
    case 7: LAUNCH_LM(7); break;
    case 27:
      if (G == 3) LAUNCH_LM_G(27, 3);
      else LAUNCH_LM_G(27, 1);
      break;
    default: LAUNCH_LM(0); break;
  }
#undef LAUNCH_LM_G
#undef LAUNCH_LM
  prof_end(h, h->stream);
  h->launches++;
  CU_TRY(h, cudaGetLastError());
  return VGICP_OK;
}

int check_ready_for_eval(vgicp_handle h, const char* who) {
  if (h->problem != 0) {
    if (!h->source.has_pts || !h->target.has_pts) return fail(h, VGICP_ERR_BAD_STATE, std::string(who) + ": NDT needs source and target clouds");
    if (!h->has_lin) return fail(h, VGICP_ERR_BAD_STATE, std::string(who) + ": update_correspondences has not been called");
    return VGICP_OK;
  }
  if (!h->source.has_pts || !h->source.has_cov) return fail(h, VGICP_ERR_BAD_STATE, std::string(who) + ": source points and covariances required");
  if (!h->map.built && !h->map.pending) return fail(h, VGICP_ERR_BAD_STATE, std::string(who) + ": target voxel map not built");
  if (!h->has_lin) return fail(h, VGICP_ERR_BAD_STATE, std::string(who) + ": update_correspondences has not been called");
  return VGICP_OK;
}

// builds what an NDT evaluation needs (idempotent): target map, and for D2D the source map + its Gaussians as a cloud
int ndt_prepare(vgicp_handle h) {
  if (h->ndt_ready) return VGICP_OK;
  Cloud& t = h->target;
  Cloud& s = h->source;
  if (!t.has_pts || !s.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "NDT: source and target clouds required");
  if (t.n <= 0 || s.n <= 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "NDT: empty cloud");
  // create_{source,target}_voxelmap (ndt_cuda.cu:123-141): a map that exists is kept (with the resolution it was created with), a
  // missing one is created with the current resolution; P2D never builds the source map
  int rc;
  if (!h->ndt_t.built && !h->ndt_t.pending) {
    h->ndt_t.created = true;
    h->ndt_t.res = (float)h->resolution;
    if ((rc = voxelmap_begin(h, t, h->ndt_t))) return rc;
  }
  if (h->problem == 2 && !h->ndt_s.built && !h->ndt_s.pending) {
    h->ndt_s.created = true;
    h->ndt_s.res = (float)h->resolution;
    if ((rc = voxelmap_begin(h, s, h->ndt_s))) return rc;
  }
  if ((rc = voxelmap_finish(h, t, h->ndt_t))) return rc;
  if (h->problem == 2) {
    int vs = 0;
    if ((rc = voxelmap_num_voxels(h, s, h->ndt_s, &vs))) return rc;
    CU_TRY(h, h->ndt_src_pts.reserve(vs > 0 ? vs : 1));
    CU_TRY(h, h->ndt_src_covA.reserve(vs > 0 ? vs : 1));
    CU_TRY(h, h->ndt_src_covB.reserve(vs > 0 ? vs : 1));
    if (vs > 0)
      KLAUNCH_ST(h, s.st, VGICP_PROF_VOXELMAP,
                 k_vox_to_cloud<<<blocks_for(vs, 256), 256, 0, s.st>>>(h->ndt_s.vox.p, h->ndt_s.d_counters + 1, h->ndt_src_pts.p, h->ndt_src_covA.p, h->ndt_src_covB.p));
    CU_TRY(h, cudaGetLastError());
    CU_TRY(h, cudaEventRecord(s.ready, s.st));
    h->ndt_src_n = vs;
  } else {
    CU_TRY(h, h->ndt_src_covA.reserve(s.n));
    CU_TRY(h, h->ndt_src_covB.reserve(s.n));
    CU_TRY(h, cudaMemsetAsync(h->ndt_src_covA.p, 0, sizeof(float4) * (size_t)s.n, s.st));
    CU_TRY(h, cudaMemsetAsync(h->ndt_src_covB.p, 0, sizeof(float2) * (size_t)s.n, s.st));
    CU_TRY(h, cudaEventRecord(s.ready, s.st));
    h->ndt_src_n = s.n;
  }
  h->ndt_ready = true;
  return VGICP_OK;
}

int evaluate(vgicp_handle h, const double* T, double* H36, double* b6, double* err) {
  const bool want_H = (H36 != nullptr && b6 != nullptr);  // compute_derivatives.cu:160
  const bool direct = h->exec_hint == 0;  // latency mode: result written to mapped host memory, host spins on a flag
  int rc = launch_linearize(h, to_pose(T), want_H, direct);
  if (rc) return rc;
  if (direct) {
    const unsigned long long want = h->eval_seq;
    volatile unsigned long long* flag = h->h_flag;
    long spins = 0;
    while (*flag != want) {
      __builtin_ia32_pause();
      if (++spins > 2000000L) {  // ~a few ms without an answer: fall back to a blocking wait (also surfaces launch errors)
        CU_TRY(h, cudaStreamSynchronize(h->stream));
        if (*flag != want) return fail(h, VGICP_ERR_CUDA, "evaluate: kernel finished without publishing its result");
        break;
      }
    }
    __sync_synchronize();
  } else {
    CU_TRY(h, cudaMemcpyAsync(h->h_out, h->d_out, sizeof(double) * (h->comm_ranks > 1 ? kLinOutCommError + 1 : (want_H ? 43 : 1)), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(h, cudaStreamSynchronize(h->stream));
  }
  if (h->comm_ranks > 1 && h->h_out[kLinOutCommError] != 0.0) return fail(h, VGICP_ERR_COMM, "evaluate: a peer rank did not deliver its sums in time (vgicp_comm_error)");
  if (err) *err = h->h_out[0];
  if (want_H) {
    memcpy(H36, h->h_out + 1, 36 * sizeof(double));
    memcpy(b6, h->h_out + 37, 6 * sizeof(double));
  }
  return VGICP_OK;
}

// trial-pose evaluation for the LM loop: error at T over the current correspondences (*err_old) plus the linearisation at T itself
// (k_linearize_spec); h->lin stays the current linearisation point
int evaluate_spec(vgicp_handle h, const double* T, double* err_old, double* H36, double* b6, double* err_new) {
  const bool direct = h->exec_hint == 0;
  int rc = launch_linearize(h, to_pose(T), true, direct, true);
  if (rc) return rc;
  if (direct) {
    const unsigned long long want = h->eval_seq;
    volatile unsigned long long* flag = h->h_flag;
    long spins = 0;
    while (*flag != want) {
      __builtin_ia32_pause();
      if (++spins > 2000000L) {
        CU_TRY(h, cudaStreamSynchronize(h->stream));
        if (*flag != want) return fail(h, VGICP_ERR_CUDA, "evaluate: kernel finished without publishing its result");
        break;
      }
    }
    __sync_synchronize();
  } else {
    CU_TRY(h, cudaMemcpyAsync(h->h_out, h->d_out, sizeof(double) * (kLinOutCommError + 1), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(h, cudaStreamSynchronize(h->stream));
  }
  if (h->comm_ranks > 1 && h->h_out[kLinOutCommError] != 0.0) return fail(h, VGICP_ERR_COMM, "evaluate: a peer rank did not deliver its sums in time (vgicp_comm_error)");
  *err_new = h->h_out[0];
  memcpy(H36, h->h_out + 1, 36 * sizeof(double));
  memcpy(b6, h->h_out + 37, 6 * sizeof(double));
  *err_old = h->h_out[43];
  return VGICP_OK;
}

}  // namespace

// =====================================================================================================================
extern "C" {

const char* vgicp_version(void) { return "vgicp_b200 0.1 (sm_90a)"; }

int vgicp_create(int device, vgicp_handle* out) {
  if (!out) return VGICP_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return VGICP_ERR_NO_DEVICE;
  if (device < 0 || device >= ndev) return VGICP_ERR_INVALID_ARGUMENT;
  vgicp_context* h = new (std::nothrow) vgicp_context();
  if (!h) return VGICP_ERR_CUDA;
  h->device = device;
  { const char* e = getenv("VGICP_LIN_G"); h->force_lin_g = e ? atoi(e) : 0; }
  { const char* e = getenv("VGICP_LIN_STREAM"); h->lin_stream = e ? atoi(e) : 1; }
  DeviceGuard g(device);
  // the kernel image is sm_90a only: fail loudly on anything else instead of falling back
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, k_linearize<1, true, 1>) != cudaSuccess) {
    cudaGetLastError();
    delete h;
    return VGICP_ERR_NO_DEVICE;
  }
  bool ok = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&h->stream_b, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&h->ev_copy, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&h->target.ready, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&h->source.ready, cudaEventDisableTiming) == cudaSuccess;
  h->target.st = h->stream;    // the target (and its voxel map) is built on the main stream, where the evaluations run
  h->source.st = h->stream_b;  // the source's stage 1 overlaps with it
  ok = ok && cudaMalloc(&h->d_ticket, sizeof(unsigned int)) == cudaSuccess;
  for (VoxelMap* vm : {&h->map, &h->ndt_t, &h->ndt_s}) {
    ok = ok && cudaMalloc(&vm->d_counters, 16 * sizeof(int)) == cudaSuccess;
    ok = ok && cudaMallocHost(&vm->h_counters, 16 * sizeof(int)) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&vm->ev_attempt, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&vm->ev_done, cudaEventDisableTiming) == cudaSuccess;
  }
  h->ndt_t.ndt = h->ndt_s.ndt = 1;
  ok = ok && cudaMalloc(&h->d_out, 64 * sizeof(double)) == cudaSuccess;
  ok = ok && cudaHostAlloc(&h->h_out, 64 * sizeof(double), cudaHostAllocMapped) == cudaSuccess;
  ok = ok && cudaHostAlloc(&h->h_flag, 64, cudaHostAllocMapped) == cudaSuccess;
  if (ok) *h->h_flag = 0;
  ok = ok && cudaMalloc(&h->d_lm, sizeof(LmState)) == cudaSuccess;
  ok = ok && cudaMallocHost(&h->h_lm, sizeof(LmState)) == cudaSuccess;
  ok = ok && h->partials.reserve((size_t)kLinStreamMaxBlocks * kLinStride) == cudaSuccess;
  ok = ok && cudaMemsetAsync(h->d_ticket, 0, sizeof(unsigned int), h->stream) == cudaSuccess;
  ok = ok && cudaStreamSynchronize(h->stream) == cudaSuccess;
  if (!ok) {
    vgicp_destroy(h);
    return VGICP_ERR_CUDA;
  }
  h->h_offsets.assign(1, make_int4(0, 0, 0, 0));  // fast_vgicp_cuda.cu:28-29
  h->offset_mode = 1;
  *out = h;
  return VGICP_OK;
}

int vgicp_destroy(vgicp_handle h) {
  if (!h) return VGICP_OK;
  DeviceGuard g(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->stream_b) cudaStreamSynchronize(h->stream_b);
  h->source.release();
  h->target.release();
  h->d_offsets.release();
  h->staging.release();
  if (h->comm_ranks > 1) vgicp_comm_shutdown(h);
  if (h->comm_box) cudaFree(h->comm_box);
  if (h->arena) cudaFree(h->arena);
  h->partials.release();
  h->corr_ids.release();
  if (h->d_ticket) cudaFree(h->d_ticket);
  for (VoxelMap* vm : {&h->map, &h->ndt_t, &h->ndt_s}) {
    if (vm->d_counters) cudaFree(vm->d_counters);
    if (vm->h_counters) cudaFreeHost(vm->h_counters);
    if (vm->ev_attempt) cudaEventDestroy(vm->ev_attempt);
    if (vm->ev_done) cudaEventDestroy(vm->ev_done);
    vm->release();
  }
  h->ndt_src_pts.release(); h->ndt_src_covA.release(); h->ndt_src_covB.release();
  if (h->d_out) cudaFree(h->d_out);
  if (h->h_out) cudaFreeHost(h->h_out);
  if (h->h_flag) cudaFreeHost(h->h_flag);
  if (h->d_lm) cudaFree(h->d_lm);
  if (h->h_lm) cudaFreeHost(h->h_lm);
  for (auto& r : h->prof_pending) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (auto e : h->prof_pool) cudaEventDestroy(e);
  for (cudaEvent_t e : {h->ev_copy, h->target.ready, h->source.ready})
    if (e) cudaEventDestroy(e);
  if (h->stream_b) cudaStreamDestroy(h->stream_b);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return VGICP_OK;
}

const char* vgicp_last_error(vgicp_handle h) { return h ? h->err.c_str() : "null handle"; }

int vgicp_set_resolution(vgicp_handle h, double resolution) {
  CHECK_HANDLE(h);
  if (!(resolution > 0.0)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_resolution: resolution must be positive");
  h->resolution = resolution;
  return VGICP_OK;
}

int vgicp_set_kernel_params(vgicp_handle h, double kernel_width, double kernel_max_dist) {
  CHECK_HANDLE(h);
  h->kernel_width = kernel_width;
  h->kernel_max_dist = kernel_max_dist;
  return VGICP_OK;
}

int vgicp_set_neighbor_search_method(vgicp_handle h, int method, double radius) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  std::vector<int4> off;
  int mode = 0;
  switch (method) {
    case VGICP_DIRECT1:
      off.push_back(make_int4(0, 0, 0, 0));
      mode = 1;
      break;
    case VGICP_DIRECT7: {  // order of fast_vgicp_cuda.cu:57-63
      const int o[7][3] = {{0, 0, 0}, {1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
      for (auto& v : o) off.push_back(make_int4(v[0], v[1], v[2], 0));
      mode = 7;
    } break;
    case VGICP_DIRECT27:  // :68-74, i-major
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
          for (int k = 0; k < 3; k++) off.push_back(make_int4(i - 1, j - 1, k - 1, 0));
      mode = 27;
      break;
    case VGICP_DIRECT_RADIUS: {  // :79-88
      if (!(radius >= 0.0) || radius > 64.0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_neighbor_search_method: radius out of range");
      int range = (int)ceil(radius);
      for (int i = -range; i <= range; i++)
        for (int j = -range; j <= range; j++)
          for (int k = -range; k <= range; k++) {
            double nrm = sqrt((double)i * i + (double)j * j + (double)k * k);
            if (nrm <= radius + 1e-3) off.push_back(make_int4(i, j, k, 0));
          }
      mode = 0;
    } break;
    default:  // the reference abort()s here (fast_vgicp_cuda.cu:46-48)
      return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_neighbor_search_method: unknown method");
  }
  CU_TRY(h, h->d_offsets.reserve(off.size()));
  if (!off.empty()) {
    CU_TRY(h, cudaMemcpyAsync(h->d_offsets.p, off.data(), off.size() * sizeof(int4), cudaMemcpyHostToDevice, h->stream));
    CU_TRY(h, cudaStreamSynchronize(h->stream));
  }
  h->h_offsets.swap(off);
  h->offset_mode = mode;
  return VGICP_OK;
}

int vgicp_set_source_cloud(vgicp_handle h, const float* xyz, size_t n, size_t stride_bytes) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  h->source.k = 0;  // the reference keeps stale neighbours/covariances; every caller recomputes them right after
  h->source.has_cov = false;
  return set_cloud(h, h->source, xyz, n, stride_bytes);
}

int vgicp_set_target_cloud(vgicp_handle h, const float* xyz, size_t n, size_t stride_bytes) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  h->target.k = 0;
  h->target.has_cov = false;
  h->map.built = false;
  h->map.pending = false;
  return set_cloud(h, h->target, xyz, n, stride_bytes);
}

int vgicp_swap_source_and_target(vgicp_handle h) {  // fast_vgicp_cuda.cu:97-107
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  // whole Cloud records are swapped, streams and `ready` events included (sync_inputs compares each cloud's stream with the main
  // stream, so it does not matter which one ends up where); everything in flight (incl. a pending map build that reads the old
  // target) must land first
  if (h->map.pending) { int rc0 = voxelmap_finish(h, h->target, h->map); if (rc0) return rc0; }
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  CU_TRY(h, cudaStreamSynchronize(h->stream_b));
  std::swap(h->source, h->target);
  h->map.built = false;
  h->map.pending = false;
  // NDT: the reference swaps its two maps (ndt_cuda.cu:90-93); a map that does not exist (P2D never builds the source's) is built by
  // the next create_voxelmaps.  Pending builds were enqueued on the old streams: both streams are idle here.
  for (VoxelMap* vm : {&h->ndt_t, &h->ndt_s})
    if (vm->pending) { vm->pending = false; vm->built = false; }
  std::swap(h->ndt_t, h->ndt_s);
  h->ndt_ready = false;
  if (h->problem != 0) return VGICP_OK;
  if (!h->target.has_pts || !h->target.has_cov) return VGICP_OK;
  return build_voxelmap(h);
}

int vgicp_set_source_neighbors(vgicp_handle h, int k, const int* indices, size_t n_times_k) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return set_neighbors(h, h->source, k, indices, n_times_k);
}
int vgicp_set_target_neighbors(vgicp_handle h, int k, const int* indices, size_t n_times_k) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return set_neighbors(h, h->target, k, indices, n_times_k);
}
int vgicp_find_source_neighbors(vgicp_handle h, int k) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return find_neighbors(h, h->source, k);
}
int vgicp_find_target_neighbors(vgicp_handle h, int k) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return find_neighbors(h, h->target, k);
}
int vgicp_calculate_source_covariances(vgicp_handle h, int method) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return calc_covariances(h, h->source, method);
}
int vgicp_calculate_target_covariances(vgicp_handle h, int method) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return calc_covariances(h, h->target, method);
}
int vgicp_calculate_source_covariances_rbf(vgicp_handle h, int method) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return calc_covariances_rbf(h, h->source, method);
}
int vgicp_calculate_target_covariances_rbf(vgicp_handle h, int method) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return calc_covariances_rbf(h, h->target, method);
}
int vgicp_set_source_covariances(vgicp_handle h, const float* in9, size_t n) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return set_covariances(h, h->source, in9, n);
}
int vgicp_set_target_covariances(vgicp_handle h, const float* in9, size_t n) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  h->map.built = false;  // the voxel Gaussians average the target covariances: the map must be rebuilt (create_target_voxelmap)
  h->map.pending = false;
  return set_covariances(h, h->target, in9, n);
}
int vgicp_get_source_covariances(vgicp_handle h, float* out9, size_t cap) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return get_covariances(h, h->source, out9, cap);
}
int vgicp_get_target_covariances(vgicp_handle h, float* out9, size_t cap) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return get_covariances(h, h->target, out9, cap);
}
int vgicp_get_source_neighbors(vgicp_handle h, int* out, size_t cap, int* k_out) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return get_neighbors(h, h->source, out, cap, k_out);
}
int vgicp_get_target_neighbors(vgicp_handle h, int* out, size_t cap, int* k_out) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return get_neighbors(h, h->target, out, cap, k_out);
}
int vgicp_get_num_source_points(vgicp_handle h, size_t* n) {
  CHECK_HANDLE(h);
  if (!n) return VGICP_ERR_INVALID_ARGUMENT;
  *n = h->source.has_pts ? (size_t)h->source.n : 0;
  return VGICP_OK;
}
int vgicp_get_num_target_points(vgicp_handle h, size_t* n) {
  CHECK_HANDLE(h);
  if (!n) return VGICP_ERR_INVALID_ARGUMENT;
  *n = h->target.has_pts ? (size_t)h->target.n : 0;
  return VGICP_OK;
}

int vgicp_create_target_voxelmap(vgicp_handle h) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return build_voxelmap(h);
}

int vgicp_get_num_voxels(vgicp_handle h, int* nv) {
  CHECK_HANDLE(h);
  if (!nv) return VGICP_ERR_INVALID_ARGUMENT;
  DeviceGuard g(h->device);
  if (h->problem != 0) { int rc = ndt_prepare(h); if (rc) return rc; return voxelmap_num_voxels(h, h->target, h->ndt_t, nv); }
  return voxelmap_num_voxels(h, h->target, h->map, nv);
}
int vgicp_get_num_buckets(vgicp_handle h, int* nb) {
  CHECK_HANDLE(h);
  if (!nb) return VGICP_ERR_INVALID_ARGUMENT;
  DeviceGuard g(h->device);
  if (h->problem != 0) { int rc = ndt_prepare(h); if (rc) return rc; *nb = h->ndt_t.num_buckets; return VGICP_OK; }
  { int rc = voxelmap_finish(h, h->target, h->map); if (rc) return rc; }
  *nb = h->map.num_buckets;
  return VGICP_OK;
}

static int fetch_voxels(vgicp_handle h, std::vector<VoxelRec>& v) {
  int nv = 0;
  VoxelMap& vm = h->problem != 0 ? h->ndt_t : h->map;
  int rc = h->problem != 0 ? ndt_prepare(h) : VGICP_OK;
  if (rc) return rc;
  rc = voxelmap_num_voxels(h, h->target, vm, &nv);
  if (rc) return rc;
  v.resize(nv);
  if (!v.empty()) {
    CU_TRY(h, cudaMemcpyAsync(v.data(), vm.vox.p, sizeof(VoxelRec) * v.size(), cudaMemcpyDeviceToHost, h->target.st));
    CU_TRY(h, cudaStreamSynchronize(h->target.st));
  }
  return VGICP_OK;
}

int vgicp_get_voxel_num_points(vgicp_handle h, int* out, size_t cap) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  std::vector<VoxelRec> v;
  int rc = fetch_voxels(h, v);
  if (rc) return rc;
  if (!out || cap < v.size()) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_voxel_num_points: buffer too small");
  for (size_t i = 0; i < v.size(); i++) memcpy(&out[i], &v[i].mean_n.w, sizeof(int));
  return VGICP_OK;
}
int vgicp_get_voxel_means(vgicp_handle h, float* out3, size_t cap) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  std::vector<VoxelRec> v;
  int rc = fetch_voxels(h, v);
  if (rc) return rc;
  if (!out3 || cap < v.size()) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_voxel_means: buffer too small");
  for (size_t i = 0; i < v.size(); i++) {
    out3[3 * i] = v[i].mean_n.x; out3[3 * i + 1] = v[i].mean_n.y; out3[3 * i + 2] = v[i].mean_n.z;
  }
  return VGICP_OK;
}
int vgicp_get_voxel_covs(vgicp_handle h, float* out9, size_t cap) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  std::vector<VoxelRec> v;
  int rc = fetch_voxels(h, v);
  if (rc) return rc;
  if (!out9 || cap < v.size()) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_voxel_covs: buffer too small");
  for (size_t i = 0; i < v.size(); i++) {
    float* o = out9 + 9 * i;
    const float4 a = v[i].c0, b = v[i].c1;
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.y; o[4] = a.w; o[5] = b.x; o[6] = a.z; o[7] = b.x; o[8] = b.y;
  }
  return VGICP_OK;
}
int vgicp_get_voxel_buckets(vgicp_handle h, int* coords3, int* ids, size_t cap) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  VoxelMap& vm = h->problem != 0 ? h->ndt_t : h->map;
  { int rc = h->problem != 0 ? ndt_prepare(h) : voxelmap_finish(h, h->target, h->map); if (rc) return rc; }
  size_t B = (size_t)vm.num_buckets;
  if (cap < B || !coords3 || !ids) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_voxel_buckets: buffer too small");
  std::vector<int4> b(B);
  CU_TRY(h, cudaMemcpyAsync(b.data(), vm.buckets.p, sizeof(int4) * B, cudaMemcpyDeviceToHost, h->target.st));
  CU_TRY(h, cudaStreamSynchronize(h->target.st));
  for (size_t i = 0; i < B; i++) {
    coords3[3 * i] = b[i].x; coords3[3 * i + 1] = b[i].y; coords3[3 * i + 2] = b[i].z;
    ids[i] = b[i].w;
  }
  return VGICP_OK;
}

int vgicp_update_correspondences(vgicp_handle h, const double T[16]) {  // fast_vgicp_cuda.cu:265-274
  CHECK_HANDLE(h);
  if (!T) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "update_correspondences: null pose");
  if (!h->source.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "update_correspondences: source cloud not set");
  if (h->problem == 0 && !h->map.built && !h->map.pending) return fail(h, VGICP_ERR_BAD_STATE, "update_correspondences: target voxel map not built");
  if (h->problem != 0 && !h->target.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "update_correspondences: target cloud not set");
  h->lin = to_pose(T);  // linearized_x = trans.cast<float>()
  h->has_lin = true;
  // the lookup itself is fused into the evaluation kernel; the explicit list is only built by the getter
  return VGICP_OK;
}

int vgicp_get_voxel_correspondences(vgicp_handle h, int* pairs, size_t cap, size_t* n_pairs) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!h->source.has_pts || (h->problem == 0 && !h->map.built && !h->map.pending) || !h->has_lin)
    return fail(h, VGICP_ERR_BAD_STATE, "get_voxel_correspondences: update_correspondences has not been called");
  { int rc = sync_inputs(h); if (rc) return rc; }
  const LinLaunch LL = make_lin_launch(h);  // same source array / map as an evaluation (VGICP points, NDT points or voxel means)
  const int n = LL.a.n;
  const int n_off = (int)h->h_offsets.size();
  size_t total = (size_t)n * n_off;
  std::vector<int> ids(total);
  if (total) {
    CU_TRY(h, h->corr_ids.reserve(total));
    KLAUNCH(h, VGICP_PROF_OTHER,
            k_correspondence_ids<<<blocks_for(n, 128), 128, 0, h->stream>>>(LL.a.pts, n, LL.a.buckets, LL.a.mask, LL.a.max_scan, h->d_offsets.p, n_off, LL.a.res, h->lin, h->corr_ids.p));
    CU_TRY(h, cudaGetLastError());
    CU_TRY(h, cudaMemcpyAsync(ids.data(), h->corr_ids.p, total * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(h, cudaStreamSynchronize(h->stream));
  }
  size_t cnt = 0;
  for (int o = 0; o < n_off; o++)
    for (int i = 0; i < n; i++) {
      int id = ids[(size_t)o * n + i];
      if (id < 0) continue;  // remove_if(invalid_correspondence_kernel), find_voxel_correspondences.cu:109-110
      if (pairs && cnt < cap) { pairs[2 * cnt] = i; pairs[2 * cnt + 1] = id; }
      cnt++;
    }
  if (n_pairs) *n_pairs = cnt;
  if (pairs && cnt > cap) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_voxel_correspondences: buffer too small");
  return VGICP_OK;
}

int vgicp_compute_error(vgicp_handle h, const double T[16], double* H36, double* b6, double* err) {  // fast_vgicp_cuda.cu:276-284
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!T) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "compute_error: null pose");
  int rc = check_ready_for_eval(h, "compute_error");
  if (rc) return rc;
  if ((rc = sync_inputs(h))) return rc;
  return evaluate(h, T, H36, b6, err);
}

void vgicp_lsq_default_params(vgicp_lsq_params* p) {  // lsq_registration_impl.hpp:9-22
  if (!p) return;
  p->max_iterations = 64;
  p->rotation_epsilon = 2e-3;
  p->transformation_epsilon = 5e-4;
  p->use_gauss_newton = 0;
  p->lm_max_iterations = 10;
  p->lm_init_lambda_factor = 1e-9;
}

// LsqRegistration::computeTransformation (lsq_registration_impl.hpp:53-79) with step_gn (:106-120) / step_lm (:123-168);
// linearize = update_correspondences + compute_error (fast_vgicp_cuda_impl.hpp:170-173).
int vgicp_align(vgicp_handle h, const double guess[16], const vgicp_lsq_params* params, vgicp_align_result* res) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!guess || !res) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align: null argument");
  vgicp_lsq_params P;
  if (params) P = *params; else vgicp_lsq_default_params(&P);
  if (h->problem == 0) {
    if (!h->source.has_pts || !h->source.has_cov) return fail(h, VGICP_ERR_BAD_STATE, "align: source points and covariances required");
    if (!h->map.built && !h->map.pending) return fail(h, VGICP_ERR_BAD_STATE, "align: target voxel map not built");
  } else if (!h->source.has_pts || !h->target.has_pts) {
    return fail(h, VGICP_ERR_BAD_STATE, "align: NDT needs source and target clouds");
  }
  { int rc = sync_inputs(h); if (rc) return rc; }

  if (h->align_mode == 0) {
    // device-resident loop: initialise the state block, enqueue evaluation links, read the state back once per chunk
    LmState* st = h->h_lm;
    memset(st, 0, sizeof(LmState));
    memcpy(st->x0, guess, sizeof(st->x0));
    for (int i = 0; i < 6; i++) st->final_H[i * 7] = 1.0;  // final_hessian_.setIdentity()
    st->lambda = -1.0;
    st->nu = 2.0;
    st->rotation_epsilon = P.rotation_epsilon;
    st->transformation_epsilon = P.transformation_epsilon;
    st->lm_init_lambda_factor = P.lm_init_lambda_factor;
    st->max_iterations = P.max_iterations;
    st->lm_max_iterations = P.lm_max_iterations;
    st->use_gauss_newton = P.use_gauss_newton;
    st->phase = P.max_iterations > 0 ? kLmLinearize : kLmDone;
    st->lin_pose = to_pose(guess);
    st->eval_pose = st->lin_pose;
    CU_TRY(h, cudaMemcpyAsync(h->d_lm, st, sizeof(LmState), cudaMemcpyHostToDevice, h->stream));
    const LinLaunch L = make_lin_launch(h);
    const int chunk = 12;  // a typical registration needs ~10 evaluations; finished chains return immediately
    for (int guard = 0; guard < 4096; guard++) {
      for (int c = 0; c < chunk; c++) {
        int rc = launch_lm_step(h, L);
        if (rc) return rc;
      }
      CU_TRY(h, cudaMemcpyAsync(st, h->d_lm, sizeof(LmState), cudaMemcpyDeviceToHost, h->stream));
      CU_TRY(h, cudaStreamSynchronize(h->stream));
      if (st->phase == kLmDone) break;
    }
    memset(res, 0, sizeof(*res));
    memcpy(res->T, st->x0, sizeof(res->T));
    memcpy(res->H, st->final_H, sizeof(res->H));
    res->nr_iterations = st->nr_iterations;
    res->converged = st->converged;
    res->n_linearize = st->n_linearize;
    res->n_compute_error = st->n_error;
    res->lm_failed = st->lm_failed;
    h->lin = st->lin_pose;  // linearized_x of the last linearisation
    h->has_lin = true;
    return VGICP_OK;
  }

  Iso3d x0;
  memcpy(x0.m, guess, sizeof(x0.m));
  double lambda = -1.0;
  bool converged = false;
  memset(res, 0, sizeof(*res));
  for (int i = 0; i < 6; i++) res->H[i * 7] = 1.0;  // final_hessian_.setIdentity()
  // speculative evaluation: every LM trial also linearises at the trial pose, so an accepted step needs no launch of its own
  const bool speculate = h->speculate != 0 && !P.use_gauss_newton;
  bool have_next = false;
  double Hn[36], bn[6], yn = 0.0;
  for (int it = 0; it < P.max_iterations && !converged; it++) {
    res->nr_iterations = it;
    double H[36], b[6], nb[6], d[6], y0 = 0.0;
    h->lin = to_pose(x0.m);
    h->has_lin = true;
    int rc = VGICP_OK;
    if (have_next) {  // linearised at this very pose by the trial evaluation that accepted it
      memcpy(H, Hn, sizeof(H)); memcpy(b, bn, sizeof(b)); y0 = yn;
      have_next = false;
    } else {
      rc = evaluate(h, x0.m, H, b, &y0);
    }
    if (rc) return rc;
    res->n_linearize++;
    for (int j = 0; j < 6; j++) nb[j] = -b[j];
    Iso3d delta = iso_identity();
    bool ok = false;
    if (P.use_gauss_newton) {
      ldlt_solve6(H, nb, d);
      delta = se3_exp(d);
      x0 = iso_mul(delta, x0);
      memcpy(res->H, H, sizeof(H));
      ok = true;
    } else {
      if (lambda < 0.0) {
        double mx = 0.0;
        for (int j = 0; j < 6; j++) mx = fmax(mx, fabs(H[j * 7]));
        lambda = P.lm_init_lambda_factor * mx;
      }
      double nu = 2.0;
      for (int j = 0; j < P.lm_max_iterations; j++) {
        double Hl[36];
        memcpy(Hl, H, sizeof(H));
        for (int q = 0; q < 6; q++) Hl[q * 7] += lambda;
        ldlt_solve6(Hl, nb, d);
        delta = se3_exp(d);
        Iso3d xi = iso_mul(delta, x0);
        double yi = 0.0;
        rc = speculate ? evaluate_spec(h, xi.m, &yi, Hn, bn, &yn) : evaluate(h, xi.m, nullptr, nullptr, &yi);
        if (rc) return rc;
        res->n_compute_error++;
        double den = 0.0;
        for (int q = 0; q < 6; q++) den += d[q] * (lambda * d[q] - b[q]);
        double rho = (y0 - yi) / den;
        if (rho < 0) {
          if (is_converged(delta, P.rotation_epsilon, P.transformation_epsilon)) { ok = true; break; }
          lambda = nu * lambda;
          nu = 2 * nu;
          continue;
        }
        x0 = xi;
        have_next = speculate;
        double f = 1.0 - pow(2.0 * rho - 1.0, 3);
        lambda = lambda * fmax(1.0 / 3.0, f);
        memcpy(res->H, H, sizeof(H));
        ok = true;
        break;
      }
    }
    if (!ok) { res->lm_failed = 1; break; }  // "lm not converged!!"
    converged = is_converged(delta, P.rotation_epsilon, P.transformation_epsilon);
  }
  memcpy(res->T, x0.m, sizeof(x0.m));
  res->converged = converged ? 1 : 0;
  return VGICP_OK;
}

// clear + setInputTarget + setInputSource + align in one call (the body of the reference's benchmark loop, src/align.cpp:72-81)
int vgicp_register(vgicp_handle h, const float* target_xyz, size_t n_target, const float* source_xyz, size_t n_source, size_t stride_bytes, int on_device, int k,
                   int regularization_method, const double guess[16], const vgicp_lsq_params* params, vgicp_align_result* result) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  int rc;
  h->target.k = 0; h->target.has_cov = false; h->map.built = false; h->map.pending = false;
  if ((rc = set_cloud(h, h->target, target_xyz, n_target, stride_bytes, on_device != 0))) return rc;
  if ((rc = find_neighbors(h, h->target, k))) return rc;
  // NORMALIZED_MIN_EIG: raw covariances kept and VGICP_ERR_UNSUPPORTED reported (the reference prints a message and carries on,
  // covariance_regularization.cu:121-123); the class wrappers tolerate that code, so does the one-call registration
  if ((rc = calc_covariances(h, h->target, regularization_method)) && rc != VGICP_ERR_UNSUPPORTED) return rc;
  if ((rc = build_voxelmap(h))) return rc;
  h->source.k = 0; h->source.has_cov = false;
  if ((rc = set_cloud(h, h->source, source_xyz, n_source, stride_bytes, on_device != 0))) return rc;
  if ((rc = find_neighbors(h, h->source, k))) return rc;
  if ((rc = calc_covariances(h, h->source, regularization_method)) && rc != VGICP_ERR_UNSUPPORTED) return rc;
  double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  return vgicp_align(h, guess ? guess : I, params, result);
}

int vgicp_transform_source(vgicp_handle h, const double T[16], float* out_xyz, size_t cap, size_t stride) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!T || !out_xyz) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "transform_source: null argument");
  if (!h->source.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "transform_source: source cloud not set");
  const int n = h->source.n;
  if (cap < (size_t)n || stride < 12 || stride % 4) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "transform_source: bad capacity/stride");
  if (n == 0) return VGICP_OK;
  if (h->source.st != h->stream) CU_TRY(h, cudaStreamWaitEvent(h->stream, h->source.ready, 0));
  CU_TRY(h, h->staging.reserve((size_t)n * stride));
  // keep the non-xyz bytes of the caller's records untouched: copy in, overwrite xyz, copy out
  if (stride > 12) CU_TRY(h, cudaMemcpyAsync(h->staging.p, out_xyz, (size_t)n * stride, cudaMemcpyHostToDevice, h->stream));
  KLAUNCH(h, VGICP_PROF_OTHER, k_transform_points<<<blocks_for(n, 256), 256, 0, h->stream>>>(h->source.pts.p, n, to_pose(T), h->staging.p, stride));
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(out_xyz, h->staging.p, (size_t)n * stride, cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  return VGICP_OK;
}

int vgicp_set_source_cloud_device(vgicp_handle h, const float* d_xyz, size_t n, size_t stride_bytes) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  h->source.k = 0;
  h->source.has_cov = false;
  return set_cloud(h, h->source, d_xyz, n, stride_bytes, true);
}

int vgicp_set_target_cloud_device(vgicp_handle h, const float* d_xyz, size_t n, size_t stride_bytes) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  h->target.k = 0;
  h->target.has_cov = false;
  h->map.built = false;
  h->map.pending = false;
  return set_cloud(h, h->target, d_xyz, n, stride_bytes, true);
}

// ---- multi-GPU: source sharding with an in-kernel exchange of the linear system over NVLink peer memory ----
int vgicp_comm_export(vgicp_handle h, unsigned char* handle64) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!handle64) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "comm_export: null buffer");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  if (!h->comm_box) {
    CU_TRY(h, cudaMalloc(&h->comm_box, sizeof(CommMailbox)));
    CU_TRY(h, cudaMemset(h->comm_box, 0, sizeof(CommMailbox)));
  }
  cudaIpcMemHandle_t ipc;
  CU_TRY(h, cudaIpcGetMemHandle(&ipc, h->comm_box));
  memcpy(handle64, &ipc, 64);
  return VGICP_OK;
}

int vgicp_comm_init(vgicp_handle h, int rank, int nranks, const unsigned char* all_handles) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (nranks < 1 || nranks > kCommMaxRanks || rank < 0 || rank >= nranks || !all_handles) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "comm_init: need 1 <= nranks <= 8 and all handles");
  if (!h->comm_box) return fail(h, VGICP_ERR_BAD_STATE, "comm_init: call vgicp_comm_export first");
  for (int r = 0; r < nranks; r++) {
    if (r == rank) { h->comm_peers[r] = h->comm_box; continue; }
    cudaIpcMemHandle_t ipc;
    memcpy(&ipc, all_handles + (size_t)r * 64, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail(h, VGICP_ERR_COMM, std::string("comm_init: cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
    h->comm_peers[r] = reinterpret_cast<CommMailbox*>(p);
  }
  h->comm_rank = rank;
  h->comm_ranks = nranks;
  h->comm_seq = 0;
  // the mailbox outlives vgicp_comm_shutdown: flags left by a previous session could equal the first tags of this one.  Clear it
  // here; the caller puts a host barrier between vgicp_comm_init on all ranks and the first evaluation (see the header), so no
  // peer writes into it before the clear has landed.
  CU_TRY(h, cudaMemsetAsync(h->comm_box, 0, sizeof(CommMailbox), h->stream));
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  return VGICP_OK;
}

// ---- stage-1 sharding: the exchange arena ----
int vgicp_comm_export_arena(vgicp_handle h, size_t max_points, unsigned char* handle64) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!handle64 || max_points == 0 || max_points > ((size_t)1 << 28)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "comm_export_arena: bad argument");
  max_points = (max_points + 15) & ~(size_t)15;  // the two clouds' float4 / float2 arrays follow each other: keep every array 16-byte aligned
  if (h->arena && h->arena_points != max_points) return fail(h, VGICP_ERR_BAD_STATE, "comm_export_arena: arena already allocated with another capacity");
  if (!h->arena) {
    CU_TRY(h, cudaStreamSynchronize(h->stream));
    CU_TRY(h, cudaStreamSynchronize(h->stream_b));
    const size_t bytes = kCommArenaHeaderBytes + 2 * max_points * 24 + 64;  // (+ padding: bulk copies read covB in 16-byte units)
    CU_TRY(h, cudaMalloc(&h->arena, bytes));
    CU_TRY(h, cudaMemset(h->arena, 0, bytes));
    h->arena_points = max_points;
    // the covariance arrays of both clouds now live in the arena (previous covariances are dropped)
    Cloud* cl[2] = {&h->target, &h->source};
    for (int j = 0; j < 2; j++) {
      unsigned char* base = h->arena + kCommArenaHeaderBytes + (size_t)j * max_points * 24;
      cl[j]->covA.attach(reinterpret_cast<float4*>(base), max_points);
      cl[j]->covB.attach(reinterpret_cast<float2*>(base + max_points * 16), max_points);
      cl[j]->arena_slot = j;
      cl[j]->arena_seq = 0;
      cl[j]->has_cov = false;
    }
    h->map.built = false;
    h->map.pending = false;
  }
  cudaIpcMemHandle_t ipc;
  CU_TRY(h, cudaIpcGetMemHandle(&ipc, h->arena));
  memcpy(handle64, &ipc, 64);
  return VGICP_OK;
}

int vgicp_comm_init_arena(vgicp_handle h, const unsigned char* all_handles) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!all_handles) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "comm_init_arena: null handles");
  if (h->comm_ranks < 1 || !h->arena) return fail(h, VGICP_ERR_BAD_STATE, "comm_init_arena: call vgicp_comm_init and vgicp_comm_export_arena first");
  for (int r = 0; r < h->comm_ranks; r++) {
    if (r == h->comm_rank) { h->arena_peers[r] = h->arena; continue; }
    cudaIpcMemHandle_t ipc;
    memcpy(&ipc, all_handles + (size_t)r * 64, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail(h, VGICP_ERR_COMM, std::string("comm_init_arena: cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
    h->arena_peers[r] = reinterpret_cast<unsigned char*>(p);
  }
  return VGICP_OK;
}

int vgicp_set_stage1_sharding(vgicp_handle h, int enable) {
  CHECK_HANDLE(h);
  h->stage1_sharding = enable ? 1 : 0;
  return VGICP_OK;
}

int vgicp_comm_shutdown(vgicp_handle h) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->stream_b) cudaStreamSynchronize(h->stream_b);
  for (int r = 0; r < h->comm_ranks; r++)
    if (r != h->comm_rank && h->arena_peers[r]) cudaIpcCloseMemHandle(h->arena_peers[r]);
  for (int r = 0; r < kCommMaxRanks; r++) h->arena_peers[r] = nullptr;
  for (int r = 0; r < h->comm_ranks; r++)
    if (r != h->comm_rank && h->comm_peers[r]) cudaIpcCloseMemHandle(h->comm_peers[r]);
  for (int r = 0; r < kCommMaxRanks; r++) h->comm_peers[r] = nullptr;
  h->comm_ranks = 0;
  h->comm_rank = 0;
  return VGICP_OK;
}

int vgicp_comm_error(vgicp_handle h, int* error) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!error) return VGICP_ERR_INVALID_ARGUMENT;
  *error = 0;
  if (h->comm_box) {
    CommMailbox tmp;
    CU_TRY(h, cudaMemcpy(&tmp, h->comm_box, sizeof(CommMailbox), cudaMemcpyDeviceToHost));
    *error = tmp.error;
  }
  if (h->arena) {
    CommArenaHeader hdr;
    CU_TRY(h, cudaMemcpy(&hdr, h->arena, sizeof(hdr), cudaMemcpyDeviceToHost));
    *error |= hdr.error;
  }
  return VGICP_OK;
}

int vgicp_set_source_shard(vgicp_handle h, size_t begin, size_t end) {
  CHECK_HANDLE(h);
  if (end < begin) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_source_shard: end < begin");
  h->shard_begin = (int)begin;
  h->shard_end = (int)end;
  return VGICP_OK;
}

int vgicp_clear_source_shard(vgicp_handle h) {
  CHECK_HANDLE(h);
  h->shard_begin = 0;
  h->shard_end = -1;
  return VGICP_OK;
}

// ---- NDT (NDTCudaCore, src/fast_gicp/cuda/ndt_cuda.cu) on the same handle -------------------------------------------------
int vgicp_set_problem(vgicp_handle h, int problem) {
  CHECK_HANDLE(h);
  if (problem < 0 || problem > 2) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_problem: 0 VGICP, 1 NDT P2D, 2 NDT D2D");
  if (problem != h->problem) { h->ndt_ready = false; h->has_lin = false; }
  h->problem = problem;
  return VGICP_OK;
}

int vgicp_ndt_create_voxelmaps(vgicp_handle h) {  // NDTCudaCore::create_voxelmaps, ndt_cuda.cu:118-141
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (h->problem == 0) return fail(h, VGICP_ERR_BAD_STATE, "ndt_create_voxelmaps: select an NDT problem first (vgicp_set_problem)");
  return ndt_prepare(h);  // idempotent like the reference's: existing maps are kept
}

int vgicp_set_execution_hint(vgicp_handle h, int hint) {
  CHECK_HANDLE(h);
  if (hint < 0 || hint > 1) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_execution_hint: 0 latency, 1 throughput");
  h->exec_hint = hint;
  return VGICP_OK;
}

int vgicp_set_align_mode(vgicp_handle h, int mode) {
  CHECK_HANDLE(h);
  if (mode < 0 || mode > 1) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_align_mode: 0 device-resident loop, 1 host-driven loop");
  h->align_mode = mode;
  return VGICP_OK;
}

int vgicp_set_knn_mode(vgicp_handle h, int mode) {
  CHECK_HANDLE(h);
  if (mode < 0 || mode > 2) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_knn_mode: 0 grid, 1 warp scan, 2 legacy scan");
  h->knn_mode = mode;
  return VGICP_OK;
}

int vgicp_set_speculation(vgicp_handle h, int enable) {
  CHECK_HANDLE(h);
  h->speculate = enable ? 1 : 0;
  return VGICP_OK;
}

int vgicp_set_voxel_index(vgicp_handle h, int mode) {
  CHECK_HANDLE(h);
  if (mode < 0 || mode > 1) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_voxel_index: 0 direct-mapped index when it fits, 1 hash table only");
  h->voxel_index_mode = mode;
  return VGICP_OK;
}

int vgicp_set_profiling(vgicp_handle h, int enable) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  CU_TRY(h, cudaStreamSynchronize(h->stream_b));
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  for (auto& r : h->prof_pending) { h->prof_pool.push_back(r.a); h->prof_pool.push_back(r.b); }
  h->prof_pending.clear();
  for (int i = 0; i < VGICP_PROF_NUM_CATEGORIES; i++) { h->prof_ms[i] = 0.0; h->prof_launches[i] = 0; }
  h->prof_on = enable != 0;
  return VGICP_OK;
}

int vgicp_get_profile(vgicp_handle h, double* ms, uint64_t* launches, int capacity) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!ms || !launches || capacity < VGICP_PROF_NUM_CATEGORIES) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_profile: need VGICP_PROF_NUM_CATEGORIES entries");
  CU_TRY(h, cudaStreamSynchronize(h->stream_b));
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  for (auto& r : h->prof_pending) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) h->prof_ms[r.cat] += (double)t;
    h->prof_pool.push_back(r.a);
    h->prof_pool.push_back(r.b);
  }
  h->prof_pending.clear();
  for (int i = 0; i < VGICP_PROF_NUM_CATEGORIES; i++) { ms[i] = h->prof_ms[i]; launches[i] = h->prof_launches[i]; }
  return VGICP_OK;
}

const char* vgicp_profile_category_name(int category) {
  static const char* names[VGICP_PROF_NUM_CATEGORIES] = {"unpack_points", "knn", "covariance", "voxelmap_build", "linearize", "compute_error", "other"};
  return (category >= 0 && category < VGICP_PROF_NUM_CATEGORIES) ? names[category] : "";
}

// pcl::Registration::getFitnessScore(max_range): mean squared distance from the transformed source points to their nearest
// target point over the pairs with d^2 <= max_range (PCL compares the squared distance with max_range).
int vgicp_get_fitness_score(vgicp_handle h, const double T[16], double max_range, double* score) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!T || !score) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_fitness_score: null argument");
  if (!h->source.has_pts || !h->target.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "get_fitness_score: source and target clouds required");
  const int n = h->source.n;
  *score = std::numeric_limits<double>::max();
  if (n == 0 || h->target.n == 0) return VGICP_OK;
  if (h->source.st != h->stream) CU_TRY(h, cudaStreamWaitEvent(h->stream, h->source.ready, 0));
  if (h->target.st != h->stream) CU_TRY(h, cudaStreamWaitEvent(h->stream, h->target.ready, 0));
  CU_TRY(h, h->staging.reserve((size_t)n * sizeof(float)));
  float* d_out = reinterpret_cast<float*>(h->staging.p);
  KLAUNCH(h, VGICP_PROF_OTHER, k_nn1_sqdist<<<blocks_for(n, 256), 256, 0, h->stream>>>(h->source.pts.p, n, h->target.pts.p, h->target.n, to_pose(T), d_out));
  CU_TRY(h, cudaGetLastError());
  std::vector<float> d2(n);
  CU_TRY(h, cudaMemcpyAsync(d2.data(), d_out, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  double sum = 0.0;
  long cnt = 0;
  for (int i = 0; i < n; i++)
    if ((double)d2[i] <= max_range) { sum += (double)d2[i]; cnt++; }
  if (cnt > 0) *score = sum / (double)cnt;
  return VGICP_OK;
}

int vgicp_get_launch_count(vgicp_handle h, uint64_t* launches) {
  CHECK_HANDLE(h);
  if (!launches) return VGICP_ERR_INVALID_ARGUMENT;
  *launches = h->launches;
  return VGICP_OK;
}

int vgicp_synchronize(vgicp_handle h) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (h->map.pending) { int rc = voxelmap_finish(h, h->target, h->map); if (rc) return rc; }
  CU_TRY(h, cudaStreamSynchronize(h->stream_b));
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  return VGICP_OK;
}

int vgicp_get_stream(vgicp_handle h, uint64_t* stream) {
  CHECK_HANDLE(h);
  if (!stream) return VGICP_ERR_INVALID_ARGUMENT;
  *stream = (uint64_t)(uintptr_t)h->stream;
  return VGICP_OK;
}

}  // extern "C"
