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

#include <cmath>
#include <limits>
#include <new>
#include <string>
#include <type_traits>
#include <vector>

#include "lsq_math.hpp"
#include "vgicp_kernels.cuh"
#include "vgicp_local_map.cuh"
#include "vgicp_deskew.cuh"

using namespace vgicp;

namespace {

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
  Event ready;
  DevBuf<unsigned char> staging;
  DevBuf<unsigned char> knn_scratch;
  const float4* knn_sorted = nullptr;  // the cloud in the k-NN grid's Morton order (inside knn_scratch), original index in .w
  int knn_q_begin = 0, knn_q_end = 0;  // sorted positions whose neighbour rows the last find_neighbors computed
  int arena_slot = 0;                  // which half of the exchange arena holds this cloud's covariances (stage-1 sharding)
  unsigned long long arena_seq = 0;    // slices delivered for this cloud so far
};

constexpr long long kDenseMaxCells = 16ll << 20;  // 64 MB of cell ids per map at most

struct VoxelMap {
  bool created = false;  // GaussianVoxelMap object exists (keeps its first resolution, SURVEY Q3)
  bool built = false;
  bool pending = false;    // first insertion attempt enqueued, outcome not yet read (voxelmap_finish completes the build)
  int pending_B = 0;
  bool v_pending = false;  // num_voxels still in flight
  Event ev_attempt, ev_done;
  int ndt = 0;             // 1: built from the points alone + MIN_EIG (NDT), 0: from points + covariances (VGICP)
  DevPtr<int[]> d_counters;   // [0] fail count, [1] num_voxels, [2..4] / [5..7] min / max voxel coordinate, [8] set_neighbors verdict
  HostPtr<int[]> h_counters;  // pinned
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
};

// Where the evaluation kernels leave their results: `rows` records of `len` doubles, with the partial sums and tickets of their
// fixed-order fold.  Latency hint: the kernels write the records to mapped host memory and then set each row's completion word to
// the launch's sequence number, on which the host spins; throughput hint: the records go to device memory and are copied back.
struct EvalChannel {
  int rows = 0;
  size_t len = 0;
  DevBuf<double> partials;
  DevPtr<unsigned int[]> tickets;              // [rows]: zero before the first launch; reset by each row's last block
  DevPtr<double[]> d_out;                      // [rows][len] (throughput hint)
  HostPtr<double[]> h_out;                     // pinned + mapped, same shape (latency hint)
  HostPtr<unsigned long long[]> h_done;        // pinned + mapped per-row completion words
  unsigned long long seq = 0;                // the current launch's (or round's) sequence number
  struct Dest {
    double* out;
    volatile unsigned long long* done;  // nullptr under the throughput hint
    unsigned long long seq;
  };

  // fixed-size buffers at the first call (each one a failed call left missing at the next); the partial sums grow.  The shape is
  // the same at every call on a channel.
  cudaError_t open(int n_rows, size_t rec_len, size_t n_partials, cudaStream_t st) {
    rows = n_rows;
    len = rec_len;
    cudaError_t e = cudaSuccess;
    if (!tickets) {
      if ((e = device_alloc(tickets, rows * sizeof(unsigned int))) != cudaSuccess) return e;
      if ((e = cudaMemsetAsync(tickets.get(), 0, rows * sizeof(unsigned int), st)) != cudaSuccess) {
        tickets.reset();
        return e;
      }
    }
    if (!d_out && (e = device_alloc(d_out, rows * len * sizeof(double))) != cudaSuccess) return e;
    if (!h_done) {
      if ((e = host_alloc(h_done, rows * sizeof(unsigned long long), cudaHostAllocMapped)) != cudaSuccess) return e;
      memset(h_done.get(), 0, rows * sizeof(unsigned long long));
    }
    if (!h_out && (e = host_alloc(h_out, rows * len * sizeof(double), cudaHostAllocMapped)) != cudaSuccess) return e;
    return partials.reserve(n_partials);
  }
  // where a launch writes rows [row0, ...) under the execution hint
  Dest dest(bool direct, int row0 = 0) const {
    return {(direct ? h_out.get() : d_out.get()) + (size_t)row0 * len, direct ? h_done.get() + row0 : nullptr, seq};
  }
  int wait(vgicp_handle h, int n, size_t count);
};

}  // namespace

struct vgicp_context {
  int device = 0;
  Stream stream;
  std::string err;
  uint64_t launches = 0;

  double resolution = 1.0;
  double kernel_width = 0.25;
  double kernel_max_dist = 3.0;
  int offset_mode = 1;  // 1 / 7 / 27 = fixed tables, 0 = generic list
  int robust_kind = 0;        // VGICP_ROBUST_* (vgicp_set_robust_kernel)
  double robust_scale = 1.0;  // delta, Mahalanobis units
  int voxel_index_mode = 0;  // 0: direct-mapped index when the map's bounding box fits (else the hash table), 1: hash table only
  std::vector<int4> h_offsets;
  DevBuf<int4> d_offsets;

  Cloud source, target;
  VoxelMap map;

  bool has_lin = false;
  Pose lin;  // linearized_x (float)

  DevBuf<unsigned char> staging;    // main-stream scratch (transform_source, fitness score)
  Stream stream_b;                  // second cloud stream
  Event ev_copy;                    // "host buffer consumed" marker of set_cloud
  // multi-GPU source sharding
  DevPtr<CommMailbox> comm_box;                  // this rank's mailbox (device memory, IPC-exported)
  IpcPtr<CommMailbox> comm_peers[kCommMaxRanks];  // mapped peer mailboxes (empty at comm_rank: that one is comm_box)
  int comm_rank = 0, comm_ranks = 0;
  unsigned long long comm_seq = 0;
  int shard_begin = 0, shard_end = -1;           // evaluations cover source points [begin, end)
  // stage-1 sharding: exchange arena (covariances of both clouds + delivery flags), own and peers' (IPC-mapped)
  DevPtr<unsigned char[]> arena;
  IpcPtr<unsigned char[]> arena_peers[kCommMaxRanks];  // (empty at comm_rank: that one is arena)
  bool arena_mapped = false;                         // vgicp_comm_init_arena has mapped every rank's arena
  size_t arena_points = 0;
  int stage1_sharding = 0;
  int speculate = 1;  // LM trial evaluations also linearise at the trial pose (vgicp_set_speculation)
  int exec_hint = 0;  // 0 = latency (one registration should finish as soon as possible), 1 = throughput (many concurrent handles)
  DevBuf<int> corr_ids;
  EvalChannel eval;  // single-pose evaluations: one record of 64 doubles (43 used, [44] the sharded exchange's error flag)
  // multi-pose evaluations (vgicp_align_multi / vgicp_evaluate_poses) have a channel of their own, so that they leave every piece
  // of single-pose state (lin, eval) as it was; opened at the first multi-pose call: [kMultiMaxHyp][kMultiOut], partials
  // [rows][grid][kLinStride]
  EvalChannel multi;
  DevPtr<unsigned char[]> d_multi_in;   // per-launch input: poses [hypotheses][2], then the row -> hypothesis list
  HostPtr<unsigned char[]> h_multi_in;  // pinned staging of d_multi_in

  // NDT (NDTCudaCore, ndt_cuda.cu): 0 = VGICP problem, 1 = NDT point-to-distribution, 2 = NDT distribution-to-distribution
  int problem = 0;
  VoxelMap ndt_t, ndt_s;        // target / source NDT voxel maps
  DevBuf<float4> ndt_src_pts;   // D2D: source voxel means as the evaluation's source cloud
  DevBuf<float4> ndt_src_covA;  // D2D: source voxel covariances; P2D: zeros
  DevBuf<float2> ndt_src_covB;
  int ndt_src_n = 0;
  bool ndt_ready = false;

  // local map (vgicp_append_source_to_target / vgicp_crop_target)
  Event ev_append;                  // end of the last append: the source's stream waits for it before the source is overwritten
  DevBuf<int> crop_rank;            // per target point: rank among the points that pass the radius test, or -1
  DevBuf<unsigned long long> crop_state;  // k_crop_rank look-back (epoch-tagged block totals)
  unsigned crop_epoch = 0;
  DevBuf<float4> spare_pts, spare_covA;  // the crop compacts into these and swaps them with the target's arrays
  DevBuf<float2> spare_covB;

  // optional per-kernel timing (vgicp_set_profiling): CUDA events on the handle's stream around every launch
  bool prof_on = false;
  struct ProfRec { int cat; Event a, b; };
  std::vector<ProfRec> prof_pending;
  std::vector<Event> prof_pool;
  double prof_ms[VGICP_PROF_NUM_CATEGORIES] = {0};
  uint64_t prof_launches[VGICP_PROF_NUM_CATEGORIES] = {0};

  // motion compensation (vgicp_deskew_source); last, so that no other member moves, and created at the first call, so that a handle
  // that never deskews does no extra work
  Event ev_deskew;                  // end of the work enqueued on the main stream: the in-place deskew must not overtake its reads
  std::vector<float> deskew_times;  // the caller's timestamps, packed contiguously

  // vgicp_register with resident clouds: the k-NN search and covariances of both clouds and the first voxel-map insertion attempt
  // replayed as one CUDA graph.  Kernel arguments are frozen in a graph, so it is keyed on the shapes and on every buffer it touches.
  struct Stage1Graph {
    std::vector<uintptr_t> seen;  // key of the last eager stage 1 (a second call with the same key captures)
    std::vector<uintptr_t> key;   // key of `exec`
    GraphExec exec;
    const float4* sorted[2] = {nullptr, nullptr};  // target / source k-NN order (host state the enqueue code leaves behind)
    int pending_B = 0;
    uint64_t launches = 0;  // kernel nodes, counted as launches on every replay
    uint64_t prof_launches[VGICP_PROF_NUM_CATEGORIES] = {0};
  } s1;

  // continuous-time registration (vgicp_set_source_timestamps, vgicp_compute_error_ct, vgicp_align_ct): the source's timestamps and
  // a channel of its own for the evaluation, so that it leaves the single-pose state as it was; opened at first use: one record of
  // kCtStride doubles, partials [kLinMaxBlocks][kCtStride]
  bool ct_has_times = false;
  float ct_tau = 0.0f;    // (float)t_ref
  double ct_span = 0.0;   // S = max_i |t_i - tau| (float differences)
  DevBuf<float> ct_times;
  EvalChannel ct;

  // timestamps from device memory and the deskew with the stored ones (vgicp_set_source_timestamps_device,
  // vgicp_deskew_source_stored): the raw range and t_ref kept with the timestamps, so that the stored deskew applies
  // vgicp_deskew_source's own bound in double; the spare buffer the device read packs into (swapped with ct_times on success)
  float ct_lo = 0.0f, ct_hi = 0.0f;
  double ct_t_ref = 0.0;
  DevBuf<float> ct_spare;
  DevBuf<unsigned> ct_stats;  // [3]: k_gather_times' non-finite count, ~key(min), key(max)

  // multi-source alignment (vgicp_align_sources): the sources' points and covariances back to back in one grow-only pool; stage 1
  // runs source by source on `srcs`, a cloud whose point and covariance arrays are views into the pool and whose neighbour rows and
  // k-NN scratch are reused from source to source; `src_rows` is the evaluation kernels' row descriptor table
  DevBuf<float4> src_pts, src_covA;
  DevBuf<float2> src_covB;
  Cloud srcs;
  DevBuf<SourceRow> src_rows;

  // voxel-capped thinning of the local map (vgicp_thin_target): u64 cell keys and original indices sorted stably (vgicp_sort.cuh),
  // the sort's scratch, the per-point keep mask k_crop_rank reads, and the box pass's words
  DevBuf<unsigned long long> thin_keys[2];
  DevBuf<unsigned> thin_vals[2];
  DevBuf<unsigned char> thin_scratch;
  DevBuf<unsigned char> thin_keep;
  DevBuf<unsigned> thin_box;

  // carving of the local map (vgicp_carve_target): the scan's range image, float bits of the least range per pixel (the keep
  // mask is thin_keep)
  DevBuf<unsigned> carve_img;
};

namespace {

int fail(vgicp_handle h, int code, const std::string& msg) {
  if (h) h->err = msg;
  return code;
}

Event prof_event(vgicp_handle h) {
  Event e;
  if (h->prof_pool.empty()) {
    event_create(e, cudaEventDefault);
  } else {
    e = std::move(h->prof_pool.back());
    h->prof_pool.pop_back();
  }
  return e;
}
inline void prof_begin(vgicp_handle h, int cat, cudaStream_t st) {
  h->prof_launches[cat]++;
  if (!h->prof_on) return;
  vgicp_context::ProfRec r{cat, prof_event(h), prof_event(h)};
  cudaEventRecord(r.a.get(), st);
  h->prof_pending.push_back(std::move(r));
}
inline void prof_end(vgicp_handle h, cudaStream_t st) {
  if (!h->prof_on) return;
  cudaEventRecord(h->prof_pending.back().b.get(), st);
}
// every kernel launch of the library goes through here: counts it, optionally brackets it with events on its stream
#define KLAUNCH_ST(h, st, cat, ...) \
  do {                              \
    prof_begin(h, cat, st);         \
    __VA_ARGS__;                    \
    prof_end(h, st);                \
    (h)->launches++;                \
  } while (0)
#define KLAUNCH(h, cat, ...) KLAUNCH_ST(h, (h)->stream.get(), cat, __VA_ARGS__)

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

// ---- handle state: what a change to an input invalidates ----------------------------------------------------------------------
// These flags are written here and by the functions that produce what they describe (find_neighbors, calc_covariances*,
// set_covariances, voxelmap_begin / voxelmap_finish, ndt_prepare), nowhere else; nothing here calls the CUDA API.  "Order" is the
// k-NN order: knn_sorted with its query range.  Two asymmetries are deliberate: computed target covariances keep the VGICP map
// while uploaded ones drop it (vgicp_set_target_covariances), and a deskew keeps the timestamps (the same points, moved).

void drop_map(VoxelMap& m) { m.built = m.pending = false; }

// drops the cloud's rows, order and NDT map and ndt_ready, and by kind of change:
enum class Change {
  replaced,  // set_*_cloud(_device), vgicp_register, the multi-source pool: also the covariances, the source's timestamps, the VGICP map
  moved,     // deskew: also the covariances
  edited,    // append / crop / thin: rows added or removed with their covariances; the caller begins the VGICP map build
};
void points_changed(vgicp_handle h, Cloud& c, Change what) {
  c.k = 0;
  c.knn_sorted = nullptr;
  c.knn_q_begin = c.knn_q_end = 0;
  if (what != Change::edited) c.has_cov = false;
  if (&c != &h->source && &c != &h->target) return;  // the multi-source pool's cloud belongs to no map
  h->ndt_ready = false;
  drop_map(&c == &h->target ? h->ndt_t : h->ndt_s);  // NDT: that cloud's map only (ndt_cuda.cu:104,114)
  if (what == Change::replaced && &c == &h->source) h->ct_has_times = false;  // the timestamps belong to the points they came with
  if (what == Change::replaced && &c == &h->target) drop_map(h->map);
}

// find_neighbors, the stage-1 replay; set_neighbors without an order: host rows follow none, so calc_covariances runs unsharded
void neighbors_set(Cloud& c, int k, const float4* order = nullptr, int q_begin = 0, int q_end = 0) {
  c.k = k;
  c.knn_sorted = order;
  c.knn_q_begin = q_begin;
  c.knn_q_end = q_end;
}
void covariances_set(Cloud& c) { c.has_cov = true; }
void map_begun(VoxelMap& m) { m.built = false; m.pending = true; }

void covariances_dropped(vgicp_handle h) {
  h->target.has_cov = h->source.has_cov = false;
  drop_map(h->map);
}

// with both streams idle: the reference swaps its NDT maps (ndt_cuda.cu:90-93); a pending build was enqueued on the other stream
void clouds_swapped(vgicp_handle h) {
  std::swap(h->source, h->target);
  h->ct_has_times = false;
  drop_map(h->map);
  for (VoxelMap* vm : {&h->ndt_t, &h->ndt_s})
    if (vm->pending) drop_map(*vm);
  std::swap(h->ndt_t, h->ndt_s);
  h->ndt_ready = false;
}

void problem_set(vgicp_handle h, int problem) {
  if (problem != h->problem) h->ndt_ready = h->has_lin = false;
  h->problem = problem;
}
void lin_set(vgicp_handle h, const Pose& T) {
  h->lin = T;
  h->has_lin = true;
}

// Both timestamp setters: refused unless every t_i - tau is finite as the kernels form it (a float subtraction is monotonic in t_i, so
// S = max |t_i - tau| is reached at lo or hi); then install() puts the values in ct_times
template <class F>
int timestamps_commit(vgicp_handle h, const char* who, float lo, float hi, double t_ref, F&& install) {
  const float tau = (float)t_ref;
  const double span = fmax(fabs((double)(lo - tau)), fabs((double)(hi - tau)));
  if (!std::isfinite(span)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, std::string(who) + ": t_i - t_ref overflows a float");
  if (int rc = install()) return rc;
  h->ct_has_times = true;
  h->ct_tau = tau;
  h->ct_span = span;
  h->ct_lo = lo;
  h->ct_hi = hi;
  h->ct_t_ref = t_ref;
  return VGICP_OK;
}

// What an entry point needs before it launches anything.  The conditions are tested in this order, and the first one that does
// not hold is the error: a robust kind with NDT (kNeedEval) or continuous time with NDT (kNeedCt); a multi-GPU communicator
// (kNeedOneGpu) or any sharding (kNeedCt); the clouds (VGICP: source points, their covariances with kNeedEval, the voxel map; NDT:
// source and target points); the linearisation point (kNeedLin); the source's timestamps (kNeedCt).
enum : unsigned {
  kNeedEval = 1,    // evaluates residuals: a robust kind must fit the problem (NDT has its own Cauchy weight), covariances (VGICP)
  kNeedLin = 2,     // the correspondences of vgicp_update_correspondences
  kNeedOneGpu = 4,  // not in a multi-GPU communicator
  kNeedCt = 8,      // continuous time: VGICP on one GPU without sharding, with the source's timestamps
};
int check_ready(vgicp_handle h, const char* who, unsigned need) {
  const std::string w(who);
  if ((need & kNeedCt) && h->problem != 0) return fail(h, VGICP_ERR_UNSUPPORTED, w + ": continuous-time registration is defined for the VGICP problem only");
  if ((need & kNeedEval) && h->problem != 0 && h->robust_kind != VGICP_ROBUST_NONE)
    return fail(h, VGICP_ERR_UNSUPPORTED, w + ": a robust kernel is set (vgicp_set_robust_kernel) and an NDT problem is selected; NDT has its own weight");
  if ((need & kNeedOneGpu) && h->comm_ranks > 1) return fail(h, VGICP_ERR_UNSUPPORTED, w + ": not available on a handle in a multi-GPU communicator");
  if ((need & kNeedCt) && (h->comm_ranks > 1 || h->stage1_sharding || h->shard_end >= 0))
    return fail(h, VGICP_ERR_UNSUPPORTED, w + ": not available with source or stage-1 sharding or in a multi-GPU communicator");
  if (h->problem != 0) {
    if (!h->source.has_pts || !h->target.has_pts) return fail(h, VGICP_ERR_BAD_STATE, w + ": NDT needs source and target clouds");
  } else {
    if (!h->source.has_pts) return fail(h, VGICP_ERR_BAD_STATE, w + ": source cloud not set");
    if ((need & kNeedEval) && !h->source.has_cov) return fail(h, VGICP_ERR_BAD_STATE, w + ": source covariances required");
    if (!h->map.built && !h->map.pending) return fail(h, VGICP_ERR_BAD_STATE, w + ": target voxel map not built");
  }
  if ((need & kNeedLin) && !h->has_lin) return fail(h, VGICP_ERR_BAD_STATE, w + ": update_correspondences has not been called");
  if ((need & kNeedCt) && !h->ct_has_times) return fail(h, VGICP_ERR_BAD_STATE, w + ": the source has no timestamps (vgicp_set_source_timestamps)");
  return VGICP_OK;
}

int set_cloud(vgicp_handle h, Cloud& c, const float* xyz, size_t n, size_t stride, bool on_device = false) {
  points_changed(h, c, Change::replaced);
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
    CU_TRY(h, cudaEventRecord(c.ready.get(), c.st));
    return VGICP_OK;
  }
  CU_TRY(h, c.staging.reserve(n * stride));
  CU_TRY(h, cudaMemcpyAsync(c.staging.p, xyz, n * stride, cudaMemcpyHostToDevice, c.st));
  // the caller may free/modify xyz after return: pageable copies are staged synchronously by the driver, pinned ones are
  // not -> wait for the copy itself (an event right behind it), not for the kernels that follow
  CU_TRY(h, cudaEventRecord(h->ev_copy.get(), c.st));
  KLAUNCH_ST(h, c.st, VGICP_PROF_UNPACK, k_unpack_points<<<blocks_for(n, 256), 256, 0, c.st>>>(c.staging.p, stride, (int)n, c.pts.p));
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaEventRecord(c.ready.get(), c.st));
  CU_TRY(h, cudaEventSynchronize(h->ev_copy.get()));
  return VGICP_OK;
}

int set_neighbors(vgicp_handle h, Cloud& c, int k, const int* idx, size_t nk) {
  if (!c.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "set_neighbors: cloud not set");
  if (k <= 0 || !idx || nk != (size_t)k * (size_t)c.n) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_neighbors: k * num_points != neighbors.size()");
  CU_TRY(h, c.nbr.reserve(nk));
  CU_TRY(h, cudaMemcpyAsync(c.nbr.p, idx, nk * sizeof(int), cudaMemcpyHostToDevice, c.st));
  // an index outside [0, n) would be an illegal address in k_covariance_knn and poison the context of every handle of the process:
  // one pass over the table, the verdict comes back with the synchronisation the copy needs anyway
  int* bad = h->map.d_counters.get() + 8;
  CU_TRY(h, cudaMemsetAsync(bad, 0, sizeof(int), c.st));
  KLAUNCH_ST(h, c.st, VGICP_PROF_OTHER, k_validate_indices<<<blocks_for(nk, 256) < 8 * kNumSMs ? blocks_for(nk, 256) : 8 * kNumSMs, 256, 0, c.st>>>(c.nbr.p, nk, c.n, bad));
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(h->map.h_counters.get() + 8, bad, sizeof(int), cudaMemcpyDeviceToHost, c.st));
  CU_TRY(h, cudaStreamSynchronize(c.st));
  neighbors_set(c, h->map.h_counters[8] != 0 ? 0 : k);
  if (c.k == 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_neighbors: neighbour index outside [0, num_points)");
  return VGICP_OK;
}

int find_neighbors(vgicp_handle h, Cloud& c, int k) {
  if (!c.has_pts) return fail(h, VGICP_ERR_BAD_STATE, "find_neighbors: cloud not set");
  if (k <= 0 || k > kMaxK || k > c.n) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "find_neighbors: need 1 <= k <= min(num_points, 64)");
  CU_TRY(h, c.nbr.reserve((size_t)c.n * k));
  CU_TRY(h, c.knn_scratch.reserve(knn_grid_scratch_bytes(c.n, nullptr, nullptr)));
  int q_begin = 0, q_end = c.n;
  if (h->stage1_sharding && h->comm_ranks > 1 && h->arena_mapped) {  // this rank's slice of the queries (sorted positions)
    const long long base = c.n / h->comm_ranks, rem = c.n % h->comm_ranks, r = h->comm_rank;
    q_begin = (int)(r * base + (r < rem ? r : rem));
    q_end = q_begin + (int)base + (r < rem ? 1 : 0);
  }
  cudaError_t ke = cudaSuccess;
  int nl = 0;
  const float4* sorted = nullptr;
  KLAUNCH_ST(h, c.st, VGICP_PROF_KNN, ke = launch_knn_grid(c.pts.p, c.n, k, c.nbr.p, c.knn_scratch.p, c.knn_scratch.cap, q_begin, q_end, &nl, &sorted, c.st));
  h->launches += nl > 0 ? nl - 1 : 0;
  CU_TRY(h, ke);
  CU_TRY(h, cudaEventRecord(c.ready.get(), c.st));
  neighbors_set(c, k, sorted, q_begin, q_end);
  return VGICP_OK;
}

int calc_covariances(vgicp_handle h, Cloud& c, int method) {
  if (!c.has_pts || c.k <= 0) return fail(h, VGICP_ERR_BAD_STATE, "calculate_covariances: cloud and neighbours must be set first");
  if (method < 0 || method > 4) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "calculate_covariances: bad regularization method");
  CU_TRY(h, c.covA.reserve(c.n));
  CU_TRY(h, c.covB.reserve(c.n));
  const bool sharded = h->stage1_sharding && h->comm_ranks > 1 && h->arena_mapped && c.knn_sorted && (c.knn_q_begin > 0 || c.knn_q_end < c.n);
  if (c.n > 0 && sharded) {
    // this rank computed the neighbour rows of a slice only: covariances of that slice go straight into every rank's arena
    // (peer stores), then the ranks tell each other and wait -- all in stream order, the host does not block
    if ((size_t)c.n > h->arena_points) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "calculate_covariances: cloud larger than the exchange arena (vgicp_comm_export_arena max_points)");
    float4* pa[kCommMaxRanks];
    float2* pb[kCommMaxRanks];
    ArenaPeers ap;
    for (int r = 0; r < kCommMaxRanks; r++) {
      unsigned char* base = r >= h->comm_ranks ? nullptr : r == h->comm_rank ? h->arena.get() : h->arena_peers[r].get();
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
  covariances_set(c);
  CU_TRY(h, cudaEventRecord(c.ready.get(), c.st));
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
  covariances_set(c);
  CU_TRY(h, cudaEventRecord(c.ready.get(), c.st));
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
  covariances_set(c);
  CU_TRY(h, cudaEventRecord(c.ready.get(), c.st));
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
  int* skip = m.d_counters.get() + 9;
  CU_TRY(h, cudaMemsetAsync(skip, 0, sizeof(int), t.st));
  int Bj = B;
  for (int j = 0; j < count && Bj <= B_last; j++, Bj *= 2) {
    CU_TRY(h, cudaMemsetAsync(m.d_counters.get(), 0, sizeof(int), t.st));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_fill_i32<<<blocks_for(Bj, 256), 256, 0, t.st>>>(m.slots.p, -1, (size_t)Bj, skip));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_table_insert<<<blocks_for(n, 256), 256, 0, t.st>>>(m.coords.p, n, m.slots.p, (unsigned)(Bj - 1), m.max_scan, skip));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP,
               k_table_lookup_points<<<blocks_for(n, 256), 256, 0, t.st>>>(m.coords.p, n, m.slots.p, (unsigned)(Bj - 1), m.max_scan, m.slot_of_point.p, m.d_counters.get(), skip));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_table_verdict<<<1, 1, 0, t.st>>>(m.d_counters.get(), n, Bj));
  }
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(m.h_counters.get() + 9, m.d_counters.get() + 9, sizeof(int), cudaMemcpyDeviceToHost, t.st));
  CU_TRY(h, cudaEventRecord(m.ev_attempt.get(), t.st));
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
  drop_map(m);
  const int n = t.n;
  CU_TRY(h, m.coords.reserve(n));
  CU_TRY(h, m.slot_of_point.reserve(n));
  CU_TRY(h, cudaMemsetAsync(m.d_counters.get() + 2, 0x7f, 3 * sizeof(int), t.st));  // running minimum: starts at 0x7f7f7f7f
  CU_TRY(h, cudaMemsetAsync(m.d_counters.get() + 5, 0x80, 3 * sizeof(int), t.st));  // running maximum: starts at 0x80808080
  KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_voxel_coords<<<blocks_for(n, 256), 256, 0, t.st>>>(t.pts.p, n, m.res, m.coords.p, m.d_counters.get() + 2));
  CU_TRY(h, cudaMemcpyAsync(m.h_counters.get() + 2, m.d_counters.get() + 2, 6 * sizeof(int), cudaMemcpyDeviceToHost, t.st));
  // small clouds pass with the initial 8192 buckets (1082 voxels at 17 k points); large ones are given three sizes to try at once
  int rc = voxelmap_attempt(h, t, m, m.init_num_buckets, n > 200000 ? 3 : 1);
  if (rc) return rc;
  map_begun(m);
  return VGICP_OK;
}

int voxelmap_finish(vgicp_handle h, Cloud& t, VoxelMap& m) {
  if (!m.pending) return m.built ? VGICP_OK : fail(h, VGICP_ERR_BAD_STATE, "target voxel map not built");
  const int n = t.n;
  int B = 0;
  for (;;) {  // :265 (no upper bound in the reference; bounded here)
    CU_TRY(h, cudaEventSynchronize(m.ev_attempt.get()));
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
    const int* hc = m.h_counters.get();
    const long long nx = (long long)hc[5] - hc[2] + 1, ny = (long long)hc[6] - hc[3] + 1, nz = (long long)hc[7] - hc[4] + 1;
    if (nx > 0 && ny > 0 && nz > 0 && nx <= kDenseMaxCells && ny <= kDenseMaxCells && nz <= kDenseMaxCells && nx * ny <= kDenseMaxCells && nx * ny * nz <= kDenseMaxCells) {
      const size_t cells = (size_t)(nx * ny * nz);
      CU_TRY(h, m.dense_cells.reserve(cells));
      CU_TRY(h, cudaMemsetAsync(m.dense_cells.p, 0xff, cells * sizeof(int), t.st));
      m.dense = DenseIndex{m.dense_cells.p, hc[2], hc[3], hc[4], (unsigned)nx, (unsigned)ny, (unsigned)nz};
    }
  }
  {
    const int chunks = blocks_for(B, kRankThreads);
    CU_TRY(h, lookback_next(m.chunk_state, m.chunk_epoch, chunks, t.st));
    KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP,
               k_table_assign_ids<<<chunks, kRankThreads, 0, t.st>>>(m.coords.p, m.slots.p, B, m.buckets.p, m.d_counters.get() + 1, m.dense, m.chunk_state.p, m.chunk_epoch));
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
      KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_voxel_reduce<true><<<blocks_for(vmax, 4), 128, 0, t.st>>>(t.pts.p, nullptr, nullptr, order, m.segments.p, m.d_counters.get() + 1, m.vox.p));
      cudaError_t ke = cudaSuccess;
      KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, ke = launch_regularize_voxels(m.vox.p, m.d_counters.get() + 1, vmax, VGICP_REG_MIN_EIG, t.st));  // ndt_cuda.cu:129,140
      CU_TRY(h, ke);
    } else {
      KLAUNCH_ST(h, t.st, VGICP_PROF_VOXELMAP, k_voxel_reduce<false><<<blocks_for(vmax, 4), 128, 0, t.st>>>(t.pts.p, t.covA.p, t.covB.p, order, m.segments.p, m.d_counters.get() + 1, m.vox.p));
    }
  }
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(m.h_counters.get() + 1, m.d_counters.get() + 1, sizeof(int), cudaMemcpyDeviceToHost, t.st));
  CU_TRY(h, cudaEventRecord(m.ev_done.get(), t.st));
  CU_TRY(h, cudaEventRecord(t.ready.get(), t.st));
  m.v_pending = true;
  m.built = true;
  return VGICP_OK;
}

int voxelmap_num_voxels(vgicp_handle h, Cloud& t, VoxelMap& m, int* nv) {
  int rc = voxelmap_finish(h, t, m);
  if (rc) return rc;
  if (m.v_pending) {
    CU_TRY(h, cudaEventSynchronize(m.ev_done.get()));
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
  if (h->target.st != h->stream.get() && h->target.ready) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), h->target.ready.get(), 0));
  if (h->source.st != h->stream.get() && h->source.ready) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), h->source.ready.get(), 0));
  return VGICP_OK;
}

// arguments, kernel and launch geometry of an evaluation, decided once: a multi-pose launch runs, per row, the kernel and grid of the
// single-pose launch
struct LinLaunch {
  LinArgs a;
  bool stream;  // k_linearize_stream*, else the compacted kernels (k_linearize*)
  int G;        // compacted kernels: lanes per source point in the lookup phase
  int grid;     // blocks (per row of a multi-pose launch)
};
// The evaluation of the source (pts, covA, covB, n): arguments, kernel and grid.  Every evaluation takes its shape from here -- the
// handle's source (below) and each source of vgicp_align_sources alike.  allow_stream = false: the compacted kernels' shape also where
// DIRECT1 would stream (the continuous-time evaluation has no streaming kernel)
LinLaunch make_lin_launch(vgicp_handle h, const float4* pts, const float4* covA, const float2* covB, int n, bool allow_stream = true) {
  VoxelMap& m = h->problem != 0 ? h->ndt_t : h->map;
  LinLaunch L;
  LinArgs& a = L.a;
  a.ndt = h->problem != 0 ? 1 : 0;
  a.robust = h->problem == 0 ? h->robust_kind : 0;  // (the NDT entry points refuse a robust kind before they get here)
  a.robust_d2 = a.robust ? (float)(h->robust_scale * h->robust_scale) : 0.0f;
  a.pts = pts; a.covA = covA; a.covB = covB; a.n = n;
  a.comm_ranks = h->comm_ranks; a.comm_rank = h->comm_rank; a.comm_seq = 0;
  for (int r = 0; r < kCommMaxRanks; r++) a.comm_peers[r] = r >= h->comm_ranks ? nullptr : r == h->comm_rank ? h->comm_box.get() : h->comm_peers[r].get();
  a.buckets = m.buckets.p; a.mask = (unsigned)(m.num_buckets - 1); a.max_scan = m.max_scan; a.vox = m.vox.p;
  a.dense = m.dense;
  if (h->voxel_index_mode != 0) a.dense.cells = nullptr;
  a.offsets = h->d_offsets.p; a.n_off = (int)h->h_offsets.size(); a.res = m.res;
  a.Tlin = h->lin; a.Teval = h->lin;
  a.partials = h->eval.partials.p; a.ticket = h->eval.tickets.get(); a.out = h->eval.d_out.get();
  a.done_flag = nullptr; a.done_seq = 0;
  // lanes per source point in the lookup phase: split the neighbour cells of a point over G lanes while the cloud is too small to
  // fill the GPU with one thread per point (latency-bound regime); one lane per point once it is large
  const int n_off = a.n_off;
  const bool wide = a.n < 400000 && n_off > 1;
  // small clouds: split a point's cells over 3 (DIRECT27: whole z-columns), 4 (<= 7 offsets) or 8 lanes.  With the hits compacted
  // before the arithmetic the split costs no lane efficiency, so it is used under both execution hints
  const bool cols = h->offset_mode == 27;
  L.G = !wide ? 1 : (cols ? 3 : (n_off <= 7 ? 4 : 8));
  // DIRECT1 on a large cloud with the direct-mapped index: the bandwidth-bound shape, streamed through shared memory by bulk copies
  L.stream = allow_stream && h->offset_mode == 1 && a.dense.cells != nullptr && a.n >= 65536 && (reinterpret_cast<uintptr_t>(a.covB) & 15) == 0;
  if (L.stream) {
    const int tiles = (a.n + kLinStreamTile - 1) / kLinStreamTile;
    L.grid = tiles < kLinStreamMaxBlocks ? tiles : kLinStreamMaxBlocks;
  } else {
    const int tasks_per_block = (kLinThreads / 32) * ((32 / L.G) * L.G);
    long long tasks = (long long)(a.n > 0 ? a.n : 1) * L.G;
    long long grid = (tasks + tasks_per_block - 1) / tasks_per_block;
    L.grid = (int)(grid > kLinMaxBlocks ? kLinMaxBlocks : grid);
  }
  return L;
}
// the handle's source: VGICP points and covariances (the shard's slice under source sharding), NDT points + zero covariances (P2D)
// or the source's voxel Gaussians (D2D)
LinLaunch make_lin_launch(vgicp_handle h, bool allow_stream = true) {
  Cloud& s = h->source;
  if (h->problem != 0) return make_lin_launch(h, h->problem == 2 ? h->ndt_src_pts.p : s.pts.p, h->ndt_src_covA.p, h->ndt_src_covB.p, h->ndt_src_n, allow_stream);
  const int sb = h->shard_end >= 0 ? h->shard_begin : 0;
  const int se = h->shard_end >= 0 ? (h->shard_end < s.n ? h->shard_end : s.n) : s.n;
  return make_lin_launch(h, s.pts.p + sb, s.covA.p + sb, s.covB.p + sb, se > sb ? se - sb : 0, allow_stream);
}

template <int V>
using IntC = std::integral_constant<int, V>;

// The compacted evaluation kernels that exist: offset table MODE (1 / 7 / 27, 0 = generic list) with the lanes per point G that
// make_lin_launch picks for it.  Calls f(MODE, G) as compile-time constants; false when (mode, G) is not in the table.
template <int M, int GG>
struct LinShape { static constexpr int MODE = M, G = GG; };
template <class F, class... S>
bool with_shape(int mode, int G, F& f, S...) {
  return ((S::MODE == mode && S::G == G && (f(IntC<S::MODE>{}, IntC<S::G>{}), true)) || ...);
}
template <class F>
bool with_lin_shape(int mode, int G, F&& f) {
  return with_shape(mode, G, f, LinShape<1, 1>{}, LinShape<7, 1>{}, LinShape<7, 4>{}, LinShape<27, 1>{}, LinShape<27, 3>{}, LinShape<0, 1>{},
                    LinShape<0, 4>{}, LinShape<0, 8>{});
}

// Every evaluation launch: profiled under its kind's category and counted.  launch(WHAT, RB) gets the evaluation kind and the
// robust flag as compile-time constants, launches the kernel and returns false when none exists for the shape.
template <class F>
int launch_eval(vgicp_handle h, int kind, bool robust, F&& launch) {
  prof_begin(h, kind == kEvalError ? VGICP_PROF_ERROR : VGICP_PROF_LINEARIZE, h->stream.get());
  bool launched;
  auto with_kind = [&](auto rb) {
    if (kind == kEvalSpec) launched = launch(IntC<kEvalSpec>{}, rb);
    else if (kind == kEvalLinearize) launched = launch(IntC<kEvalLinearize>{}, rb);
    else launched = launch(IntC<kEvalError>{}, rb);
  };
  if (robust) with_kind(std::true_type{});
  else with_kind(std::false_type{});
  prof_end(h, h->stream.get());
  if (!launched) return fail(h, VGICP_ERR_UNSUPPORTED, "no evaluation kernel for this offset table and lane split");
  h->launches++;
  CU_TRY(h, cudaGetLastError());
  return VGICP_OK;
}

// one evaluation: launches the fused lookup+derivative kernel at Teval over the correspondences of h->lin
int launch_linearize(vgicp_handle h, const Pose& Teval, int kind) {
  LinLaunch L = make_lin_launch(h);
  LinArgs& a = L.a;
  a.Teval = Teval;
  a.comm_seq = h->comm_seq++;
  h->eval.seq++;
  // latency hint: the result goes straight to mapped host memory (UVA: the pinned pointers are valid on the device)
  const EvalChannel::Dest d = h->eval.dest(h->exec_hint == 0);
  a.out = d.out; a.done_flag = d.done; a.done_seq = d.seq;
  return launch_eval(h, kind, a.robust, [&](auto what, auto rb) {
    constexpr int WHAT = decltype(what)::value;
    constexpr bool RB = decltype(rb)::value;
    if (L.stream) {
      k_linearize_stream<WHAT, RB><<<L.grid, kLinThreads, sizeof(LinStreamSmem), h->stream.get()>>>(a);
      return true;
    }
    return with_lin_shape(h->offset_mode, L.G, [&](auto mode, auto g) {
      k_linearize<decltype(mode)::value, WHAT, decltype(g)::value, RB><<<L.grid, kLinThreads, 0, h->stream.get()>>>(a);
    });
  });
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
                 k_vox_to_cloud<<<blocks_for(vs, 256), 256, 0, s.st>>>(h->ndt_s.vox.p, h->ndt_s.d_counters.get() + 1, h->ndt_src_pts.p, h->ndt_src_covA.p, h->ndt_src_covB.p));
    CU_TRY(h, cudaGetLastError());
    CU_TRY(h, cudaEventRecord(s.ready.get(), s.st));
    h->ndt_src_n = vs;
  } else {
    CU_TRY(h, h->ndt_src_covA.reserve(s.n));
    CU_TRY(h, h->ndt_src_covB.reserve(s.n));
    CU_TRY(h, cudaMemsetAsync(h->ndt_src_covA.p, 0, sizeof(float4) * (size_t)s.n, s.st));
    CU_TRY(h, cudaMemsetAsync(h->ndt_src_covB.p, 0, sizeof(float2) * (size_t)s.n, s.st));
    CU_TRY(h, cudaEventRecord(s.ready.get(), s.st));
    h->ndt_src_n = s.n;
  }
  h->ndt_ready = true;
  return VGICP_OK;
}

// Waits for rows [0, n) of the launch (or round) just enqueued and leaves their records in h_out: under the latency hint by spinning
// on the completion words, under the throughput hint by copying `count` doubles back behind the launch.
int EvalChannel::wait(vgicp_handle h, int n, size_t count) {
  if (h->exec_hint == 0) {
    const volatile unsigned long long* done = h_done.get();
    for (int r = 0; r < n; r++) {
      long spins = 0;
      while (done[r] != seq) {
        __builtin_ia32_pause();
        if (++spins > 2000000L) {  // ~a few ms without an answer: fall back to a blocking wait (also surfaces launch errors)
          CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
          if (done[r] != seq) return fail(h, VGICP_ERR_CUDA, "evaluation kernel finished without publishing its result");
          break;
        }
      }
    }
    __sync_synchronize();
  } else {
    CU_TRY(h, cudaMemcpyAsync(h_out.get(), d_out.get(), count * sizeof(double), cudaMemcpyDeviceToHost, h->stream.get()));
    CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
  }
  return VGICP_OK;
}

// One single-pose evaluation at Teval over the correspondences of h->lin.  *rec: the result mailbox, valid until the next one:
// [0] err, [1..36] H and [37..42] b (kEvalLinearize, kEvalSpec: at Teval itself), [43] err over the correspondences of h->lin (kEvalSpec)
int evaluate(vgicp_handle h, const Pose& Teval, int kind, const double** rec) {
  int rc = launch_linearize(h, Teval, kind);
  if (rc) return rc;
  const size_t count = (h->comm_ranks > 1 || kind == kEvalSpec) ? kLinOutCommError + 1 : (kind == kEvalLinearize ? 43 : 1);
  if ((rc = h->eval.wait(h, 1, count))) return rc;
  if (h->comm_ranks > 1 && h->eval.h_out[kLinOutCommError] != 0.0) return fail(h, VGICP_ERR_COMM, "evaluate: a peer rank did not deliver its sums in time (vgicp_comm_error)");
  *rec = h->eval.h_out.get();
  return VGICP_OK;
}

// ---- multi-pose evaluation (vgicp_align_multi, vgicp_evaluate_poses) -------------------------------------------------------
// fixed-size buffers on first use; the partial sums grow with rows x grid (256 bytes per block and row)
int multi_reserve(vgicp_handle h, int rows, int grid) {
  const size_t in_bytes = (size_t)kMultiMaxHyp * (2 * sizeof(Pose) + sizeof(int)) + 16;
  if (!h->d_multi_in) CU_TRY(h, device_alloc(h->d_multi_in, in_bytes));
  if (!h->h_multi_in) CU_TRY(h, host_alloc(h->h_multi_in, in_bytes, cudaHostAllocDefault));
  CU_TRY(h, h->multi.open(kMultiMaxHyp, kMultiOut, (size_t)rows * grid * kLinStride, h->stream.get()));
  return VGICP_OK;
}

// Staged input of one round, in h->h_multi_in: Pose[n_hyp][2] (Tlin, Teval per hypothesis), then the row list (hypothesis per
// row, the rows of all launches of the round back to back).  One copy to the device per round.
size_t multi_rows_offset(int n_hyp) { return ((size_t)n_hyp * 2 * sizeof(Pose) + 15) & ~(size_t)15; }
struct MultiRound {
  vgicp_handle h;
  int n_hyp;
  int n = 0;  // rows staged
  Pose* poses = reinterpret_cast<Pose*>(h->h_multi_in.get());
  int* rows = reinterpret_cast<int*>(h->h_multi_in.get() + multi_rows_offset(n_hyp));
  // the next row: hypothesis i, evaluated at Te over the correspondences of Tl
  void add(int i, const double* Tl, const double* Te) {
    rows[n++] = i;
    poses[2 * i] = to_pose(Tl);
    poses[2 * i + 1] = to_pose(Te);
  }
  // a new sequence number for the round's records, and the copy
  int upload() {
    h->multi.seq++;
    CU_TRY(h, cudaMemcpyAsync(h->d_multi_in.get(), h->h_multi_in.get(), multi_rows_offset(n_hyp) + (size_t)n * sizeof(int), cudaMemcpyHostToDevice, h->stream.get()));
    return VGICP_OK;
  }
};

// one launch over rows [row0, row0 + n) of the staged row list, all computing `kind`; the records land in rows [row0, row0 + n)
// of the multi-pose output.  count: also count the hits (kEvalLinearize / kEvalError only).  src: the multi-source kernels, each
// row on its own source and grid from this descriptor table (L: the launch class's kernel, grid = the largest of its rows)
int launch_multi(vgicp_handle h, const LinLaunch& L, int n_hyp, int kind, bool count, int row0, int n, const SourceRow* src) {
  const LinArgs& a = L.a;
  const EvalChannel::Dest d = h->multi.dest(h->exec_hint == 0, row0);
  MultiArgs m;
  m.hyp = reinterpret_cast<const int*>(h->d_multi_in.get() + multi_rows_offset(n_hyp)) + row0;
  m.poses = reinterpret_cast<const Pose*>(h->d_multi_in.get());
  m.partials = h->multi.partials.p;  // (the launches of a round run one after the other on the stream: slices and tickets are reused)
  m.tickets = h->multi.tickets.get();
  m.out = d.out; m.done = d.done; m.done_seq = d.seq;
  m.src = src;
  const dim3 grid(L.grid, n);
  return launch_eval(h, kind, a.robust, [&](auto what, auto rb) {
    constexpr int WHAT = decltype(what)::value;
    constexpr bool RB = decltype(rb)::value;
    auto with_rows = [&](auto cnt, auto per_source) {
      constexpr bool COUNT = decltype(cnt)::value && WHAT != kEvalSpec;  // (the speculative evaluation counts no hits)
      constexpr bool SRC = decltype(per_source)::value;
      if (L.stream) {
        k_linearize_stream_multi<WHAT, COUNT, RB, SRC><<<grid, kLinThreads, sizeof(LinStreamSmem), h->stream.get()>>>(a, m);
        return true;
      }
      return with_lin_shape(h->offset_mode, L.G, [&](auto mode, auto g) {
        k_linearize_multi<decltype(mode)::value, WHAT, decltype(g)::value, COUNT, RB, SRC><<<grid, kLinThreads, 0, h->stream.get()>>>(a, m);
      });
    };
    if (m.src) return with_rows(std::false_type{}, std::true_type{});  // (the multi-source rows count no hits)
    return count ? with_rows(std::true_type{}, std::false_type{}) : with_rows(std::false_type{}, std::false_type{});
  });
}

// ---- LsqRegistration::computeTransformation (lsq_registration_impl.hpp:53-79) with step_gn (:106-120) / step_lm (:123-168) --------
// as a state machine that takes one evaluation record at a time, in host double arithmetic.  vgicp_align drives one with single-pose
// launches, vgicp_align_multi many with shared multi-pose launches.  The lookup pose of every evaluation is the float image of x0
// (x0 does not move between a linearisation and its trials); it is evaluated at x0 in phase kLmLinearize, at xi in phase kLmError.
// N = 6: the pose (vgicp_align, vgicp_align_multi).  N = 12: the pose and the sweep's body twist (vgicp_align_ct): the evaluation
// record is [err, H (12 x 12), b (12)] and a step d = [d_T; d_xi] moves T <- Exp(d_T) T, xi <- xi + d_xi.
template <int N>
struct LmState {
  vgicp_lsq_params p;
  Iso3d x0, xi, delta;  // estimate, LM trial pose, increment of the last step
  double tw0[6], twi[6];  // N = 12: twist estimate, LM trial twist
  double span;            // N = 12: S = max_i |s_i| (the sweep's reach from t_ref)
  double H[N * N], b[N], d[N], final_H[N * N];
  double y0, lambda, nu;
  int phase;  // kLmLinearize: err, H, b at x0;  kLmError: err at xi over the correspondences of x0;  kLmDone
  int it, lm_j, converged, lm_failed, n_linearize, n_error, nr_iterations;
};
enum { kLmLinearize = 0, kLmError = 1, kLmDone = 2 };

// the caller's parameters, or the defaults when it passes none
vgicp_lsq_params lsq_params(const vgicp_lsq_params* params) {
  vgicp_lsq_params P;
  if (params) P = *params; else vgicp_lsq_default_params(&P);
  return P;
}

template <int N>
LmState<N> lm_init(const double* guess, const vgicp_lsq_params& P) {
  LmState<N> st;
  memset(&st, 0, sizeof(st));
  st.p = P;
  memcpy(st.x0.m, guess, sizeof(st.x0.m));
  for (int j = 0; j < N; j++) st.final_H[j * (N + 1)] = 1.0;  // final_hessian_.setIdentity()
  st.lambda = -1.0;
  st.nu = 2.0;
  st.phase = P.max_iterations > 0 ? kLmLinearize : kLmDone;
  return st;
}

// the rotation of a twist over the sweep, |omega| S, stays within the series of deskew_point
bool twist_in_series(const double* xi, double span) { return sqrt(xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2]) * span <= 1.5707963267948966; }

// is_converged(delta) (:65-75); N = 12: and the step's motion of the sweep's end, Exp(S d_xi), as well
template <int N>
bool lm_step_converged(const LmState<N>& st) {
  bool c = is_converged(st.delta, st.p.rotation_epsilon, st.p.transformation_epsilon);
  if constexpr (N == 12) {
    double sd[6];
    for (int j = 0; j < 6; j++) sd[j] = st.span * st.d[6 + j];
    c = c && is_converged(se3_exp(sd), st.p.rotation_epsilon, st.p.transformation_epsilon);
  }
  return c;
}

template <int N>
void lm_reject(LmState<N>* st);

template <int N>
void lm_propose(LmState<N>* st) {  // solve (H + lambda I) d = -b, delta = exp(d), xi = delta * x0   (:134-139)
  double Hl[N * N], nb[N];
  memcpy(Hl, st->H, sizeof(Hl));
  for (int q = 0; q < N; q++) { Hl[q * (N + 1)] += st->lambda; nb[q] = -st->b[q]; }
  ldlt_solve<N>(Hl, nb, st->d);
  st->delta = se3_exp(st->d);
  st->xi = iso_mul(st->delta, st->x0);
  if constexpr (N == 12) {
    for (int j = 0; j < 6; j++) st->twi[j] = st->tw0[j] + st->d[6 + j];
    if (!twist_in_series(st->twi, st->span)) {  // outside the series: a rejected step, nothing to evaluate
      lm_reject(st);
      return;
    }
  }
  st->phase = kLmError;
}

template <int N>
void lm_finish_outer(LmState<N>* st) {  // end of step_optimize: converged_ = is_converged(delta), next outer iteration (:65-75)
  st->converged = lm_step_converged(*st) ? 1 : 0;
  st->it++;
  if (st->converged || st->it >= st->p.max_iterations) { st->phase = kLmDone; return; }
  st->nr_iterations = st->it;
  st->phase = kLmLinearize;
}

template <int N>
void lm_reject(LmState<N>* st) {  // a trial with rho < 0 (:151-159)
  if (lm_step_converged(*st)) { lm_finish_outer(st); return; }  // :151-154
  st->lambda = st->nu * st->lambda;
  st->nu = 2 * st->nu;
  st->lm_j++;
  if (st->lm_j >= st->p.lm_max_iterations) {  // step_lm returns false -> "lm not converged!!" (:69-72)
    st->lm_failed = 1;
    st->phase = kLmDone;
    return;
  }
  lm_propose(st);
}

template <int N>
void lm_advance(LmState<N>* st, const double* out /*err, H, b*/) {
  if (st->phase == kLmLinearize) {
    st->y0 = out[0];
    memcpy(st->H, out + 1, sizeof(st->H));
    memcpy(st->b, out + 1 + N * N, sizeof(st->b));
    st->n_linearize++;
    if (st->p.use_gauss_newton) {  // step_gn
      double nb[N];
      for (int q = 0; q < N; q++) nb[q] = -st->b[q];
      ldlt_solve<N>(st->H, nb, st->d);
      st->delta = se3_exp(st->d);
      if constexpr (N == 12) {
        double tw[6];
        for (int j = 0; j < 6; j++) tw[j] = st->tw0[j] + st->d[6 + j];
        if (!twist_in_series(tw, st->span)) {  // a step outside the series cannot be taken: stop with the last estimate
          st->lm_failed = 1;
          st->phase = kLmDone;
          return;
        }
        memcpy(st->tw0, tw, sizeof(tw));
      }
      st->x0 = iso_mul(st->delta, st->x0);
      memcpy(st->final_H, st->H, sizeof(st->H));
      lm_finish_outer(st);
      return;
    }
    if (st->lambda < 0.0) {  // :128-130
      double mx = 0.0;
      for (int j = 0; j < N; j++) mx = fmax(mx, fabs(st->H[j * (N + 1)]));
      st->lambda = st->p.lm_init_lambda_factor * mx;
    }
    st->nu = 2.0;
    st->lm_j = 0;
    if (st->p.lm_max_iterations <= 0) {  // step_lm tries no step and returns false: "lm not converged!!"
      st->lm_failed = 1;
      st->phase = kLmDone;
      return;
    }
    lm_propose(st);
    return;
  }
  // phase == kLmError  (:140-164)
  const double yi = out[0];
  st->n_error++;
  double den = 0.0;
  for (int q = 0; q < N; q++) den += st->d[q] * (st->lambda * st->d[q] - st->b[q]);
  const double rho = (st->y0 - yi) / den;
  if (rho < 0) {
    lm_reject(st);
    return;
  }
  st->x0 = st->xi;  // :161-164
  if constexpr (N == 12) memcpy(st->tw0, st->twi, sizeof(st->tw0));
  const double f = 1.0 - pow(2.0 * rho - 1.0, 3);
  st->lambda = st->lambda * fmax(1.0 / 3.0, f);
  memcpy(st->final_H, st->H, sizeof(st->H));
  lm_finish_outer(st);
}

// Takes one evaluation record (the single-pose mailbox and a multi-pose row share the layout: err, H, b in [0..42], [43] the trial's
// error over the current correspondences in a kEvalSpec record).  A speculative record's [43] decides the trial; when the trial is
// accepted and the optimisation goes on, the linearisation at the trial pose in [0..42] is taken at once.  Returns true in that case.
bool lm_consume(LmState<6>* st, const double* rec, bool spec) {
  if (!spec) {
    lm_advance(st, rec);
    return false;
  }
  lm_advance(st, rec + 43);
  if (st->phase != kLmLinearize) return false;
  lm_advance(st, rec);
  return true;
}

// a finished run's estimate, final system matrix and counters: the whole vgicp_align_result, all of vgicp_align_ct_result but the twist
template <int N, class R>
void lm_result(const LmState<N>& st, R* res) {
  static_assert(sizeof(res->H) == sizeof(st.final_H), "the result's H is the state's N x N final_H");
  memset(res, 0, sizeof(*res));
  memcpy(res->T, st.x0.m, sizeof(res->T));
  memcpy(res->H, st.final_H, sizeof(res->H));
  res->nr_iterations = st.nr_iterations;
  res->converged = st.converged;
  res->n_linearize = st.n_linearize;
  res->n_compute_error = st.n_error;
  res->lm_failed = st.lm_failed;
}

// ---- continuous-time registration (vgicp_compute_error_ct, vgicp_align_ct) ------------------------------------------------------
bool all_finite(const double* v, int n, bool as_float) {
  for (int j = 0; j < n; j++)
    if (!(as_float ? std::isfinite((float)v[j]) : std::isfinite(v[j]))) return false;
  return true;
}

// One evaluation at (Te, xe) over the correspondences of (Tl, xl): the compacted kernel and grid make_lin_launch picks (DIRECT1 on
// large clouds included) with the CT flag.  *raw: kCtValues folded sums (want_H) or err alone, valid until the next one.
int ct_evaluate(vgicp_handle h, const double* Tl, const double* xl, const double* Te, const double* xe, bool want_H, const double** raw) {
  LinLaunch L = make_lin_launch(h, false);
  LinArgs& a = L.a;
  a.Tlin = to_pose(Tl);
  a.Teval = to_pose(Te);
  CtArgs c;
  c.times = h->ct_times.p;
  c.tau = h->ct_tau;
  for (int j = 0; j < 6; j++) {
    c.xl[j] = (float)xl[j];
    c.xe[j] = (float)xe[j];
  }
  c.partials = h->ct.partials.p;
  c.ticket = h->ct.tickets.get();
  h->ct.seq++;
  const EvalChannel::Dest d = h->ct.dest(h->exec_hint == 0);
  c.out = d.out; c.done_flag = d.done; c.done_seq = d.seq;
  int rc = launch_eval(h, want_H ? kEvalLinearize : kEvalError, a.robust, [&](auto what, auto rb) {
    return with_lin_shape(h->offset_mode, L.G, [&](auto mode, auto g) {
      k_linearize_ct<decltype(mode)::value, decltype(what)::value == kEvalLinearize, decltype(g)::value, decltype(rb)::value><<<L.grid, kLinThreads, 0, h->stream.get()>>>(a, c);
    });
  });
  if (rc || (rc = h->ct.wait(h, 1, want_H ? kCtValues : 1))) return rc;
  *raw = h->ct.h_out.get();
  return VGICP_OK;
}

// the unique entries s[1..21] of a 6x6 block in apply_jacobian's order -> column-major 6x6 (lin_unpack's mapping)
void ct_unpack6(const double* s, double* H) {
  auto set = [&](int r, int c, double v) { H[c * 6 + r] = v; H[r * 6 + c] = v; };
  set(0, 0, s[1]); set(0, 1, s[2]); set(0, 2, s[3]); set(1, 1, s[4]); set(1, 2, s[5]); set(2, 2, s[6]);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) set(r, 3 + c, s[7 + r * 3 + c]);
  set(3, 3, s[16]); set(3, 4, s[17]); set(3, 5, s[18]); set(4, 4, s[19]); set(4, 5, s[20]); set(5, 5, s[21]);
}

// The 12 x 12 system (column-major) and b12 from the raw sums at T_eval:  H = [[H0, H1 K], [K^T H1, K^T H2 K]], b = [b0; K^T b1],
// K = [[R, 0], [[t]x R, R]] with (R, t) the float image of T_eval (include/vgicp_b200.h)
void ct_system(const double* raw, const double* Teval, double* H144, double* b12) {
  double H0[36], H1[36], H2[36], K[36] = {0};
  ct_unpack6(raw, H0);
  ct_unpack6(raw + 27, H1);
  ct_unpack6(raw + 54, H2);
  const double* b0 = raw + 22;
  const double* b1 = raw + 49;
  const Pose P = to_pose(Teval);
  double R[3][3], tx[3][3];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) R[r][c] = (double)P.r[r * 3 + c];
  const double t0 = P.t[0], t1 = P.t[1], t2 = P.t[2];
  const double S[3][3] = {{0.0, -t2, t1}, {t2, 0.0, -t0}, {-t1, t0, 0.0}};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) tx[r][c] = S[r][0] * R[0][c] + S[r][1] * R[1][c] + S[r][2] * R[2][c];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      K[c * 6 + r] = R[r][c];
      K[(3 + c) * 6 + 3 + r] = R[r][c];
      K[c * 6 + 3 + r] = tx[r][c];
    }
  double H1K[36], H2K[36];  // column-major products
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      double u = 0.0, v = 0.0;
      for (int k = 0; k < 6; k++) {
        u += H1[k * 6 + r] * K[c * 6 + k];
        v += H2[k * 6 + r] * K[c * 6 + k];
      }
      H1K[c * 6 + r] = u;
      H2K[c * 6 + r] = v;
    }
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      H144[c * 12 + r] = H0[c * 6 + r];
      H144[(6 + c) * 12 + r] = H1K[c * 6 + r];
      H144[c * 12 + 6 + r] = H1K[r * 6 + c];
    }
  for (int r = 0; r < 6; r++)
    for (int c = r; c < 6; c++) {  // K^T H2 K, symmetric by construction
      double v = 0.0;
      for (int k = 0; k < 6; k++) v += K[r * 6 + k] * H2K[c * 6 + k];
      H144[(6 + c) * 12 + 6 + r] = v;
      H144[(6 + r) * 12 + 6 + c] = v;
    }
  for (int r = 0; r < 6; r++) {
    b12[r] = b0[r];
    double v = 0.0;
    for (int k = 0; k < 6; k++) v += K[r * 6 + k] * b1[k];
    b12[6 + r] = v;
  }
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
  DeviceGuard g(device);
  // the kernel image is sm_90a only: fail loudly on anything else instead of falling back
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, k_linearize<1, kEvalLinearize, 1, false>) != cudaSuccess) {
    cudaGetLastError();
    delete h;
    return VGICP_ERR_NO_DEVICE;
  }
  bool ok = stream_create(h->stream, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && stream_create(h->stream_b, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && event_create(h->ev_copy, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && event_create(h->ev_append, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && event_create(h->target.ready, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && event_create(h->source.ready, cudaEventDisableTiming) == cudaSuccess;
  h->target.st = h->stream.get();    // the target (and its voxel map) is built on the main stream, where the evaluations run
  h->source.st = h->stream_b.get();  // the source's stage 1 overlaps with it
  for (VoxelMap* vm : {&h->map, &h->ndt_t, &h->ndt_s}) {
    ok = ok && device_alloc(vm->d_counters, 16 * sizeof(int)) == cudaSuccess;
    ok = ok && host_alloc(vm->h_counters, 16 * sizeof(int), cudaHostAllocDefault) == cudaSuccess;
    ok = ok && event_create(vm->ev_attempt, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && event_create(vm->ev_done, cudaEventDisableTiming) == cudaSuccess;
  }
  h->ndt_t.ndt = h->ndt_s.ndt = 1;
  ok = ok && h->eval.open(1, 64, (size_t)kLinStreamMaxBlocks * kLinStride, h->stream.get()) == cudaSuccess;
  ok = ok && cudaStreamSynchronize(h->stream.get()) == cudaSuccess;
  // fast_vgicp_cuda.cu:28-29, with the table on the device as well: the correspondence getter reads it under every method
  ok = ok && vgicp_set_neighbor_search_method(h, VGICP_DIRECT1, -1.0) == VGICP_OK;
  if (!ok) {
    delete h;
    return VGICP_ERR_CUDA;
  }
  *out = h;
  return VGICP_OK;
}

int vgicp_destroy(vgicp_handle h) {
  if (!h) return VGICP_OK;
  DeviceGuard g(h->device);  // (the members free their resources on the handle's device)
  if (h->stream) cudaStreamSynchronize(h->stream.get());
  if (h->stream_b) cudaStreamSynchronize(h->stream_b.get());
  if (h->comm_ranks > 1) vgicp_comm_shutdown(h);
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

static_assert((int)kRobustNone == (int)VGICP_ROBUST_NONE && (int)kRobustHuber == (int)VGICP_ROBUST_HUBER && (int)kRobustCauchy == (int)VGICP_ROBUST_CAUCHY &&
                  (int)kRobustGemanMcClure == (int)VGICP_ROBUST_GEMAN_MCCLURE,
              "the kernels' robust kinds are the C ABI's");
int vgicp_set_robust_kernel(vgicp_handle h, int kind, double scale) {
  CHECK_HANDLE(h);
  if (kind < VGICP_ROBUST_NONE || kind > VGICP_ROBUST_GEMAN_MCCLURE) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_robust_kernel: unknown kind");
  if (kind != VGICP_ROBUST_NONE && !(std::isfinite(scale) && scale > 0.0)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_robust_kernel: scale must be finite and positive");
  h->robust_kind = kind;
  h->robust_scale = kind != VGICP_ROBUST_NONE ? scale : 1.0;
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
    CU_TRY(h, cudaMemcpyAsync(h->d_offsets.p, off.data(), off.size() * sizeof(int4), cudaMemcpyHostToDevice, h->stream.get()));
    CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
  }
  h->h_offsets.swap(off);
  h->offset_mode = mode;
  return VGICP_OK;
}

int vgicp_set_source_cloud(vgicp_handle h, const float* xyz, size_t n, size_t stride_bytes) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return set_cloud(h, h->source, xyz, n, stride_bytes);
}

int vgicp_set_target_cloud(vgicp_handle h, const float* xyz, size_t n, size_t stride_bytes) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return set_cloud(h, h->target, xyz, n, stride_bytes);
}

int vgicp_swap_source_and_target(vgicp_handle h) {  // fast_vgicp_cuda.cu:97-107
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  // whole Cloud records are swapped, streams and `ready` events included (sync_inputs compares each cloud's stream with the main
  // stream, so it does not matter which one ends up where); everything in flight (incl. a pending map build that reads the old
  // target) must land first
  if (h->map.pending) { int rc0 = voxelmap_finish(h, h->target, h->map); if (rc0) return rc0; }
  CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
  CU_TRY(h, cudaStreamSynchronize(h->stream_b.get()));
  clouds_swapped(h);
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
  drop_map(h->map);  // the voxel Gaussians average the target covariances: the map must be rebuilt (create_target_voxelmap)
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
  if (int rc = check_ready(h, "update_correspondences", 0)) return rc;
  lin_set(h, to_pose(T));  // linearized_x = trans.cast<float>()
  // the lookup itself is fused into the evaluation kernel; the explicit list is only built by the getter
  return VGICP_OK;
}

int vgicp_get_voxel_correspondences(vgicp_handle h, int* pairs, size_t cap, size_t* n_pairs) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  { int rc = check_ready(h, "get_voxel_correspondences", kNeedLin); if (!rc) rc = sync_inputs(h); if (rc) return rc; }
  const LinLaunch LL = make_lin_launch(h);  // same source array / map as an evaluation (VGICP points, NDT points or voxel means)
  const int n = LL.a.n;
  const int n_off = (int)h->h_offsets.size();
  size_t total = (size_t)n * n_off;
  std::vector<int> ids(total);
  if (total) {
    CU_TRY(h, h->corr_ids.reserve(total));
    KLAUNCH(h, VGICP_PROF_OTHER,
            k_correspondence_ids<<<blocks_for(n, 128), 128, 0, h->stream.get()>>>(LL.a.pts, n, LL.a.buckets, LL.a.mask, LL.a.max_scan, h->d_offsets.p, n_off, LL.a.res, h->lin, h->corr_ids.p));
    CU_TRY(h, cudaGetLastError());
    CU_TRY(h, cudaMemcpyAsync(ids.data(), h->corr_ids.p, total * sizeof(int), cudaMemcpyDeviceToHost, h->stream.get()));
    CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
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
  int rc = check_ready(h, "compute_error", kNeedEval | kNeedLin);
  if (rc || (rc = sync_inputs(h))) return rc;
  const bool want_H = (H36 != nullptr && b6 != nullptr);  // compute_derivatives.cu:160
  const double* rec = nullptr;
  if ((rc = evaluate(h, to_pose(T), want_H ? kEvalLinearize : kEvalError, &rec))) return rc;
  if (err) *err = rec[0];
  if (want_H) {
    memcpy(H36, rec + 1, 36 * sizeof(double));
    memcpy(b6, rec + 37, 6 * sizeof(double));
  }
  return VGICP_OK;
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
// linearize = update_correspondences + compute_error (fast_vgicp_cuda_impl.hpp:170-173).  One single-pose launch per step of the
// state machine.  With LM and speculation every trial also linearises at the trial pose, so an accepted step needs no launch of its own.
int vgicp_align(vgicp_handle h, const double guess[16], const vgicp_lsq_params* params, vgicp_align_result* res) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!guess || !res) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align: null argument");
  { int rc = check_ready(h, "align", kNeedEval); if (!rc) rc = sync_inputs(h); if (rc) return rc; }
  const vgicp_lsq_params P = lsq_params(params);
  const bool speculate = h->speculate != 0 && !P.use_gauss_newton;
  LmState<6> st = lm_init<6>(guess, P);
  while (st.phase != kLmDone) {
    const bool lin = st.phase == kLmLinearize;
    const Pose Teval = to_pose(lin ? st.x0.m : st.xi.m);
    if (lin) {  // linearized_x: the correspondences of this evaluation and of the trials from it
      lin_set(h, Teval);
    }
    const double* rec = nullptr;
    int rc = evaluate(h, Teval, lin ? kEvalLinearize : (speculate ? kEvalSpec : kEvalError), &rec);
    if (rc) return rc;
    if (lm_consume(&st, rec, !lin && speculate)) h->lin = Teval;  // accepted trial, linearised at its pose by the same launch
  }
  lm_result(st, res);
  return VGICP_OK;
}

// The optimiser rounds of B LM states over shared multi-row launches (vgicp_align_multi, vgicp_align_sources).  Each round stages
// the running rows -- the linearisations first, then the trials, class by class within each -- and issues one launch per class and
// evaluation kind, with the largest grid of its rows; then every record goes to its state.  classes: the kernel and arguments of
// each launch class; cls[i], grid[i]: state i's class and its single-pose grid; src: the multi-source descriptor table (state i on
// source i), or nullptr (every state on the handle's source).
int lm_rounds(vgicp_handle h, std::vector<LmState<6>>& st, const std::vector<LinLaunch>& classes, const std::vector<int>& cls,
              const std::vector<int>& grid, const SourceRow* src, bool speculate) {
  const int B = (int)st.size();
  int grid_max = 0;
  for (int i = 0; i < B; i++) grid_max = grid[i] > grid_max ? grid[i] : grid_max;
  int rc = multi_reserve(h, B, grid_max);
  if (rc) return rc;
  struct Group { int row0, n, cls, grid; bool lin; };
  std::vector<Group> groups;
  for (;;) {
    MultiRound round{h, B};
    int n_lin = 0;
    groups.clear();
    for (int lin = 1; lin >= 0; lin--) {
      for (int q = 0; q < (int)classes.size(); q++) {
        Group gr{round.n, 0, q, 0, lin != 0};
        for (int i = 0; i < B; i++) {
          if (cls[i] != q || st[i].phase != (lin ? kLmLinearize : kLmError)) continue;
          round.add(i, st[i].x0.m, lin ? st[i].x0.m : st[i].xi.m);
          gr.grid = grid[i] > gr.grid ? grid[i] : gr.grid;
        }
        gr.n = round.n - gr.row0;
        if (gr.n) groups.push_back(gr);
      }
      if (lin) n_lin = round.n;
    }
    if (round.n == 0) return VGICP_OK;
    if ((rc = round.upload())) return rc;
    for (const Group& gr : groups) {
      LinLaunch L = classes[gr.cls];
      L.grid = gr.grid;
      if ((rc = launch_multi(h, L, B, gr.lin ? kEvalLinearize : (speculate ? kEvalSpec : kEvalError), false, gr.row0, gr.n, src))) return rc;
    }
    if ((rc = h->multi.wait(h, round.n, (size_t)round.n * kMultiOut))) return rc;
    const double* rec = h->multi.h_out.get();
    for (int r = 0; r < round.n; r++) lm_consume(&st[round.rows[r]], rec + (size_t)r * kMultiOut, r >= n_lin && speculate);
  }
}

// B registrations from B initial guesses.  Each hypothesis runs vgicp_align's state machine; every round stages the poses of the
// running hypotheses and evaluates all of them in one launch per evaluation kind.  With LM and speculation every round after the
// first is one k_linearize_multi<kEvalSpec> launch, whose accepted trials feed their linearisation straight back, as in vgicp_align.
int vgicp_align_multi(vgicp_handle h, const double* guesses, int n_guesses, const vgicp_lsq_params* params, vgicp_align_result* results) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!guesses || !results || n_guesses < 1 || n_guesses > kMultiMaxHyp) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_multi: null argument or n_guesses outside [1, 4096]");
  int rc = check_ready(h, "align_multi", kNeedEval | kNeedOneGpu);
  if (rc || (rc = sync_inputs(h))) return rc;
  const vgicp_lsq_params P = lsq_params(params);
  const int B = n_guesses;
  const LinLaunch L = make_lin_launch(h);
  std::vector<LmState<6>> st(B);
  for (int i = 0; i < B; i++) st[i] = lm_init<6>(guesses + 16 * i, P);
  const bool speculate = h->speculate != 0 && !P.use_gauss_newton;
  if ((rc = lm_rounds(h, st, {L}, std::vector<int>(B, 0), std::vector<int>(B, L.grid), nullptr, speculate))) return rc;
  for (int i = 0; i < B; i++) lm_result(st[i], &results[i]);
  return VGICP_OK;
}

// B poses scored in one launch: per pose, update_correspondences(T_i) + compute_error(T_i) and the hit count
int vgicp_evaluate_poses(vgicp_handle h, const double* T, int n_poses, double* err, double* H36, double* b6, int64_t* n_corr) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!T || !err || n_poses < 1 || n_poses > kMultiMaxHyp || (H36 == nullptr) != (b6 == nullptr))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "evaluate_poses: null argument, H36 without b6 (or b6 without H36), or n_poses outside [1, 4096]");
  int rc = check_ready(h, "evaluate_poses", kNeedEval | kNeedOneGpu);
  if (rc || (rc = sync_inputs(h))) return rc;
  const int B = n_poses;
  const bool want_H = H36 != nullptr;
  const LinLaunch L = make_lin_launch(h);
  if ((rc = multi_reserve(h, B, L.grid))) return rc;
  MultiRound round{h, B};
  for (int i = 0; i < B; i++) round.add(i, T + 16 * i, T + 16 * i);  // linearized_x = trans.cast<float>(), evaluated at the same pose
  if ((rc = round.upload())) return rc;
  if ((rc = launch_multi(h, L, B, want_H ? kEvalLinearize : kEvalError, true, 0, B, nullptr))) return rc;
  if ((rc = h->multi.wait(h, B, (size_t)B * kMultiOut))) return rc;
  const double* rec = h->multi.h_out.get();
  for (int i = 0; i < B; i++) {
    const double* o = rec + (size_t)i * kMultiOut;
    err[i] = o[0];
    if (want_H) {
      memcpy(H36 + 36 * (size_t)i, o + 1, 36 * sizeof(double));
      memcpy(b6 + 6 * (size_t)i, o + 37, 6 * sizeof(double));
    }
    if (n_corr) n_corr[i] = (int64_t)o[kMultiOutCount];
  }
  return VGICP_OK;
}

// B source clouds against the current map.  Stage 1 of each source is the handle's own set_cloud / find_neighbors / calc_covariances
// on a cloud whose arrays are views into the source pool; the optimisers then run as in vgicp_align_multi, one row per source.  The
// rows of a round are grouped by launch class (streaming or compacted kernel and lanes per point G; the offset table is the
// handle's): one launch per class and evaluation kind, with the largest grid of its rows.
int vgicp_align_sources(vgicp_handle h, const float* const* xyz, const size_t* n, size_t stride_bytes, int on_device, int k, int regularization_method,
                        const double* guesses, int n_sources, const vgicp_lsq_params* params, vgicp_align_result* results) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!xyz || !n || !results || n_sources < 1 || n_sources > kMultiMaxHyp) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_sources: null argument or n_sources outside [1, 4096]");
  if (stride_bytes < 12 || (stride_bytes % 4) != 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_sources: stride_bytes must be a multiple of 4 and >= 12");
  if (k < 1 || k > kMaxK) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_sources: need 1 <= k <= 64");
  if (regularization_method < 0 || regularization_method > 4) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_sources: bad regularization method");
  const int B = n_sources;
  for (int i = 0; i < B; i++) {
    if (!xyz[i]) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_sources: null points for source " + std::to_string(i));
    if (n[i] < (size_t)k || n[i] > (size_t)0x7fffffff / 64)
      return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_sources: source " + std::to_string(i) + " needs k <= num_points <= 2^31 / 64");
  }
  if (h->problem != 0) return fail(h, VGICP_ERR_UNSUPPORTED, "align_sources: defined for the VGICP problem only");
  if (h->comm_ranks > 1 || h->stage1_sharding || h->shard_end >= 0)
    return fail(h, VGICP_ERR_UNSUPPORTED, "align_sources: not available with source or stage-1 sharding or in a multi-GPU communicator");
  if (!h->map.built && !h->map.pending) return fail(h, VGICP_ERR_BAD_STATE, "align_sources: target voxel map not built");
  int rc = sync_inputs(h);
  if (rc) return rc;
  const vgicp_lsq_params P = lsq_params(params);

  // pool slots: at least one spare element per source (the streaming kernel reads covB in whole 16-byte units) and an even start,
  // so that every source's covB is 16-byte aligned like a cloud of its own
  std::vector<size_t> off(B + 1, 0);
  size_t n_max = 0;
  for (int i = 0; i < B; i++) {
    off[i + 1] = off[i] + ((n[i] + 32) & ~(size_t)31);
    n_max = n[i] > n_max ? n[i] : n_max;
  }
  CU_TRY(h, h->src_pts.reserve(off[B]));
  CU_TRY(h, h->src_covA.reserve(off[B]));
  CU_TRY(h, h->src_covB.reserve(off[B]));
  CU_TRY(h, h->src_rows.reserve(B));
  Cloud& c = h->srcs;
  if (!c.ready) {
    CU_TRY(h, event_create(c.ready, cudaEventDisableTiming));
    c.st = h->stream_b.get();
  }
  CU_TRY(h, c.nbr.reserve(n_max * k));  // (find_neighbors reserves as well; this keeps the buffers from growing source by source)
  CU_TRY(h, c.knn_scratch.reserve(knn_grid_scratch_bytes((int)n_max, nullptr, nullptr)));
  // the pool is rewritten on the cloud stream only after everything already enqueued on the main stream (which may read it)
  CU_TRY(h, cudaEventRecord(c.ready.get(), h->stream.get()));
  CU_TRY(h, cudaStreamWaitEvent(c.st, c.ready.get(), 0));

  // stage 1, source by source, and each source's launch shape and class: sources that share a kernel share the launches
  std::vector<SourceRow> desc(B);
  std::vector<LinLaunch> classes;  // per class, the kernel and arguments of its first source
  std::vector<int> cls(B), grid(B);
  for (int i = 0; i < B; i++) {
    const size_t cap = off[i + 1] - off[i];
    c.pts.attach(h->src_pts.p + off[i], cap);
    c.covA.attach(h->src_covA.p + off[i], cap);
    c.covB.attach(h->src_covB.p + off[i], cap);
    if ((rc = set_cloud(h, c, xyz[i], n[i], stride_bytes, on_device != 0))) return rc;
    if ((rc = find_neighbors(h, c, k))) return rc;
    rc = calc_covariances(h, c, regularization_method);
    if (rc && !(rc == VGICP_ERR_UNSUPPORTED && regularization_method == VGICP_REG_NORMALIZED_MIN_EIG)) return rc;  // (raw covariances, as vgicp_register)
    const LinLaunch L = make_lin_launch(h, c.pts.p, c.covA.p, c.covB.p, c.n);
    desc[i] = SourceRow{c.pts.p, c.covA.p, c.covB.p, c.n, L.grid};
    grid[i] = L.grid;
    cls[i] = 0;
    while (cls[i] < (int)classes.size() && !(classes[cls[i]].stream == L.stream && classes[cls[i]].G == L.G)) cls[i]++;
    if (cls[i] == (int)classes.size()) classes.push_back(L);
  }
  CU_TRY(h, cudaMemcpyAsync(h->src_rows.p, desc.data(), sizeof(SourceRow) * B, cudaMemcpyHostToDevice, h->stream.get()));
  CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), c.ready.get(), 0));

  std::vector<LmState<6>> st(B);
  const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  for (int i = 0; i < B; i++) st[i] = lm_init<6>(guesses ? guesses + 16 * i : I, P);
  const bool speculate = h->speculate != 0 && !P.use_gauss_newton;
  if ((rc = lm_rounds(h, st, classes, cls, grid, h->src_rows.p, speculate))) return rc;
  for (int i = 0; i < B; i++) lm_result(st[i], &results[i]);
  return VGICP_OK;
}

// ---- vgicp_register's stage 1 as a CUDA graph ------------------------------------------------------------------------------
// With both clouds resident, one registration enqueues ~30 kernels, ~10 memsets and two small copies before the host first waits;
// from many host threads at once the submission of these, not the GPU, limits the throughput.  The sequence depends only on the
// shapes and the buffers, so after one eager run with a given key the next call captures it (the same enqueue code, on the same
// streams) and later calls replay it with one cudaGraphLaunch.  The unpack kernels stay outside: their input pointers change on
// every call.  The host waits, the growth of the voxel table and everything after them (voxelmap_finish, the LM loop) stay eager.

// the plain VGICP path: no profiling (per-launch events), no sharding
static bool stage1_graph_eligible(vgicp_handle h, int reg) {
  return h->problem == 0 && !h->prof_on && !h->stage1_sharding && h->comm_ranks <= 1 && h->shard_end < 0 &&
         reg != VGICP_REG_NORMALIZED_MIN_EIG;
}

// everything the captured launches depend on besides the point data: shapes, settings, and the address and capacity of every
// buffer (grow-only buffers move when they grow; a crop or a swap exchanges arrays)
static void stage1_key(vgicp_handle h, int k, int reg, std::vector<uintptr_t>& key) {
  const VoxelMap& m = h->map;
  unsigned res_bits;
  memcpy(&res_bits, &m.res, sizeof(res_bits));
  key.assign({(uintptr_t)h->target.n, (uintptr_t)h->source.n, (uintptr_t)k, (uintptr_t)reg, (uintptr_t)m.created, (uintptr_t)res_bits,
              (uintptr_t)h->target.st, (uintptr_t)h->source.st, (uintptr_t)m.coords.p, m.coords.cap, (uintptr_t)m.slot_of_point.p, m.slot_of_point.cap,
              (uintptr_t)m.slots.p, m.slots.cap});
  for (const Cloud* c : {&h->target, &h->source})
    key.insert(key.end(), {(uintptr_t)c->pts.p, c->pts.cap, (uintptr_t)c->nbr.p, c->nbr.cap, (uintptr_t)c->covA.p, c->covA.cap, (uintptr_t)c->covB.p,
                           c->covB.cap, (uintptr_t)c->knn_scratch.p, c->knn_scratch.cap});
}

// k-NN + covariances of the target, first voxel-map attempt, k-NN + covariances of the source (each cloud on its own stream)
static int stage1_enqueue(vgicp_handle h, int k, int reg) {
  int rc;
  if ((rc = find_neighbors(h, h->target, k))) return rc;
  // NORMALIZED_MIN_EIG: raw covariances kept and VGICP_ERR_UNSUPPORTED reported (the reference prints a message and carries on,
  // covariance_regularization.cu:121-123); the class wrappers tolerate that code, so does the one-call registration
  if ((rc = calc_covariances(h, h->target, reg)) && rc != VGICP_ERR_UNSUPPORTED) return rc;
  if ((rc = build_voxelmap(h))) return rc;
  if ((rc = find_neighbors(h, h->source, k))) return rc;
  if ((rc = calc_covariances(h, h->source, reg)) && rc != VGICP_ERR_UNSUPPORTED) return rc;
  return VGICP_OK;
}

// after a launch of the graph: the `ready` events were recorded inside the capture and mean nothing outside it; both clouds are
// ready once the graph has run, and later work on a cloud stream must not overtake it
static int stage1_graph_done(vgicp_handle h) {
  CU_TRY(h, cudaEventRecord(h->map.ev_attempt.get(), h->stream.get()));
  for (Cloud* c : {&h->target, &h->source}) {
    CU_TRY(h, cudaEventRecord(c->ready.get(), h->stream.get()));
    if (c->st != h->stream.get()) CU_TRY(h, cudaStreamWaitEvent(c->st, c->ready.get(), 0));
  }
  return VGICP_OK;
}

// both clouds set (unpacked); enqueues stage 1 eagerly, or captures it, or replays the captured graph
static int stage1_resident(vgicp_handle h, int k, int reg) {
  vgicp_context::Stage1Graph& G = h->s1;
  std::vector<uintptr_t> key;
  stage1_key(h, k, reg, key);
  if (G.exec && key == G.key) {
    for (Cloud* c : {&h->target, &h->source})  // the unpacks (eager, on the cloud streams)
      if (c->st != h->stream.get()) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), c->ready.get(), 0));
    CU_TRY(h, cudaGraphLaunch(G.exec.get(), h->stream.get()));
    // the host state the enqueue code leaves behind, as it left it when the graph was captured
    Cloud* cl[2] = {&h->target, &h->source};
    for (int j = 0; j < 2; j++) {
      neighbors_set(*cl[j], k, G.sorted[j], 0, cl[j]->n);
      covariances_set(*cl[j]);
    }
    map_begun(h->map);
    h->map.pending_B = G.pending_B;
    h->launches += G.launches;
    for (int i = 0; i < VGICP_PROF_NUM_CATEGORIES; i++) h->prof_launches[i] += G.prof_launches[i];
    return stage1_graph_done(h);
  }
  if (key != G.seen) {  // first call with this key: eager (buffers reserved, arguments checked), remembered for the next call
    int rc = stage1_enqueue(h, k, reg);
    if (rc) return rc;
    stage1_key(h, k, reg, G.seen);
    return VGICP_OK;
  }
  // second call with this key: every reserve is a no-op now, so the enqueue code only enqueues -- capture it
  G.exec.reset();
  G.key.clear();
  const uint64_t l0 = h->launches;
  uint64_t p0[VGICP_PROF_NUM_CATEGORIES];
  memcpy(p0, h->prof_launches, sizeof(p0));
  for (Cloud* c : {&h->target, &h->source})
    if (c->st != h->stream.get()) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), c->ready.get(), 0));
  // thread-local: other host threads keep issuing their own work while this one captures
  CU_TRY(h, cudaStreamBeginCapture(h->stream.get(), cudaStreamCaptureModeThreadLocal));
  int rc = VGICP_OK;
  cudaError_t e = cudaSuccess;
  for (Cloud* c : {&h->target, &h->source})  // fork: the cloud streams join the capture
    if (c->st != h->stream.get() && e == cudaSuccess && (e = cudaEventRecord(c->ready.get(), h->stream.get())) == cudaSuccess) e = cudaStreamWaitEvent(c->st, c->ready.get(), 0);
  if (e == cudaSuccess) rc = stage1_enqueue(h, k, reg);
  for (Cloud* c : {&h->target, &h->source})  // join (also after a failure: the capture must end with every stream joined)
    if (c->st != h->stream.get()) cudaStreamWaitEvent(h->stream.get(), c->ready.get(), 0);
  cudaGraph_t graph = nullptr;
  const cudaError_t ee = cudaStreamEndCapture(h->stream.get(), &graph);
  if (e == cudaSuccess) e = ee;
  cudaGraphExec_t exec = nullptr;
  if (e == cudaSuccess && rc == VGICP_OK && (e = cudaGraphInstantiate(&exec, graph, 0)) == cudaSuccess) G.exec.reset(exec);
  if (graph) cudaGraphDestroy(graph);
  if (rc) return rc;
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(h, VGICP_ERR_CUDA, std::string("register: stage-1 graph capture: ") + cudaGetErrorString(e));
  }
  G.key = key;
  G.sorted[0] = h->target.knn_sorted;
  G.sorted[1] = h->source.knn_sorted;
  G.pending_B = h->map.pending_B;
  G.launches = h->launches - l0;
  for (int i = 0; i < VGICP_PROF_NUM_CATEGORIES; i++) G.prof_launches[i] = h->prof_launches[i] - p0[i];
  CU_TRY(h, cudaGraphLaunch(G.exec.get(), h->stream.get()));
  return stage1_graph_done(h);
}

// clear + setInputTarget + setInputSource + align in one call (the body of the reference's benchmark loop, src/align.cpp:72-81)
int vgicp_register(vgicp_handle h, const float* target_xyz, size_t n_target, const float* source_xyz, size_t n_source, size_t stride_bytes, int on_device, int k,
                   int regularization_method, const double guess[16], const vgicp_lsq_params* params, vgicp_align_result* result) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  int rc;
  if ((rc = set_cloud(h, h->target, target_xyz, n_target, stride_bytes, on_device != 0))) return rc;
  if ((rc = set_cloud(h, h->source, source_xyz, n_source, stride_bytes, on_device != 0))) return rc;
  // resident clouds on the plain path: stage 1 through the graph (one launch once it is captured)
  const bool graph = on_device && n_target > 0 && n_source > 0 && stage1_graph_eligible(h, regularization_method);
  if ((rc = graph ? stage1_resident(h, k, regularization_method) : stage1_enqueue(h, k, regularization_method))) return rc;
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
  if (h->source.st != h->stream.get()) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), h->source.ready.get(), 0));
  CU_TRY(h, h->staging.reserve((size_t)n * stride));
  // keep the non-xyz bytes of the caller's records untouched: copy in, overwrite xyz, copy out
  if (stride > 12) CU_TRY(h, cudaMemcpyAsync(h->staging.p, out_xyz, (size_t)n * stride, cudaMemcpyHostToDevice, h->stream.get()));
  KLAUNCH(h, VGICP_PROF_OTHER, k_transform_points<<<blocks_for(n, 256), 256, 0, h->stream.get()>>>(h->source.pts.p, n, to_pose(T), h->staging.p, stride));
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(out_xyz, h->staging.p, (size_t)n * stride, cudaMemcpyDeviceToHost, h->stream.get()));
  CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
  return VGICP_OK;
}

int vgicp_set_source_cloud_device(vgicp_handle h, const float* d_xyz, size_t n, size_t stride_bytes) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return set_cloud(h, h->source, d_xyz, n, stride_bytes, true);
}

int vgicp_set_target_cloud_device(vgicp_handle h, const float* d_xyz, size_t n, size_t stride_bytes) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  return set_cloud(h, h->target, d_xyz, n, stride_bytes, true);
}

// ---- local map: append the registered source to the target, crop the target ----
static int local_map_check(vgicp_handle h, const char* who) {
  if (h->problem != 0) return fail(h, VGICP_ERR_UNSUPPORTED, std::string(who) + ": NDT maps are built from the points alone; select the VGICP problem");
  if (h->stage1_sharding || h->target.covA.external)
    return fail(h, VGICP_ERR_UNSUPPORTED, std::string(who) + ": the target covariances live in the fixed-capacity exchange arena (stage-1 sharding)");
  if (!h->target.has_pts || !h->target.has_cov) return fail(h, VGICP_ERR_BAD_STATE, std::string(who) + ": target points and covariances required");
  return VGICP_OK;
}

// the target's arrays were replaced on its stream: leave the state set_target_cloud + set_target_covariances +
// create_target_voxelmap would leave (covariances, no neighbour rows, the map build enqueued at the map's first resolution)
static int local_map_rebuild(vgicp_handle h) {
  Cloud& t = h->target;
  points_changed(h, t, Change::edited);
  int rc = voxelmap_begin(h, t, h->map);
  if (rc) return rc;
  CU_TRY(h, cudaEventRecord(t.ready.get(), t.st));
  return VGICP_OK;
}

int vgicp_append_source_to_target(vgicp_handle h, const double T[16]) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!T) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "append_source_to_target: null pose");
  for (int i = 0; i < 16; i++)
    if (!std::isfinite(T[i])) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "append_source_to_target: non-finite pose");
  int rc = local_map_check(h, "append_source_to_target");
  if (rc) return rc;
  Cloud& s = h->source;
  Cloud& t = h->target;
  if (!s.has_pts || !s.has_cov) return fail(h, VGICP_ERR_BAD_STATE, "append_source_to_target: source points and covariances required");
  const size_t n = (size_t)t.n + (size_t)s.n;
  if (n > (size_t)0x7fffffff / 64) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "append_source_to_target: the merged target would exceed the points a cloud may hold");
  if (s.st != t.st) CU_TRY(h, cudaStreamWaitEvent(t.st, s.ready.get(), 0));
  CU_TRY(h, t.pts.grow(n, t.n, t.st));
  CU_TRY(h, t.covA.grow(n, t.n, t.st));
  CU_TRY(h, t.covB.grow(n, t.n, t.st));
  if (s.n > 0) {
    KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER,
               k_append_transformed<<<blocks_for(s.n, 256), 256, 0, t.st>>>(s.pts.p, s.covA.p, s.covB.p, s.n, to_pose(T), t.pts.p + t.n, t.covA.p + t.n, t.covB.p + t.n));
    CU_TRY(h, cudaGetLastError());
    // the next upload into the source's arrays (on the source's stream) must not overtake this read of them
    CU_TRY(h, cudaEventRecord(h->ev_append.get(), t.st));
    if (s.st != t.st) CU_TRY(h, cudaStreamWaitEvent(s.st, h->ev_append.get(), 0));
  }
  t.n = (int)n;
  return local_map_rebuild(h);
}

// k_crop_rank over the target (keep: the optional per-point mask, which replaces the radius test) and the read-back of the number of passing points, the one
// synchronisation of a crop and the second of a thinning; also sizes the spare arrays k_crop_scatter compacts into
static int local_map_rank(vgicp_handle h, const unsigned char* keep, float cx, float cy, float cz, float r2, size_t* passed) {
  Cloud& t = h->target;
  const int n = t.n;
  const int blocks = blocks_for(n, kRankThreads);
  CU_TRY(h, h->crop_rank.reserve(n));
  CU_TRY(h, lookback_next(h->crop_state, h->crop_epoch, blocks, t.st));
  CU_TRY(h, h->spare_pts.reserve(n));
  CU_TRY(h, h->spare_covA.reserve(n));
  CU_TRY(h, h->spare_covB.reserve(n));
  int* d_count = h->map.d_counters.get() + 10;
  KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER,
             k_crop_rank<<<blocks, kRankThreads, 0, t.st>>>(t.pts.p, keep, n, cx, cy, cz, r2, h->crop_rank.p, d_count, h->crop_state.p, h->crop_epoch));
  CU_TRY(h, cudaGetLastError());
  // the host needs the new size (and must refuse an empty result before anything is modified)
  CU_TRY(h, cudaMemcpyAsync(h->map.h_counters.get() + 10, d_count, sizeof(int), cudaMemcpyDeviceToHost, t.st));
  CU_TRY(h, cudaStreamSynchronize(t.st));
  *passed = (size_t)h->map.h_counters[10];
  return VGICP_OK;
}

// rows with rank >= first go to the spare arrays, which become the target's; then the map is rebuilt
static int local_map_compact(vgicp_handle h, int first, int kept) {
  Cloud& t = h->target;
  const int n = t.n;
  KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER,
             k_crop_scatter<<<blocks_for(n, 256), 256, 0, t.st>>>(t.pts.p, t.covA.p, t.covB.p, h->crop_rank.p, n, first, h->spare_pts.p, h->spare_covA.p, h->spare_covB.p));
  CU_TRY(h, cudaGetLastError());
  std::swap(t.pts, h->spare_pts);
  std::swap(t.covA, h->spare_covA);
  std::swap(t.covB, h->spare_covB);
  t.n = kept;
  return local_map_rebuild(h);
}

int vgicp_crop_target(vgicp_handle h, const double center[3], double radius, size_t max_points) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!center) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "crop_target: null center");
  if (!(radius >= 0.0)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "crop_target: radius must be >= 0 (NaN is rejected; +inf keeps every point)");
  int rc = local_map_check(h, "crop_target");
  if (rc) return rc;
  if (h->target.n == 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "crop_target: the crop would leave no points");
  size_t passed = 0;
  if ((rc = local_map_rank(h, nullptr, (float)center[0], (float)center[1], (float)center[2], (float)(radius * radius), &passed))) return rc;
  const size_t first = (max_points > 0 && passed > max_points) ? passed - max_points : 0;
  const int kept = (int)(passed - first);
  if (kept == 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "crop_target: the crop would leave no points");
  return local_map_compact(h, (int)first, kept);
}

// Thinning: the cells' box and the refusals the points decide (sync 1), u64 cell keys of the box's width with their digit
// histograms, the stable radix sort, the keep mask from the run test, then the crop's rank (sync 2: the new size) and scatter
int vgicp_thin_target(vgicp_handle h, double leaf_size, int max_points_per_voxel) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!std::isfinite(leaf_size) || !(leaf_size > 0.0)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "thin_target: leaf_size must be finite and > 0");
  const float l = (float)leaf_size;
  const float inv = 1.0f / l;
  if (!(std::isfinite(l) && l > 0.0f && std::isfinite(inv) && inv > 0.0f))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "thin_target: (float)leaf_size and its reciprocal must be finite and > 0");
  if (max_points_per_voxel < 1) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "thin_target: max_points_per_voxel must be >= 1");
  int rc = local_map_check(h, "thin_target");
  if (rc) return rc;
  Cloud& t = h->target;
  const int n = t.n;
  if (n == 0) return fail(h, VGICP_ERR_BAD_STATE, "thin_target: the target has no points");
  // 1. the box of the cells, read back: the refusals and the key width are decided before anything is modified
  CU_TRY(h, h->thin_box.reserve(kBoxWords));
  CU_TRY(h, cudaMemsetAsync(h->thin_box.p, 0, kBoxWords * sizeof(unsigned), t.st));
  const int bb = blocks_for(n, kThinBoxThreads);
  KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER, k_thin_box<<<bb < 4 * kNumSMs ? bb : 4 * kNumSMs, kThinBoxThreads, 0, t.st>>>(t.pts.p, n, inv, h->thin_box.p));
  CU_TRY(h, cudaGetLastError());
  unsigned box[kBoxWords];
  CU_TRY(h, cudaMemcpyAsync(box, h->thin_box.p, sizeof(box), cudaMemcpyDeviceToHost, t.st));
  CU_TRY(h, cudaStreamSynchronize(t.st));
  if (box[6]) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "thin_target: a target point has a non-finite coordinate");
  if (box[7]) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "thin_target: a cell floor(p * (1 / leaf)) lies outside [-2^31, 2^31)");
  int lo[3], bits[3];
  for (int a = 0; a < 3; a++) {
    lo[a] = cell_dec(~box[a]);
    const unsigned span = box[3 + a] - ~box[a];  // max - min
    bits[a] = span ? 32 - __builtin_clz(span) : 0;
  }
  const int key_bits = bits[0] + bits[1] + bits[2];
  if (key_bits > 64) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "thin_target: the cell key would be wider than 64 bits (leaf too small for the map's extent)");
  // 2. keys and digit histograms; 3. the sort (nothing to sort when every point is in one cell)
  const int passes = key_bits ? sort_num_passes(key_bits) : 0;
  for (int j = 0; j < 2; j++) {
    CU_TRY(h, h->thin_keys[j].reserve(n));
    CU_TRY(h, h->thin_vals[j].reserve(n));
  }
  CU_TRY(h, h->thin_keep.reserve(n));
  if (passes) {
    const size_t sb = sort_scratch_bytes(n, passes);
    CU_TRY(h, h->thin_scratch.reserve(sb));
    CU_TRY(h, cudaMemsetAsync(h->thin_scratch.p, 0, sb, t.st));
  }
  unsigned* hist = reinterpret_cast<unsigned*>(h->thin_scratch.p);
  const int kb = blocks_for(n, kSortThreads);
  KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER,
             k_thin_keys<<<kb < 4 * kNumSMs ? kb : 4 * kNumSMs, kSortThreads, 0, t.st>>>(t.pts.p, n, inv, make_int3(lo[0], lo[1], lo[2]), bits[0], bits[0] + bits[1], passes,
                                                                                         h->thin_keys[0].p, hist));
  CU_TRY(h, cudaGetLastError());
  const unsigned long long* skeys = h->thin_keys[0].p;
  const unsigned* svals = nullptr;
  if (passes) {
    int nl = 0;
    cudaError_t se = cudaSuccess;
    KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER,
               se = launch_sort_pairs<unsigned long long>(h->thin_keys[0].p, h->thin_vals[0].p, h->thin_keys[1].p, h->thin_vals[1].p, n, key_bits, h->thin_scratch.p, true,
                                                          nullptr, nullptr, &nl, t.st));
    CU_TRY(h, se);
    h->launches += nl > 0 ? nl - 1 : 0;
    skeys = h->thin_keys[passes & 1].p;
    svals = h->thin_vals[passes & 1].p;
  }
  // 4. the keep mask; 5. the crop's compaction with it (the mask alone decides)
  KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER, k_thin_keep<<<blocks_for(n, 256), 256, 0, t.st>>>(skeys, svals, n, max_points_per_voxel, h->thin_keep.p));
  CU_TRY(h, cudaGetLastError());
  size_t kept = 0;
  if ((rc = local_map_rank(h, h->thin_keep.p, 0.0f, 0.0f, 0.0f, std::numeric_limits<float>::infinity(), &kept))) return rc;
  return local_map_compact(h, 0, (int)kept);
}

void vgicp_carve_default_params(vgicp_carve_params* p) {
  if (!p) return;
  p->width = 1024;
  p->height = 64;
  p->elevation_min = -25.0 * M_PI / 180.0;
  p->elevation_max = 3.0 * M_PI / 180.0;
  p->window = 1;
  p->margin = 0.3;
  p->margin_rel = 0.02;
}

// Carving: the scan's range image (memset, k_carve_image on the target's stream after the source is ready), the keep mask
// (k_carve_keep), then thinning's compaction with it (the one synchronisation: the new size)
int vgicp_carve_target(vgicp_handle h, const double T[16], const vgicp_carve_params* params, size_t* removed) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!T || !params) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: null pose or params");
  for (int i = 0; i < 16; i++)
    if (!std::isfinite(T[i])) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: non-finite pose");
  const vgicp_carve_params& P = *params;
  if (P.width < 1 || P.height < 1 || (long long)P.width * P.height > (1ll << 24))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: width and height must be >= 1 with width * height <= 2^24");
  const double half_pi = 0.5 * M_PI;
  if (!(P.elevation_min > -half_pi && P.elevation_max < half_pi && P.elevation_min < P.elevation_max))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: the elevation limits must lie in (-pi/2, pi/2) with elevation_min < elevation_max");
  const double t_lo = tan(P.elevation_min), t_hi = tan(P.elevation_max);
  CarveImage im;
  im.W = P.width;
  im.H = P.height;
  im.wq = (float)P.width * 0.25f;
  im.e_lo = (float)t_lo;
  im.inv_de = (float)(P.height / (t_hi - t_lo));
  if (!std::isfinite(im.e_lo) || !(std::isfinite(im.inv_de) && im.inv_de > 0.0f))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: (float)tan(elevation_min) must be finite and the float row scale finite and > 0");
  if (P.window < 0 || P.window > 8) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: window must lie in [0, 8]");
  if (!(P.margin >= 0.0) || !std::isfinite((float)P.margin)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: margin must be finite and >= 0");
  if (!(P.margin_rel >= 0.0 && P.margin_rel < 1.0)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: margin_rel must lie in [0, 1)");
  int rc = local_map_check(h, "carve_target");
  if (rc) return rc;
  Cloud& s = h->source;
  Cloud& t = h->target;
  if (!s.has_pts || s.n == 0) return fail(h, VGICP_ERR_BAD_STATE, "carve_target: the source has no points");
  const int n = t.n;
  if (n == 0) return fail(h, VGICP_ERR_BAD_STATE, "carve_target: the target has no points");
  // Ti = [R^T | -R^T t] in double, cast once
  Pose Ti;
  for (int j = 0; j < 3; j++) {
    for (int k = 0; k < 3; k++) Ti.r[j * 3 + k] = (float)T[j * 4 + k];  // R_kj
    Ti.t[j] = (float)(-((T[j * 4 + 0] * T[12] + T[j * 4 + 1] * T[13]) + T[j * 4 + 2] * T[14]));
  }
  const size_t pixels = (size_t)P.width * (size_t)P.height;
  CU_TRY(h, h->carve_img.reserve(pixels));
  CU_TRY(h, h->thin_keep.reserve(n));
  // 1. the range image, from the source on the target's stream; the next upload into the source must not overtake this read
  CU_TRY(h, cudaMemsetAsync(h->carve_img.p, 0xFF, pixels * sizeof(unsigned), t.st));
  if (s.st != t.st) CU_TRY(h, cudaStreamWaitEvent(t.st, s.ready.get(), 0));
  KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER, k_carve_image<<<blocks_for(s.n, 256), 256, 0, t.st>>>(s.pts.p, s.n, im, h->carve_img.p));
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaEventRecord(h->ev_append.get(), t.st));
  if (s.st != t.st) CU_TRY(h, cudaStreamWaitEvent(s.st, h->ev_append.get(), 0));
  // 2. the keep mask; 3. thinning's compaction with it (the mask alone decides: a non-finite point it keeps stays)
  KLAUNCH_ST(h, t.st, VGICP_PROF_OTHER,
             k_carve_keep<<<blocks_for(n, 256), 256, 0, t.st>>>(t.pts.p, n, Ti, im, h->carve_img.p, P.window, (float)P.margin, (float)P.margin_rel, h->thin_keep.p));
  CU_TRY(h, cudaGetLastError());
  size_t kept = 0;
  if ((rc = local_map_rank(h, h->thin_keep.p, 0.0f, 0.0f, 0.0f, std::numeric_limits<float>::infinity(), &kept))) return rc;
  if (kept == 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "carve_target: the carve would leave no points");
  if (removed) *removed = (size_t)n - kept;
  return local_map_compact(h, 0, (int)kept);
}

// ---- motion compensation: deskew the source from per-point timestamps and a constant body twist ----
// The checks of a timestamp array that come before the values: stride, a source to match, its size, a t_ref finite as a float
static int timestamps_check(vgicp_handle h, const char* who, size_t n, size_t stride_bytes, double t_ref) {
  if (stride_bytes < 4 || (stride_bytes % 4) != 0) return fail(h, VGICP_ERR_INVALID_ARGUMENT, std::string(who) + ": stride_bytes must be a multiple of 4 and >= 4");
  const Cloud& s = h->source;
  if (!s.has_pts || s.n == 0) return fail(h, VGICP_ERR_BAD_STATE, std::string(who) + ": no source points");
  if (n != (size_t)s.n) return fail(h, VGICP_ERR_INVALID_ARGUMENT, std::string(who) + ": the number of timestamps differs from the number of source points");
  // the kernels take every value as a float: a value finite in double but not in float is rejected too
  if (!std::isfinite((float)t_ref)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, std::string(who) + ": non-finite t_ref");
  return VGICP_OK;
}
// one pass over the caller's strided array: validate, find the time range, pack contiguously into `packed`
static int timestamps_pack(vgicp_handle h, const char* who, const float* t, size_t n, size_t stride_bytes, std::vector<float>& packed, float* lo_out, float* hi_out) {
  packed.resize(n);
  const unsigned char* raw = reinterpret_cast<const unsigned char*>(t);
  float lo = 0.0f, hi = 0.0f;
  for (size_t i = 0; i < n; i++) {
    float v;
    memcpy(&v, raw + i * stride_bytes, sizeof(float));
    if (!std::isfinite(v)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, std::string(who) + ": non-finite timestamp");
    if (i == 0 || v < lo) lo = v;
    if (i == 0 || v > hi) hi = v;
    packed[i] = v;
  }
  *lo_out = lo;
  *hi_out = hi;
  return VGICP_OK;
}

// the twist as the kernel takes it (float) must be finite; checked before the timestamps are read
static int deskew_twist_check(vgicp_handle h, const char* who, const double twist[6]) {
  for (int j = 0; j < 6; j++)
    if (!std::isfinite((float)twist[j])) return fail(h, VGICP_ERR_INVALID_ARGUMENT, std::string(who) + ": non-finite twist");
  return VGICP_OK;
}

// Both deskews: the series bound in double against t_ref, then k_deskew_points over the source on its stream with the timestamps
// d_t (device memory, one float per point), ordered after the main stream's reads of the source points and after an append
static int deskew_enqueue(vgicp_handle h, const char* who, const float* d_t, const double twist[6], float lo, float hi, double t_ref) {
  Cloud& s = h->source;
  float xi[6];
  for (int j = 0; j < 6; j++) xi[j] = (float)twist[j];
  const double span = fmax(fabs((double)lo - t_ref), fabs((double)hi - t_ref));
  const double omega = sqrt(twist[0] * twist[0] + twist[1] * twist[1] + twist[2] * twist[2]);
  if (omega * span > 1.5707963267948966)
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, std::string(who) + ": the rotation over the sweep exceeds pi/2 (|omega| * max |t_i - t_ref|), beyond the series");
  if (s.st != h->stream.get()) {
    if (!h->ev_deskew) CU_TRY(h, event_create(h->ev_deskew, cudaEventDisableTiming));
    CU_TRY(h, cudaEventRecord(h->ev_deskew.get(), h->stream.get()));
    CU_TRY(h, cudaStreamWaitEvent(s.st, h->ev_deskew.get(), 0));
  }
  if (s.st != h->target.st) CU_TRY(h, cudaStreamWaitEvent(s.st, h->ev_append.get(), 0));
  KLAUNCH_ST(h, s.st, VGICP_PROF_OTHER,
             k_deskew_points<<<blocks_for(s.n, 256), 256, 0, s.st>>>(s.pts.p, d_t, s.n, (float)t_ref, xi[0], xi[1], xi[2], xi[3], xi[4], xi[5]));
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaEventRecord(s.ready.get(), s.st));
  points_changed(h, s, Change::moved);
  return VGICP_OK;
}

int vgicp_deskew_source(vgicp_handle h, const float* t, size_t n, size_t stride_bytes, const double twist[6], double t_ref) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (n > 0 && (!t || !twist)) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "deskew_source: null timestamps or twist");
  int rc = timestamps_check(h, "deskew_source", n, stride_bytes, t_ref);
  if (rc) return rc;
  if ((rc = deskew_twist_check(h, "deskew_source", twist))) return rc;
  std::vector<float>& packed = h->deskew_times;
  float lo = 0.0f, hi = 0.0f;
  if ((rc = timestamps_pack(h, "deskew_source", t, n, stride_bytes, packed, &lo, &hi))) return rc;
  Cloud& s = h->source;
  CU_TRY(h, s.staging.reserve(n * sizeof(float)));
  CU_TRY(h, cudaMemcpyAsync(s.staging.p, packed.data(), n * sizeof(float), cudaMemcpyHostToDevice, s.st));
  CU_TRY(h, cudaEventRecord(h->ev_copy.get(), s.st));
  rc = deskew_enqueue(h, "deskew_source", reinterpret_cast<const float*>(s.staging.p), twist, lo, hi, t_ref);
  // the packed timestamps are reused by the next call: the copy out of them must have landed
  CU_TRY(h, cudaEventSynchronize(h->ev_copy.get()));
  return rc;
}

// ---- continuous-time registration: the sweep's body twist estimated with the pose from per-point timestamps ----
int vgicp_set_source_timestamps(vgicp_handle h, const float* t, size_t n, size_t stride_bytes, double t_ref) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (n > 0 && !t) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_source_timestamps: null timestamps");
  int rc = timestamps_check(h, "set_source_timestamps", n, stride_bytes, t_ref);
  if (rc) return rc;
  std::vector<float> packed;
  float lo = 0.0f, hi = 0.0f;
  if ((rc = timestamps_pack(h, "set_source_timestamps", t, n, stride_bytes, packed, &lo, &hi))) return rc;
  return timestamps_commit(h, "set_source_timestamps", lo, hi, t_ref, [&]() -> int {
    CU_TRY(h, h->ct_times.reserve(n));
    CU_TRY(h, cudaMemcpyAsync(h->ct_times.p, packed.data(), n * sizeof(float), cudaMemcpyHostToDevice, h->stream.get()));
    CU_TRY(h, cudaStreamSynchronize(h->stream.get()));  // (`packed` goes out of scope)
    return VGICP_OK;
  });
}

// The same state from timestamps already in this GPU's memory: one kernel packs them into the spare buffer, counting the
// non-finite values and finding min and max in the same pass; one readback; the spare becomes ct_times only when every value passed
int vgicp_set_source_timestamps_device(vgicp_handle h, const float* d_t, size_t n, size_t stride_bytes, double t_ref) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (n > 0 && !d_t) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_source_timestamps_device: null timestamps");
  int rc = timestamps_check(h, "set_source_timestamps_device", n, stride_bytes, t_ref);
  if (rc) return rc;
  // after the source's pending work (a set_source_cloud_device read of the same buffer): the readback below then also tells the
  // caller that buffer is free
  const Cloud& s = h->source;
  if (s.st != h->stream.get() && s.ready) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), s.ready.get(), 0));
  CU_TRY(h, h->ct_spare.reserve(n));
  CU_TRY(h, h->ct_stats.reserve(3));
  CU_TRY(h, cudaMemsetAsync(h->ct_stats.p, 0, 3 * sizeof(unsigned), h->stream.get()));
  KLAUNCH(h, VGICP_PROF_OTHER,
          k_gather_times<<<blocks_for(n, 256), 256, 0, h->stream.get()>>>(reinterpret_cast<const unsigned char*>(d_t), stride_bytes, (int)n, h->ct_spare.p, h->ct_stats.p));
  CU_TRY(h, cudaGetLastError());
  unsigned st[3];
  CU_TRY(h, cudaMemcpyAsync(st, h->ct_stats.p, sizeof(st), cudaMemcpyDeviceToHost, h->stream.get()));
  CU_TRY(h, cudaStreamSynchronize(h->stream.get()));  // (the caller may reuse d_t after return)
  if (st[0]) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "set_source_timestamps_device: non-finite timestamp");
  auto from_key = [](unsigned k) {
    const unsigned b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    float v;
    memcpy(&v, &b, sizeof(v));
    return v;
  };
  // min and max are exact in any order (only the sign of a zero can differ from the host pass, which leaves every |t - tau| alike)
  return timestamps_commit(h, "set_source_timestamps_device", from_key(~st[1]), from_key(st[2]), t_ref, [&]() -> int {
    std::swap(h->ct_times, h->ct_spare);
    return VGICP_OK;
  });
}

// vgicp_deskew_source with the stored timestamps and t_ref: k_deskew_points reads ct_times, nothing is uploaded
int vgicp_deskew_source_stored(vgicp_handle h, const double twist[6]) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!twist) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "deskew_source_stored: null twist");
  if (!h->ct_has_times) return fail(h, VGICP_ERR_BAD_STATE, "deskew_source_stored: the source has no timestamps (vgicp_set_source_timestamps(_device))");
  int rc = deskew_twist_check(h, "deskew_source_stored", twist);
  if (!rc) rc = deskew_enqueue(h, "deskew_source_stored", h->ct_times.p, twist, h->ct_lo, h->ct_hi, h->ct_t_ref);
  if (rc) return rc;
  // the next write of the timestamp buffers (on the main stream) must not overtake this read of ct_times
  if (h->source.st != h->stream.get()) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), h->source.ready.get(), 0));
  return VGICP_OK;
}

int vgicp_compute_error_ct(vgicp_handle h, const double T_lin[16], const double xi_lin[6], const double T_eval[16], const double xi_eval[6], double* H144, double* b12,
                           double* err) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!T_lin || !xi_lin || !T_eval || !xi_eval || (H144 == nullptr) != (b12 == nullptr))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "compute_error_ct: null pose or twist, or H144 without b12 (or b12 without H144)");
  if (!all_finite(T_lin, 16, false) || !all_finite(T_eval, 16, false) || !all_finite(xi_lin, 6, true) || !all_finite(xi_eval, 6, true))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "compute_error_ct: non-finite pose or twist");
  int rc = check_ready(h, "compute_error_ct", kNeedEval | kNeedCt);
  if (rc) return rc;
  if (!twist_in_series(xi_lin, h->ct_span) || !twist_in_series(xi_eval, h->ct_span))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "compute_error_ct: the rotation over the sweep (|omega| * max |s_i|) exceeds pi/2, beyond the series");
  if ((rc = sync_inputs(h))) return rc;
  CU_TRY(h, h->ct.open(1, kCtStride, (size_t)kLinMaxBlocks * kCtStride, h->stream.get()));
  const bool want_H = H144 != nullptr;
  const double* raw = nullptr;
  if ((rc = ct_evaluate(h, T_lin, xi_lin, T_eval, xi_eval, want_H, &raw))) return rc;
  if (err) *err = raw[0];
  if (want_H) ct_system(raw, T_eval, H144, b12);
  return VGICP_OK;
}

// vgicp_align's state machine with N = 12: every evaluation looks the voxels up at (x0, tw0) and evaluates at (x0, tw0) (linearise)
// or at the trial (xi, twi) (error only); the prior is added on the host
int vgicp_align_ct(vgicp_handle h, const double guess[16], const double twist_guess[6], const double twist_prior[6], const double twist_weight[6],
                   const vgicp_lsq_params* params, vgicp_align_ct_result* res) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!guess || !twist_guess || !twist_prior || !twist_weight || !res) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_ct: null argument");
  if (!all_finite(guess, 16, false) || !all_finite(twist_guess, 6, true) || !all_finite(twist_prior, 6, false))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_ct: non-finite guess, twist guess or prior");
  for (int j = 0; j < 6; j++)
    if (!(twist_weight[j] > 0.0 && std::isfinite(twist_weight[j]))) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_ct: every twist weight must be finite and > 0");
  int rc = check_ready(h, "align_ct", kNeedEval | kNeedCt);
  if (rc) return rc;
  if (!twist_in_series(twist_guess, h->ct_span) || !twist_in_series(twist_prior, h->ct_span))
    return fail(h, VGICP_ERR_INVALID_ARGUMENT, "align_ct: the twist guess or prior rotates more than pi/2 over the sweep (|omega| * max |s_i|), beyond the series");
  const vgicp_lsq_params P = lsq_params(params);
  if ((rc = sync_inputs(h))) return rc;
  CU_TRY(h, h->ct.open(1, kCtStride, (size_t)kLinMaxBlocks * kCtStride, h->stream.get()));
  LmState<12> st = lm_init<12>(guess, P);
  memcpy(st.tw0, twist_guess, sizeof(st.tw0));
  st.span = h->ct_span;
  double rec[1 + 144 + 12];
  while (st.phase != kLmDone) {
    const bool lin = st.phase == kLmLinearize;
    const double* Te = lin ? st.x0.m : st.xi.m;
    const double* xe = lin ? st.tw0 : st.twi;
    const double* raw = nullptr;
    if ((rc = ct_evaluate(h, st.x0.m, st.tw0, Te, xe, lin, &raw))) return rc;
    double prior = 0.0;
    for (int j = 0; j < 6; j++) prior += twist_weight[j] * (xe[j] - twist_prior[j]) * (xe[j] - twist_prior[j]);
    rec[0] = raw[0] + prior;
    if (lin) {
      ct_system(raw, Te, rec + 1, rec + 145);
      for (int j = 0; j < 6; j++) {
        rec[1 + (6 + j) * 13] += twist_weight[j];
        rec[145 + 6 + j] += twist_weight[j] * (xe[j] - twist_prior[j]);
      }
    }
    lm_advance(&st, rec);
  }
  lm_result(st, res);
  memcpy(res->twist, st.tw0, sizeof(res->twist));
  return VGICP_OK;
}

// ---- multi-GPU: source sharding with an in-kernel exchange of the linear system over NVLink peer memory ----
int vgicp_comm_export(vgicp_handle h, unsigned char* handle64) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!handle64) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "comm_export: null buffer");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  if (!h->comm_box) {
    CU_TRY(h, device_alloc(h->comm_box, sizeof(CommMailbox)));
    CU_TRY(h, cudaMemset(h->comm_box.get(), 0, sizeof(CommMailbox)));
  }
  cudaIpcMemHandle_t ipc;
  CU_TRY(h, cudaIpcGetMemHandle(&ipc, h->comm_box.get()));
  memcpy(handle64, &ipc, 64);
  return VGICP_OK;
}

int vgicp_comm_init(vgicp_handle h, int rank, int nranks, const unsigned char* all_handles) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (nranks < 1 || nranks > kCommMaxRanks || rank < 0 || rank >= nranks || !all_handles) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "comm_init: need 1 <= nranks <= 8 and all handles");
  if (!h->comm_box) return fail(h, VGICP_ERR_BAD_STATE, "comm_init: call vgicp_comm_export first");
  IpcPtr<CommMailbox> peers[kCommMaxRanks];  // (closed again if a later rank fails)
  for (int r = 0; r < nranks; r++) {
    if (r == rank) continue;
    cudaIpcMemHandle_t ipc;
    memcpy(&ipc, all_handles + (size_t)r * 64, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail(h, VGICP_ERR_COMM, std::string("comm_init: cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
    peers[r].reset(static_cast<CommMailbox*>(p));
  }
  for (int r = 0; r < kCommMaxRanks; r++) h->comm_peers[r] = std::move(peers[r]);
  h->comm_rank = rank;
  h->comm_ranks = nranks;
  h->comm_seq = 0;
  // the mailbox outlives vgicp_comm_shutdown: flags left by a previous session could equal the first tags of this one.  Clear it
  // here; the caller puts a host barrier between vgicp_comm_init on all ranks and the first evaluation (see the header), so no
  // peer writes into it before the clear has landed.
  CU_TRY(h, cudaMemsetAsync(h->comm_box.get(), 0, sizeof(CommMailbox), h->stream.get()));
  CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
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
    CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
    CU_TRY(h, cudaStreamSynchronize(h->stream_b.get()));
    const size_t bytes = kCommArenaHeaderBytes + 2 * max_points * 24 + 64;  // (+ padding: bulk copies read covB in 16-byte units)
    CU_TRY(h, device_alloc(h->arena, bytes));
    CU_TRY(h, cudaMemset(h->arena.get(), 0, bytes));
    h->arena_points = max_points;
    // the covariance arrays of both clouds now live in the arena (previous covariances are dropped)
    Cloud* cl[2] = {&h->target, &h->source};
    for (int j = 0; j < 2; j++) {
      unsigned char* base = h->arena.get() + kCommArenaHeaderBytes + (size_t)j * max_points * 24;
      cl[j]->covA.attach(reinterpret_cast<float4*>(base), max_points);
      cl[j]->covB.attach(reinterpret_cast<float2*>(base + max_points * 16), max_points);
      cl[j]->arena_slot = j;
      cl[j]->arena_seq = 0;
    }
    covariances_dropped(h);
  }
  cudaIpcMemHandle_t ipc;
  CU_TRY(h, cudaIpcGetMemHandle(&ipc, h->arena.get()));
  memcpy(handle64, &ipc, 64);
  return VGICP_OK;
}

int vgicp_comm_init_arena(vgicp_handle h, const unsigned char* all_handles) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!all_handles) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "comm_init_arena: null handles");
  if (h->comm_ranks < 1 || !h->arena) return fail(h, VGICP_ERR_BAD_STATE, "comm_init_arena: call vgicp_comm_init and vgicp_comm_export_arena first");
  IpcPtr<unsigned char[]> peers[kCommMaxRanks];  // (closed again if a later rank fails)
  for (int r = 0; r < h->comm_ranks; r++) {
    if (r == h->comm_rank) continue;
    cudaIpcMemHandle_t ipc;
    memcpy(&ipc, all_handles + (size_t)r * 64, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail(h, VGICP_ERR_COMM, std::string("comm_init_arena: cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
    peers[r].reset(static_cast<unsigned char*>(p));
  }
  for (int r = 0; r < kCommMaxRanks; r++) h->arena_peers[r] = std::move(peers[r]);
  h->arena_mapped = true;
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
  if (h->stream) cudaStreamSynchronize(h->stream.get());
  if (h->stream_b) cudaStreamSynchronize(h->stream_b.get());
  for (auto& p : h->arena_peers) p.reset();
  for (auto& p : h->comm_peers) p.reset();
  h->arena_mapped = false;
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
    CU_TRY(h, cudaMemcpy(&tmp, h->comm_box.get(), sizeof(CommMailbox), cudaMemcpyDeviceToHost));
    *error = tmp.error;
  }
  if (h->arena) {
    CommArenaHeader hdr;
    CU_TRY(h, cudaMemcpy(&hdr, h->arena.get(), sizeof(hdr), cudaMemcpyDeviceToHost));
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
  problem_set(h, problem);
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
  CU_TRY(h, cudaStreamSynchronize(h->stream_b.get()));
  CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
  for (auto& r : h->prof_pending) { h->prof_pool.push_back(std::move(r.a)); h->prof_pool.push_back(std::move(r.b)); }
  h->prof_pending.clear();
  for (int i = 0; i < VGICP_PROF_NUM_CATEGORIES; i++) { h->prof_ms[i] = 0.0; h->prof_launches[i] = 0; }
  h->prof_on = enable != 0;
  return VGICP_OK;
}

int vgicp_get_profile(vgicp_handle h, double* ms, uint64_t* launches, int capacity) {
  CHECK_HANDLE(h);
  DeviceGuard g(h->device);
  if (!ms || !launches || capacity < VGICP_PROF_NUM_CATEGORIES) return fail(h, VGICP_ERR_INVALID_ARGUMENT, "get_profile: need VGICP_PROF_NUM_CATEGORIES entries");
  CU_TRY(h, cudaStreamSynchronize(h->stream_b.get()));
  CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
  for (auto& r : h->prof_pending) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, r.a.get(), r.b.get()) == cudaSuccess) h->prof_ms[r.cat] += (double)t;
    h->prof_pool.push_back(std::move(r.a));
    h->prof_pool.push_back(std::move(r.b));
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
  if (h->source.st != h->stream.get()) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), h->source.ready.get(), 0));
  if (h->target.st != h->stream.get()) CU_TRY(h, cudaStreamWaitEvent(h->stream.get(), h->target.ready.get(), 0));
  CU_TRY(h, h->staging.reserve((size_t)n * sizeof(float)));
  float* d_out = reinterpret_cast<float*>(h->staging.p);
  KLAUNCH(h, VGICP_PROF_OTHER, k_nn1_sqdist<<<blocks_for(n, 256), 256, 0, h->stream.get()>>>(h->source.pts.p, n, h->target.pts.p, h->target.n, to_pose(T), d_out));
  CU_TRY(h, cudaGetLastError());
  std::vector<float> d2(n);
  CU_TRY(h, cudaMemcpyAsync(d2.data(), d_out, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, h->stream.get()));
  CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
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
  CU_TRY(h, cudaStreamSynchronize(h->stream_b.get()));
  CU_TRY(h, cudaStreamSynchronize(h->stream.get()));
  return VGICP_OK;
}

int vgicp_get_stream(vgicp_handle h, uint64_t* stream) {
  CHECK_HANDLE(h);
  if (!stream) return VGICP_ERR_INVALID_ARGUMENT;
  *stream = (uint64_t)(uintptr_t)h->stream.get();
  return VGICP_OK;
}

}  // extern "C"
