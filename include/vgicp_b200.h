/*
 * vgicp_b200.h -- C ABI of libvgicp_b200.so, the H100 (sm_90a) VGICP registration core.
 *
 * This is the drop-in seam for fast_gicp's device core: every function below replaces one member of
 * fast_gicp::cuda::FastVGICPCudaCore (reference include/fast_gicp/cuda/fast_vgicp_cuda.cuh:28-92, implemented in
 * src/fast_gicp/cuda/fast_vgicp_cuda.cu:18-284) and is called from exactly the places
 * include/fast_gicp/gicp/impl/fast_vgicp_cuda_impl.hpp calls that member.  Plain pointers and sizes only: no
 * Eigen, thrust, PCL or torch types cross this boundary.
 *
 * Conventions
 *   - every call returns a vgicp_status (0 = OK); it never throws, asserts or aborts (the reference asserts /
 *     abort()s, fast_vgicp_cuda.cu:46-48,128,139,...).  vgicp_last_error() gives the message of the last failure.
 *   - one handle <-> one FastVGICPCudaCore: owns one CUDA stream and all device buffers; calls on one handle are
 *     stream-ordered; a handle must not be used from two host threads at once (same as the reference).
 *   - clouds: float32 xyz, `stride_bytes` between consecutive points (12 for packed Eigen::Vector3f, 16 for
 *     pcl::PointXYZ, 32 for pcl::PointXYZI ...).  Inputs are copied; the caller keeps ownership.
 *   - poses: 16 doubles, column-major 4x4 == Eigen::Isometry3d::data().
 *   - 3x3 matrices returned to the host: 9 floats column-major == Eigen::Matrix3f::data() (36 B), as in the
 *     reference's get_*_covariances / get_voxel_covs.
 *   - H: 36 doubles column-major 6x6 == Eigen::Matrix<double,6,6>::data(); b: 6 doubles.
 *   - enums are passed as int with the reference's numeric order (include/fast_gicp/gicp/gicp_settings.hpp:6-10).
 */
#ifndef VGICP_B200_H
#define VGICP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define VGICP_API __attribute__((visibility("default")))
#else
#define VGICP_API
#endif

typedef struct vgicp_context* vgicp_handle;

typedef enum {
  VGICP_OK = 0,
  VGICP_ERR_INVALID_ARGUMENT = 1, /* null pointer, bad enum, k out of range, size mismatch */
  VGICP_ERR_BAD_STATE = 2,        /* a prerequisite call is missing (e.g. covariances before the cloud) */
  VGICP_ERR_CUDA = 3,             /* a CUDA runtime call failed; message has the cudaError string */
  VGICP_ERR_UNSUPPORTED = 4,      /* regularisation method not implemented on the GPU path (as in the reference) */
  VGICP_ERR_NO_DEVICE = 5,        /* no CUDA device / kernel image not loadable on this GPU (needs sm_90a) */
  VGICP_ERR_COMM = 6              /* multi-GPU exchange failed */
} vgicp_status;

/* fast_gicp::RegularizationMethod, gicp_settings.hpp:6 */
enum { VGICP_REG_NONE = 0, VGICP_REG_MIN_EIG = 1, VGICP_REG_NORMALIZED_MIN_EIG = 2, VGICP_REG_PLANE = 3, VGICP_REG_FROBENIUS = 4 };
/* fast_gicp::NeighborSearchMethod, gicp_settings.hpp:8 */
enum { VGICP_DIRECT27 = 0, VGICP_DIRECT7 = 1, VGICP_DIRECT1 = 2, VGICP_DIRECT_RADIUS = 3 };

/* ---- lifetime ------------------------------------------------------------------------------------------------ */
/* FastVGICPCudaCore::FastVGICPCudaCore()  fast_vgicp_cuda.cu:18-30.  `device` = CUDA ordinal (the reference uses the
 * current device); defaults installed: resolution 1.0, kernel_width 0.25, kernel_max_dist 3.0, offsets = DIRECT1. */
VGICP_API int vgicp_create(int device, vgicp_handle* out);
VGICP_API int vgicp_destroy(vgicp_handle h);
VGICP_API const char* vgicp_last_error(vgicp_handle h); /* valid until the next call on h; "" if none */
VGICP_API const char* vgicp_version(void);

/* ---- settings ------------------------------------------------------------------------------------------------ */
VGICP_API int vgicp_set_resolution(vgicp_handle h, double resolution);                              /* :32-34 */
VGICP_API int vgicp_set_kernel_params(vgicp_handle h, double kernel_width, double kernel_max_dist); /* :36-39 */
VGICP_API int vgicp_set_neighbor_search_method(vgicp_handle h, int method, double radius);          /* :41-95 */

/* ---- clouds -------------------------------------------------------------------------------------------------- */
VGICP_API int vgicp_set_source_cloud(vgicp_handle h, const float* xyz, size_t n, size_t stride_bytes); /* :109-116 */
VGICP_API int vgicp_set_target_cloud(vgicp_handle h, const float* xyz, size_t n, size_t stride_bytes); /* :118-125 */
VGICP_API int vgicp_swap_source_and_target(vgicp_handle h); /* :97-107: swaps points/neighbours/covariances and, when the
                                                               new target has covariances, rebuilds the voxel map */

/* ---- stage 1: neighbours + covariances ----------------------------------------------------------------------- */
/* set_{source,target}_neighbors :127-147 -- host-computed k-NN indices, row i = neighbours of point i; n_times_k must
 * equal k * cloud size (the reference asserts it). */
VGICP_API int vgicp_set_source_neighbors(vgicp_handle h, int k, const int* indices, size_t n_times_k);
VGICP_API int vgicp_set_target_neighbors(vgicp_handle h, int k, const int* indices, size_t n_times_k);
/* find_{source,target}_neighbors :155-181 -- exact k-NN of every point within its own cloud (self included) on the GPU.
 * Rows come out ascending in (squared distance, index) -- the kd-tree order; the reference's brute-force mode leaves heap
 * order, same set.  1 <= k <= min(n, 64). */
VGICP_API int vgicp_find_source_neighbors(vgicp_handle h, int k);
VGICP_API int vgicp_find_target_neighbors(vgicp_handle h, int k);
/* calculate_{source,target}_covariances :183-203 -- covariance_estimation + covariance_regularization(method).
 * NONE leaves the raw covariance; NORMALIZED_MIN_EIG is not implemented on the reference's GPU path (it prints an error and
 * leaves the raw covariance): same here, with VGICP_ERR_UNSUPPORTED returned after the raw covariances are in place. */
VGICP_API int vgicp_calculate_source_covariances(vgicp_handle h, int regularization_method);
VGICP_API int vgicp_calculate_target_covariances(vgicp_handle h, int regularization_method);
/* calculate_{source,target}_covariances_rbf :205-219 -- kernel-weighted covariances, w = exp(-kernel_width * d^2), d <= max_dist */
VGICP_API int vgicp_calculate_source_covariances_rbf(vgicp_handle h, int regularization_method);
VGICP_API int vgicp_calculate_target_covariances_rbf(vgicp_handle h, int regularization_method);
/* get_{source,target}_covariances :245-255 -- out9: n x 9 floats */
VGICP_API int vgicp_get_source_covariances(vgicp_handle h, float* out9, size_t capacity_points);
VGICP_API int vgicp_get_target_covariances(vgicp_handle h, float* out9, size_t capacity_points);
/* Caller-supplied covariances instead of the k-NN ones: the CUDA counterpart of FastGICP::setSourceCovariances /
 * setTargetCovariances (include/fast_gicp/gicp/fast_gicp.hpp:60-62, CPU classes only in the reference): in9 = n x 9 floats,
 * column-major 3x3 per point (the layout get_*_covariances returns); the symmetric part is stored.  n must equal the cloud size. */
VGICP_API int vgicp_set_source_covariances(vgicp_handle h, const float* in9, size_t n_points);
VGICP_API int vgicp_set_target_covariances(vgicp_handle h, const float* in9, size_t n_points);
/* public members source_neighbors / target_neighbors (fast_vgicp_cuda.cuh:80-81) read back: n x k ints */
VGICP_API int vgicp_get_source_neighbors(vgicp_handle h, int* out, size_t capacity_ints, int* k_out);
VGICP_API int vgicp_get_target_neighbors(vgicp_handle h, int* out, size_t capacity_ints, int* k_out);
VGICP_API int vgicp_get_num_source_points(vgicp_handle h, size_t* n);
VGICP_API int vgicp_get_num_target_points(vgicp_handle h, size_t* n);

/* ---- stage 2: Gaussian voxel map ----------------------------------------------------------------------------- */
/* create_target_voxelmap :257-263 (GaussianVoxelMap::create_voxelmap(points, covs), gaussian_voxelmap.cu:233-289).
 * As in the reference the map object keeps the resolution it was first created with (SURVEY Q3). */
VGICP_API int vgicp_create_target_voxelmap(vgicp_handle h);
VGICP_API int vgicp_get_num_voxels(vgicp_handle h, int* num_voxels);   /* voxelmap_info.num_voxels */
VGICP_API int vgicp_get_num_buckets(vgicp_handle h, int* num_buckets); /* voxelmap_info.num_buckets */
VGICP_API int vgicp_get_voxel_num_points(vgicp_handle h, int* out, size_t capacity_voxels); /* :227-231 */
VGICP_API int vgicp_get_voxel_means(vgicp_handle h, float* out3, size_t capacity_voxels);   /* :233-237 */
VGICP_API int vgicp_get_voxel_covs(vgicp_handle h, float* out9, size_t capacity_voxels);    /* :239-243 */
/* public member voxelmap->buckets (gaussian_voxelmap.cuh:32): per bucket {coord xyz, voxel id}; empty = {0,0,0,-1} */
VGICP_API int vgicp_get_voxel_buckets(vgicp_handle h, int* coords3, int* ids, size_t capacity_buckets);

/* ---- stage 2b + 3: correspondences and the linear system ----------------------------------------------------- */
/* update_correspondences :265-274 -- fixes the linearisation pose (cast to float like the reference). */
VGICP_API int vgicp_update_correspondences(vgicp_handle h, const double T[16]);
/* get_voxel_correspondences :221-225 -- (source index, voxel id) pairs, offset-major / point-minor like the reference's list.
 * Pass pairs=NULL to query the count. */
VGICP_API int vgicp_get_voxel_correspondences(vgicp_handle h, int* pairs, size_t capacity_pairs, size_t* n_pairs);
/* compute_error :276-284 -> compute_derivatives (compute_derivatives.cu:151-184).  H36 and b6 may both be NULL
 * (error only).  *err receives the return value of the reference's compute_error. */
VGICP_API int vgicp_compute_error(vgicp_handle h, const double T[16], double* H36, double* b6, double* err);

/* ---- extensions (not in the reference core) ------------------------------------------------------------------ */
/* LsqRegistration defaults, include/fast_gicp/gicp/impl/lsq_registration_impl.hpp:9-22 */
typedef struct {
  int max_iterations;            /* 64 */
  double rotation_epsilon;       /* 2e-3 */
  double transformation_epsilon; /* 5e-4 */
  int use_gauss_newton;          /* 0: Levenberg-Marquardt (default), 1: Gauss-Newton */
  int lm_max_iterations;         /* 10 */
  double lm_init_lambda_factor;  /* 1e-9 */
} vgicp_lsq_params;

typedef struct {
  double T[16];        /* final pose x0 (double, before the reference's cast to float) */
  double H[36];        /* final_hessian_ */
  int nr_iterations;   /* nr_iterations_ */
  int converged;       /* converged_ */
  int n_linearize;     /* evaluations with H,b */
  int n_compute_error; /* error-only evaluations */
  int lm_failed;       /* 1 when the reference would print "lm not converged!!" */
} vgicp_align_result;

VGICP_API void vgicp_lsq_default_params(vgicp_lsq_params* p);
/* Whole LsqRegistration::computeTransformation loop (lsq_registration_impl.hpp:53-79,106-168) inside the library: the same
 * linearize / compute_error evaluations and the same LM / GN logic in double, without crossing the ABI once per evaluation.
 * Driven from the host by default (one 344-byte result per evaluation through mapped memory); vgicp_set_align_mode selects the
 * device-resident state machine, vgicp_set_speculation the fused trial evaluation.  result->T = final_transformation_. */
VGICP_API int vgicp_align(vgicp_handle h, const double guess[16], const vgicp_lsq_params* params, vgicp_align_result* result);
/* One whole registration: clearTarget/clearSource + setInputTarget + setInputSource + align (the body of the reference's
 * benchmark loop, src/align.cpp:72-81) with GPU k-NN covariances.  xyz are host pointers, or device pointers when on_device != 0. */
VGICP_API int vgicp_register(vgicp_handle h, const float* target_xyz, size_t n_target, const float* source_xyz, size_t n_source, size_t stride_bytes, int on_device, int k,
                             int regularization_method, const double guess[16], const vgicp_lsq_params* params, vgicp_align_result* result);
/* pcl::transformPointCloud of the source by T (lsq_registration_impl.hpp:78) on the device; out: n x stride floats */
VGICP_API int vgicp_transform_source(vgicp_handle h, const double T[16], float* out_xyz, size_t capacity_points, size_t stride_bytes);
/* set_{source,target}_cloud with the points already resident in this GPU's memory (device pointer, same layout rules);
 * the read is stream-ordered on the handle's stream, the caller keeps the buffer alive until the next synchronising call */
VGICP_API int vgicp_set_source_cloud_device(vgicp_handle h, const float* d_xyz, size_t n, size_t stride_bytes);
VGICP_API int vgicp_set_target_cloud_device(vgicp_handle h, const float* d_xyz, size_t n, size_t stride_bytes);
/* ---- multi-GPU source sharding (SURVEY.md 8e; not in the reference, which is single-GPU) --------------------------------
 * Every rank (one process per GPU) holds the whole target and voxel map and evaluates only a slice of the source
 * (vgicp_set_source_shard); the last block of each evaluation kernel stores its 28 folded sums into every peer's mailbox over
 * NVLink peer memory, waits for the peers' sums and adds them in rank order, so vgicp_compute_error / vgicp_align return the
 * same H, b, err on every rank.  Setup: each rank calls vgicp_comm_export, the 64-byte handles are all-gathered by any host
 * transport (torch.distributed, MPI, files), then vgicp_comm_init (which clears this rank's mailbox), then a host barrier over all
 * ranks before the first evaluation.  Ranks must issue the same sequence of evaluations.  An evaluation whose wait for a peer times
 * out returns VGICP_ERR_COMM (the sums are incomplete); vgicp_comm_error reads the sticky flag. */
VGICP_API int vgicp_comm_export(vgicp_handle h, unsigned char* handle64);
VGICP_API int vgicp_comm_init(vgicp_handle h, int rank, int nranks, const unsigned char* all_handles /* nranks x 64 bytes */);
VGICP_API int vgicp_comm_shutdown(vgicp_handle h);
VGICP_API int vgicp_comm_error(vgicp_handle h, int* error);  /* 1 when a wait for a peer timed out */
VGICP_API int vgicp_set_source_shard(vgicp_handle h, size_t begin, size_t end);  /* evaluations cover source points [begin, end) */
/* Stage 1 sharded as well (k-NN queries + covariances, SURVEY.md 8e): every rank builds the k-NN grid of the whole cloud but searches
 * only its 1/nranks slice of the queries, computes the covariances of that slice and stores them straight into the covariance arrays
 * of EVERY rank (peer stores over NVLink from inside the covariance kernel); a one-block kernel then tells the peers and waits for
 * their slices, in stream order.  For that the covariance arrays of both clouds live in an IPC-exported arena of fixed capacity:
 * vgicp_comm_export_arena(max_points) after vgicp_comm_init, all-gather the 64-byte handles, vgicp_comm_init_arena, host barrier,
 * vgicp_set_stage1_sharding(1).  All ranks must then make the same sequence of set_*_cloud / find_*_neighbors /
 * calculate_*_covariances / swap calls.  get_*_neighbors returns this rank's rows only; the covariances are complete everywhere. */
VGICP_API int vgicp_comm_export_arena(vgicp_handle h, size_t max_points, unsigned char* handle64);
VGICP_API int vgicp_comm_init_arena(vgicp_handle h, const unsigned char* all_handles /* nranks x 64 bytes */);
VGICP_API int vgicp_set_stage1_sharding(vgicp_handle h, int enable);
VGICP_API int vgicp_clear_source_shard(vgicp_handle h);
/* ---- NDT (next-tier component: fast_gicp::cuda::NDTCudaCore, include/fast_gicp/cuda/ndt_cuda.cuh:28-68, src/fast_gicp/cuda/ndt_cuda.cu) ----
 * The same handle solves the NDT problems: vgicp_set_problem selects VGICP (0, default), NDT point-to-distribution (1) or NDT
 * distribution-to-distribution (2; NDTDistanceMode order P2D, D2D of ndt_settings.hpp:6, plus one).  With an NDT problem selected
 *   set_{source,target}_cloud, set_resolution, set_neighbor_search_method, swap_source_and_target   as NDTCudaCore's members (:36-48)
 *   vgicp_ndt_create_voxelmaps      NDTCudaCore::create_voxelmaps (ndt_cuda.cu:118-141): points-only voxel Gaussians + MIN_EIG; a map
 *                                   that exists is kept with the resolution it was built with (set_*_cloud resets that cloud's map,
 *                                   swap_source_and_target swaps the two maps), exactly as the reference's early returns (:125,136)
 *   vgicp_update_correspondences    NDTCudaCore::update_correspondences (:143-162): source points (P2D) or source voxel means (D2D)
 *   vgicp_compute_error / vgicp_align   NDTCudaCore::compute_error (:164-177) -> {p2d,d2d}_ndt_compute_derivatives
 *   vgicp_get_voxel_* / vgicp_get_num_voxels / vgicp_get_voxel_buckets   read the NDT target map
 * No kNN and no per-point covariances are involved (the reference's NDTCuda never computes them). */
VGICP_API int vgicp_set_problem(vgicp_handle h, int problem);
VGICP_API int vgicp_ndt_create_voxelmaps(vgicp_handle h);
/* Execution hint: 0 = latency (default: the persistent k-NN kernel takes 4 blocks per SM; every evaluation writes its 43 doubles
 * straight into mapped host memory and the calling thread spins on a completion word), 1 = throughput / polite (2 k-NN blocks per SM;
 * evaluations are read back with a copy and a stream wait, so the host thread sleeps instead of spinning).  Results are identical.
 * bench.py uses the latency shape. */
VGICP_API int vgicp_set_execution_hint(vgicp_handle h, int hint);
/* vgicp_align driver: 1 = host-driven loop over the evaluation kernels (default; one 344-byte readback per evaluation, like
 * the reference), 0 = device-resident loop (the LM state machine runs in the last block of each evaluation kernel, the host
 * reads one state block back per chunk of launches).  Both walk the same iterates; the serial double-precision LM step
 * on one GPU thread costs about what the host round trip saves, so the host-driven loop stays the default. */
VGICP_API int vgicp_set_align_mode(vgicp_handle h, int mode);
/* k-NN engine used by find_*_neighbors: 0 = multi-level hash grid (default), 1 = warp-cooperative scan of the whole cloud,
 * 2 = one-thread-per-query scan (the shape of the reference's brute_force_knn.cu).  All three return identical rows. */
VGICP_API int vgicp_set_knn_mode(vgicp_handle h, int mode);
/* Voxel lookup structure used by the evaluation kernels (update_correspondences + compute_derivatives fused): 0 = a direct-mapped
 * cell -> voxel-id array over the bounding box of the target's voxel coordinates, built next to the hash table whenever that box
 * has at most 16 Mi cells (default; any LiDAR-like cloud), 1 = always probe the reference-layout hash table
 * (gaussian_voxelmap.cu:12-73 / find_voxel_correspondences.cu:32-60).  Both return the same voxel ids: a table lookup answers
 * "is this coordinate a voxel of the map, and which", and the map's set of voxels (including the reference's drop rule for
 * voxels that fall off the 10-probe window) is decided by the table build alone. */
VGICP_API int vgicp_set_voxel_index(vgicp_handle h, int mode);
/* vgicp_align, Levenberg-Marquardt: 1 (default) = each trial evaluation (compute_error at x0*delta, lsq_registration_impl.hpp:141)
 * also linearises at the trial pose in the same launch, so that the next iteration of an accepted step
 * (update_correspondences + compute_error(H, b), fast_vgicp_cuda_impl.hpp:170-173) is already there: ~6 instead of ~9 launches
 * and host round trips per registration; a rejected trial discards it.  0 = one launch per evaluation, as the reference.
 * The iterates, the result and the n_linearize / n_compute_error counters are identical either way. */
VGICP_API int vgicp_set_speculation(vgicp_handle h, int enable);
/* per-kernel timing with CUDA events on the handle's stream (off by default; enabling resets the counters) */
enum {
  VGICP_PROF_UNPACK = 0, VGICP_PROF_KNN = 1, VGICP_PROF_COVARIANCE = 2, VGICP_PROF_VOXELMAP = 3, VGICP_PROF_LINEARIZE = 4, VGICP_PROF_ERROR = 5,
  VGICP_PROF_OTHER = 6, VGICP_PROF_NUM_CATEGORIES = 7
};
VGICP_API int vgicp_set_profiling(vgicp_handle h, int enable);
VGICP_API int vgicp_get_profile(vgicp_handle h, double* ms_per_category, uint64_t* launches_per_category, int capacity);
VGICP_API const char* vgicp_profile_category_name(int category);
/* pcl::Registration::getFitnessScore(max_range) for the current source/target under T (used by src/align.cpp:67 and pygicp's
 * get_fitness_score, src/python/main.cpp:158): mean squared nearest-neighbour distance over pairs with d^2 <= max_range;
 * DBL_MAX when no pair qualifies. */
VGICP_API int vgicp_get_fitness_score(vgicp_handle h, const double T[16], double max_range, double* score);
/* number of kernels this handle has launched since creation (bench.py's gpu_launches) */
VGICP_API int vgicp_get_launch_count(vgicp_handle h, uint64_t* launches);
VGICP_API int vgicp_synchronize(vgicp_handle h);
/* cudaStream_t of the handle as an integer, for CUDA-event timing on the launching stream */
VGICP_API int vgicp_get_stream(vgicp_handle h, uint64_t* stream);

#ifdef __cplusplus
}
#endif
#endif /* VGICP_B200_H */
