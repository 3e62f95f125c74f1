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
 * Driven from the host (one 344-byte result per evaluation through mapped memory); vgicp_set_speculation selects the fused trial
 * evaluation.  result->T = final_transformation_. */
VGICP_API int vgicp_align(vgicp_handle h, const double guess[16], const vgicp_lsq_params* params, vgicp_align_result* result);
/* ---- multi-hypothesis alignment (global localisation, relocalisation, loop-closure checks) ----------------------------------
 * B registrations of the current source against the current target map, from B initial guesses (B x 16 doubles, column-major),
 * with the evaluations of all still-running hypotheses in shared launches: one evaluation kernel per optimiser round and kind
 * (with LM and speculation, one launch per round; with GN, one linearisation launch per round), each hypothesis a row of blocks
 * with the single-pose launch's grid, so its sums are the single-pose sums.  results[i] equals vgicp_align(h, guesses + 16 i,
 * params) bit for bit (T, H, nr_iterations, converged, n_linearize, n_compute_error, lm_failed), under either execution hint and
 * speculation setting: both calls run the same optimiser state machine on the host.  1 <= n_guesses <= 4096.
 * The handle's linearisation point and the rest of its single-pose state are left as they were.  Working memory: 256 bytes per
 * evaluation block and hypothesis (about 0.1 MB per hypothesis at 17 k points, 0.27 MB at 1 M points with DIRECT1), grow-only.
 * Errors: VGICP_ERR_INVALID_ARGUMENT (null pointer, n_guesses out of range), VGICP_ERR_BAD_STATE (the preconditions of
 * vgicp_align), VGICP_ERR_UNSUPPORTED (handle in a multi-GPU communicator); none of them launches a kernel. */
VGICP_API int vgicp_align_multi(vgicp_handle h, const double* guesses, int n_guesses, const vgicp_lsq_params* params, vgicp_align_result* results);
/* B poses scored in one launch: err[i] (and H36 + 36 i, b6 + 6 i when H36 and b6 are not NULL; both or neither) equal
 * vgicp_update_correspondences(T_i) + vgicp_compute_error(T_i) bit for bit; n_corr[i] (optional) is the number of (source point,
 * voxel) correspondences at T_i, the count vgicp_get_voxel_correspondences reports.  A pose without overlap has err 0 and no
 * correspondences, so rank hypotheses by err normalised with n_corr, not by err alone.  Handle state unchanged; 1 <= n_poses <= 4096;
 * errors as vgicp_align_multi. */
VGICP_API int vgicp_evaluate_poses(vgicp_handle h, const double* T, int n_poses, double* err, double* H36, double* b6, int64_t* n_corr);
/* ---- multi-source alignment (multi-LiDAR rigs, keyframes against one submap, a recorded log against a prebuilt map) ----------
 * B source clouds registered against the current target map in one call.  Source i is xyz[i] with n[i] points, stride_bytes apart
 * (one stride for all), host pointers or device pointers when on_device != 0; guesses: B x 16 doubles (column-major), NULL = the
 * identity for every source.  Stage 1 runs source by source on the library's k-NN and covariance kernels (k neighbours,
 * regularization_method); the optimisers of all sources then share their evaluation launches, as in vgicp_align_multi: each round
 * groups the running sources by launch class (streaming or compacted kernel, lanes per point; sources of different sizes can fall in
 * different classes, e.g. DIRECT1 streams from 65 536 points with the direct index) and issues one launch per class and evaluation
 * kind, each source a row of blocks with the grid of its own single-pose launch.
 * results[i] equals, bit for bit (T, H, nr_iterations, converged, n_linearize, n_compute_error, lm_failed), what the same handle
 * returns for vgicp_set_source_cloud(xyz[i], n[i], stride_bytes) (or _device) + vgicp_find_source_neighbors(k) +
 * vgicp_calculate_source_covariances(regularization_method) + vgicp_align(guesses + 16 i, params), under either execution hint and
 * speculation setting, with every neighbour search, voxel index and robust kind.  NORMALIZED_MIN_EIG behaves as in vgicp_register:
 * the raw covariances are used and the call registers.
 * The handle's own source (points, neighbour rows, covariances, timestamps), its linearisation point and the rest of its
 * single-pose state are left as they were; so are the target and its map.  1 <= n_sources <= 4096, 1 <= k <= min(n[i], 64).
 * Working memory, grow-only: the sources live in one pool of about 40 bytes per point (float4 point, float4 + float2 covariance);
 * neighbour rows are not kept (one table of the largest source's rows is reused), plus vgicp_align_multi's 256 bytes per evaluation
 * block and source.
 * Errors, every one returned before anything is launched or modified: VGICP_ERR_INVALID_ARGUMENT (null handle or pointer, n_sources
 * out of range, a bad k, size, stride or regularization method), VGICP_ERR_BAD_STATE (no target voxel map), VGICP_ERR_UNSUPPORTED
 * (an NDT problem, source or stage-1 sharding, a multi-GPU communicator). */
VGICP_API int vgicp_align_sources(vgicp_handle h, const float* const* xyz, const size_t* n, size_t stride_bytes, int on_device, int k, int regularization_method,
                                  const double* guesses /* B x 16, NULL = identity */, int n_sources, const vgicp_lsq_params* params, vgicp_align_result* results);
/* One whole registration: clearTarget/clearSource + setInputTarget + setInputSource + align (the body of the reference's
 * benchmark loop, src/align.cpp:72-81) with GPU k-NN covariances.  xyz are host pointers, or device pointers when on_device != 0. */
VGICP_API int vgicp_register(vgicp_handle h, const float* target_xyz, size_t n_target, const float* source_xyz, size_t n_source, size_t stride_bytes, int on_device, int k,
                             int regularization_method, const double guess[16], const vgicp_lsq_params* params, vgicp_align_result* result);
/* ---- robust kernels (outlier down-weighting; not in the reference) -------------------------------------------------------
 * Per correspondence (source point i, voxel v) at the evaluation pose, with e = mu_v - T a_i, M = (C_v + R C_i R^T)^-1 as always
 * and s = e^T M e (squared Mahalanobis residual):
 *   err += sqrt(n_v) rho(s),   H += sqrt(n_v) rho'(s) J^T M J,   b += sqrt(n_v) rho'(s) J^T M e
 * (iteratively reweighted least squares: the rho'' term is dropped; b is half the gradient of err at fixed correspondences).
 *   kind            rho(s)                                          rho'(s)
 *   NONE (default)  s                                               1
 *   HUBER           s if s <= d^2, else 2 d sqrt(s) - d^2           1 if s <= d^2, else d / sqrt(s)
 *   CAUCHY          d^2 ln(1 + s / d^2)                             d^2 / (d^2 + s)
 *   GEMAN_MCCLURE   d^2 s / (d^2 + s)                               (d^2 / (d^2 + s))^2
 * The scale d > 0 is in Mahalanobis units (dimensionless: s is a squared residual in standard deviations); the kernels use
 * d^2 = (float)(d * d).  A handle setting like the resolution: it survives set_*_cloud and swap_source_and_target and applies to
 * vgicp_compute_error, vgicp_align, vgicp_align_multi, vgicp_evaluate_poses and vgicp_register.  NONE reproduces the plain sums bit
 * for bit.  Errors: VGICP_ERR_INVALID_ARGUMENT for an unknown kind or a scale that is not finite and > 0 (the scale is ignored for
 * NONE).  NDT carries its own Cauchy weight: with an NDT problem selected and a kind other than NONE, vgicp_compute_error,
 * vgicp_align, vgicp_align_multi and vgicp_evaluate_poses return VGICP_ERR_UNSUPPORTED without launching anything. */
enum { VGICP_ROBUST_NONE = 0, VGICP_ROBUST_HUBER = 1, VGICP_ROBUST_CAUCHY = 2, VGICP_ROBUST_GEMAN_MCCLURE = 3 };
VGICP_API int vgicp_set_robust_kernel(vgicp_handle h, int kind, double scale);
/* ---- local map for scan-to-map odometry (not in the reference) -------------------------------------------------------------
 * Each frame: register the new scan against the map (vgicp_align), append it at the pose found, thin the cells that hold too
 * many points, crop what is too far or too old.  These calls work on the device arrays in place (no PCIe traffic for the map) and
 * leave the state that set_target_cloud + set_target_covariances + create_target_voxelmap with the resulting arrays would leave:
 * the target has covariances, no neighbour rows (vgicp_get_target_neighbors returns VGICP_ERR_BAD_STATE; find_target_neighbors +
 * calculate_target_covariances recompute k-NN covariances of the merged map if wanted), and the voxel map is rebuilt over the
 * whole target at the resolution it was first created with.  Handle settings (robust kernel, neighbour search, ...) are kept.
 * None is available with an NDT problem selected or with stage-1 sharding (VGICP_ERR_UNSUPPORTED); source sharding is unaffected
 * (every rank makes the same deterministic change).  Every error below is returned before anything is modified, and all but the
 * empty crop and the thinning's checks of the points before any launch.
 *
 * vgicp_append_source_to_target: the target grows from n_t to n_t + n_s points; rows n_t .. n_t + n_s - 1 hold the current source
 * transformed by T (column-major 4x4, cast to float like every pose):
 *   point i       = what vgicp_transform_source(h, T) returns for source point i, bit for bit;
 *   covariance i  = R C_i R^T, R the float rotation of T, in IEEE single operations without contraction, in this order:
 *                     M_ik = (R_i0 C_0k + R_i1 C_1k) + R_i2 C_2k,
 *                     N_ij = (M_i0 R_j0 + M_i1 R_j1) + M_i2 R_j2,
 *                   stored as set_covariances stores a 3x3: the diagonal N_ii and 0.5f * (N_ij + N_ji) off it.
 * The source is not changed.  Grow-only, amortised storage; the existing rows are copied on the device when it grows.
 * Errors: VGICP_ERR_INVALID_ARGUMENT (null or non-finite T, a merged target larger than a cloud may be: 2^31 / 64 points),
 * VGICP_ERR_BAD_STATE (source or target without points or covariances). */
VGICP_API int vgicp_append_source_to_target(vgicp_handle h, const double T[16]);
/* vgicp_crop_target: keep the target points within `radius` of `center`, then at most the newest `max_points` of them; rebuild the map.
 *   radius test   c = (float)center, dx = p.x - c.x (y, z alike), d^2 = (dx dx + dy dy) + dz dz in IEEE single operations;
 *                 point p passes when d^2 <= (float)(radius * radius).  radius = +inf keeps every point.
 *   point cap     when more than max_points points pass, only the last max_points of them in array order are kept (appends go
 *                 to the end, so these are the newest).  max_points = 0: no cap.
 * Kept points and their covariances stay in their original order.  One host synchronisation (the new size).
 * Errors: VGICP_ERR_INVALID_ARGUMENT (null center, NaN or negative radius, a crop that would leave no points: target and map are
 * then left exactly as they were), VGICP_ERR_BAD_STATE (target without points or covariances). */
VGICP_API int vgicp_crop_target(vgicp_handle h, const double center[3], double radius, size_t max_points);
/* vgicp_thin_target: keep at most M = max_points_per_voxel points per cell of a grid of leaf_size, the oldest; rebuild the map.
 *   cells   l = (float)leaf_size, inv = 1.0f / l; per axis c_a = floorf(p_a * inv) (one IEEE single multiplication).
 *   rule    target row i is kept iff fewer than M earlier rows (in array order) share its cell.  Appends go to the end, so a new
 *           scan only fills the cells that still have room, and a vehicle that stands still adds nothing to full cells.
 * Kept points and their covariances are unchanged and stay in their original order (a stable subsequence of the rows).  The state
 * afterwards is the one described above, also when nothing is dropped.  Two host synchronisations (the cells' box, the new size).
 * Per frame: vgicp_align, vgicp_carve_target, vgicp_append_source_to_target, vgicp_thin_target, then vgicp_crop_target (radius,
 * optional cap).
 * Errors, all returned before anything is modified (target and map stay exactly as they were):
 *   VGICP_ERR_INVALID_ARGUMENT  leaf_size not finite and > 0, l or inv not finite and > 0, M < 1; found by the first pass over
 *                               the points: a non-finite target coordinate, a cell outside [-2^31, 2^31), or a cell box too wide
 *                               for a 64-bit key (sum over the axes of bits(max c_a - min c_a) > 64);
 *   VGICP_ERR_BAD_STATE         target without points or covariances;
 *   VGICP_ERR_UNSUPPORTED       an NDT problem selected, or stage-1 sharding. */
VGICP_API int vgicp_thin_target(vgicp_handle h, double leaf_size, int max_points_per_voxel);
/* vgicp_carve_target: remove the moving objects' trails from the map.  The current source is the scan in its sensor frame (the
 * sensor at the origin) and T (column-major 4x4) maps it into the target frame, e.g. the vgicp_align result.  Every target point
 * that lies clearly in front of what the scan measured in its direction was seen through by the scan's rays: free space now, so
 * it is removed.  All arithmetic below is IEEE single operations without contraction, in the order written.
 *   pixel      of a sensor-frame point (x, y, z) in a height x width range image, without trigonometry:
 *                q = |y| / (|x| + |y|);  a = q (x >= 0, y >= 0), 2 - q (x < 0, y >= 0), 2 + q (x < 0, y < 0), 4 - q (x >= 0, y < 0)
 *                (the "diamond angle", monotone in the azimuth over [0, 4));  col = (int)floorf(a * wq), wq = width * 0.25f, and
 *                col == width becomes 0.  A column spans 4 / width rad of azimuth on the axes and 8 / width on the diagonals.
 *                rho = sqrtf(x x + y y), e = z / rho (the tangent of the elevation), u = (e - e_lo) * inv_de; the point has a
 *                pixel iff 0 <= u < height, row = (int)floorf(u).  e_lo = (float)tan(elevation_min) and
 *                inv_de = (float)(height / (tan(elevation_max) - tan(elevation_min))), in double with the C library's tan.
 *                A point with |x| + |y| == 0 or a non-finite coordinate has no pixel.
 *   range      r = sqrtf((x x + y y) + z z).
 *   image      per pixel, the least r of the source points that land in it (atomicMin on the float bits: r >= 0, so the bit
 *              order is the numeric order; independent of the order of the points); a pixel no point lands in is empty.
 *   map point  into the sensor frame with Ti = [R^T | -R^T t], formed from T in double (Ti_jk = R_kj,
 *              Ti_j3 = -((R_0j t_0 + R_1j t_1) + R_2j t_2)) and cast to float once:  s_j = ((Ti_j0 m_0 + Ti_j1 m_1) + Ti_j2 m_2) + Ti_j3.
 *   test       r_min = the least r over the non-empty pixels within `window` rows and columns of the point's pixel (rows clipped at
 *              the image's edges, columns modulo width); thr = r_min - (margin + margin_rel * r_min) with margin and margin_rel
 *              cast to float.  The point is removed iff it has a pixel, its window holds a non-empty pixel, and r < thr.  A point
 *              outside the vertical field of view, with an empty window, behind or on the measured surface, or with a non-finite
 *              coordinate (in the map or after the transform) is kept.
 * Kept points and their covariances are unchanged and stay in their original order; the state afterwards is the one described
 * above, also when nothing is removed.  *removed (optional) receives the number of removed points.  One host synchronisation (the
 * new size).  The source is not changed.  Call it after vgicp_align and before vgicp_append_source_to_target, so that the scan is
 * not tested against its own points, and before vgicp_thin_target, so that the cells it frees can fill again.
 * Errors, all returned before anything is modified (target and map stay exactly as they were):
 *   VGICP_ERR_INVALID_ARGUMENT  null or non-finite T, null params, width or height < 1, width * height > 2^24, elevation limits
 *                               not in (-pi/2, pi/2) with min < max, e_lo not finite or inv_de not finite and > 0, window not
 *                               in [0, 8], margin negative or not finite as a float, margin_rel not in [0, 1), a carve that
 *                               would leave no points;
 *   VGICP_ERR_BAD_STATE         source without points, target without points or covariances;
 *   VGICP_ERR_UNSUPPORTED       an NDT problem selected, or stage-1 sharding. */
typedef struct {
  int width, height;                   /* range image: columns (azimuth) x rows (elevation); 1024 x 64 */
  double elevation_min, elevation_max; /* vertical field of view in rad, lower and upper edge: -25 and +3 degrees */
  int window;                          /* pixels searched in each direction around the point's pixel, 0 .. 8; 1 */
  double margin;                       /* m: a point must lie this far in front of the measured range; 0.3 */
  double margin_rel;                   /* and this fraction of it in addition; 0.02 */
} vgicp_carve_params;
VGICP_API void vgicp_carve_default_params(vgicp_carve_params* p);
VGICP_API int vgicp_carve_target(vgicp_handle h, const double T[16], const vgicp_carve_params* params, size_t* removed);
/* ---- motion compensation (not in the reference) ---------------------------------------------------------------------------
 * A spinning or solid-state LiDAR fires the points of one sweep over its period while the vehicle moves; each point is in the
 * sensor frame of its own firing time.  vgicp_deskew_source re-expresses every source point in the sensor frame at t_ref under a
 * constant body velocity, so that the registration result is the pose at t_ref:
 *   source point i  <-  Exp((t_i - t_ref) xi) p_i,
 * xi = [omega, v] the twist per time unit in the sensor frame at t_ref, rotation first (the order of se3_exp, so3.hpp).  For a
 * constant-velocity guess, xi = log(T_{k-1}^-1 T_k) / dt (twist_from_motion in fast_gicp_b200/core.py).
 *   t, n, stride_bytes  host pointer to n float timestamps stride_bytes apart (stride >= 4, a multiple of 4): &cloud[0].time
 *                       with sizeof(PointT) reads them out of a PointXYZIT-like struct.  n must equal the source size.  Times
 *                       are relative (e.g. seconds since the start of the sweep): absolute epoch times have no precision
 *                       left in a float.
 * Arithmetic: IEEE single operations without contraction, in this order, so that numpy float32 rebuilds the same bytes:
 *   tau = (float)t_ref, om_j = (float)xi_j, nu_j = (float)xi_{3+j} (cast once);
 *   per point: s = t_i - tau, w_j = s om_j, u_j = s nu_j, q = (w0 w0 + w1 w1) + w2 w2  (theta^2);
 *   A, B, C by Horner, h = h q + c from the first coefficient listed (the series of sin(theta)/theta, (1 - cos(theta))/theta^2,
 *   (theta - sin(theta))/theta^3 in q, truncated below 2^-24 relative for theta <= pi/2; no trig calls):
 *     A: 1.6059044e-10f, -2.5052108e-08f, 2.7557319e-06f, -0.0001984127f, 0.008333334f, -0.16666667f, 1.0f
 *     B: -2.0876756e-09f, 2.755732e-07f, -2.4801588e-05f, 0.0013888889f, -0.041666668f, 0.5f
 *     C: -1.6059044e-10f, 2.5052108e-08f, -2.7557319e-06f, 0.0001984127f, -0.008333334f, 0.16666667f
 *   K = [w]x = [[0, -w2, w1], [w2, 0, -w0], [-w1, w0, 0]];  K2_jk = w_j w_k off the diagonal, K2_jj = w_j w_j - q;
 *   R_jk = (d_jk + A K_jk) + B K2_jk,  V_jk = (d_jk + B K_jk) + C K2_jk  (d_jk = 1 on the diagonal, else 0);
 *   p'_j = ((R_j0 p0 + R_j1 p1) + R_j2 p2) + ((V_j0 u0 + V_j1 u1) + V_j2 u2).
 * A zero twist returns every point's value unchanged (only the sign of a zero may differ).
 * Afterwards the handle is in the state set_source_cloud with the deskewed points would leave: no neighbour rows and no
 * covariances (find_source_neighbors + calculate_source_covariances come next), the NDT source map reset; handle settings, the
 * target and its map are kept.  Works under every problem and under source and stage-1 sharding (every rank makes the same
 * deterministic change).  The timestamps are packed on the host and uploaded (4 bytes per point), one kernel runs on the
 * source's stream after the work already enqueued that reads the source points.
 * Errors, all returned before anything is modified or launched: VGICP_ERR_INVALID_ARGUMENT (null t or twist with n > 0, n other
 * than the source size, a bad stride, a timestamp, twist component or t_ref that is not finite as a float, a rotation over the
 * sweep beyond the series: |omega| * max_i |t_i - t_ref| > pi/2 in double), VGICP_ERR_BAD_STATE (no source points). */
VGICP_API int vgicp_deskew_source(vgicp_handle h, const float* t, size_t n, size_t stride_bytes, const double twist[6], double t_ref);
/* ---- continuous-time registration (not in the reference) -------------------------------------------------------------------
 * Estimates the sweep's body twist together with the pose, from per-point timestamps, instead of taking the twist as given.
 * State x = (T, xi): T the pose at t_ref, xi = [omega, v] the body twist per time unit in the sensor frame at t_ref, rotation first
 * (vgicp_deskew_source's convention).  Source point i with timestamp t_i has s_i = t_i - (float)t_ref (in float) and is placed at
 *   p_i(T, xi) = T q_i,   q_i = Exp(s_i xi) a_i,
 * q_i computed by vgicp_deskew_source's recipe with xi cast to float: bit for bit the point vgicp_deskew_source(xi) would store.
 *   Correspondences  taken at (T_lin, xi_lin) with the handle's neighbour search and voxel index.  The source covariance enters as
 *                    R_lin C_i R_lin^T, as in vgicp_compute_error: the rotation of a covariance within the sweep is ignored.
 *   Per correspondence at (T_eval, xi_eval)  e, M, w, rho, rho' exactly as vgicp_compute_error forms them, with the point
 *                    p_i(T_eval, xi_eval); W = w rho'(s) M, J = [[p]x, -I] (the 6-column Jacobian of the left update).  The kernel
 *                    sums err = sum w rho, H0 = sum J^T W J, H1 = sum s_i J^T W J, H2 = sum s_i^2 J^T W J, b0 = sum J^T W e,
 *                    b1 = sum s_i J^T W e.
 *   Host, in double  with (R, t) the float image of T_eval and K = [[I, 0], [[t]x, I]] diag(R, R):
 *                      H = [[H0, H1 K], [K^T H1, K^T H2 K]] (12 x 12),  b = [b0; K^T b1],
 *                    the Gauss-Newton system of the update T <- Exp(d_T) T, xi <- xi + d_xi under Exp(s (xi + d)) ~ Exp(s d) Exp(s xi)
 *                    (the left Jacobian J_l(s xi) taken as I: exact at xi = 0, otherwise a relative error of about |s omega| / 2 in
 *                    the coupling blocks, some 1.7 % for 20 deg/s over a 0.1 s sweep).  err is exact, so the LM gain ratio judges
 *                    true errors.
 *   Twist prior      mean xi0 and weights W_j > 0: err += sum W_j (xi_j - xi0_j)^2, H_xixi += diag(W), b_xi += W o (xi - xi0).  It keeps
 *                    the system well posed when the timestamps span little or a direction is unobserved; the previous frame's
 *                    estimate is the natural xi0.
 * VGICP problem only, single GPU.  No speculation: one evaluation launch per optimiser evaluation.  The evaluation kernels are the
 * compacted kernels of vgicp_compute_error with a compile-time continuous-time flag (also where vgicp_compute_error streams DIRECT1).
 *
 * vgicp_set_source_timestamps: one float timestamp per source point, validated and packed exactly as vgicp_deskew_source takes
 * them (n equal to the source size, stride >= 4 and a multiple of 4, every value and (float)t_ref finite), kept on the device (4
 * bytes per point).  set_source_cloud(_device) and swap_source_and_target drop them; vgicp_deskew_source keeps them (a
 * continuous-time registration of a deskewed scan then estimates the residual twist).  Errors: VGICP_ERR_INVALID_ARGUMENT,
 * VGICP_ERR_BAD_STATE (no source points), before anything is changed. */
VGICP_API int vgicp_set_source_timestamps(vgicp_handle h, const float* t, size_t n, size_t stride_bytes, double t_ref);
/* vgicp_set_source_timestamps with the timestamps already in this GPU's memory (device pointer d_t, same n, stride and t_ref
 * rules): e.g. the time column of vgicp_prep_approximate_voxel_grid_fields' device output, read in place at out + 3 + j with
 * stride (3 + F) * 4.  Leaves exactly the state vgicp_set_source_timestamps leaves with the same values.  One kernel packs the
 * values into a spare device buffer, counting the non-finite ones and finding min and max in the same pass; one readback
 * follows, and the spare buffer replaces the stored timestamps only when every value passed.  The read is stream-ordered on the
 * handle's stream, after the source's pending work, and the call returns after it: the caller may then reuse d_t, and a buffer
 * just given to vgicp_set_source_cloud_device as well.  Errors: VGICP_ERR_INVALID_ARGUMENT (null d_t
 * with n > 0, n other than the source size, a bad stride, a non-finite t_ref, each before any launch; a non-finite timestamp
 * or t_i - t_ref overflowing a float, found by the kernel: the previous timestamps stay in place), VGICP_ERR_BAD_STATE (no
 * source points, before any launch). */
VGICP_API int vgicp_set_source_timestamps_device(vgicp_handle h, const float* d_t, size_t n, size_t stride_bytes, double t_ref);
/* vgicp_deskew_source with the stored timestamps and their t_ref (vgicp_set_source_timestamps(_device)): no upload, the same
 * kernel on the stored buffer, so the points are byte for byte those vgicp_deskew_source(h, the same values, ..., twist, the
 * same t_ref) stores.  The same stream ordering, the same refusal rule (|omega| * max_i |t_i - t_ref| > pi/2 in double, over the
 * stored raw min and max) and the same state afterwards: no neighbour rows, no covariances, the NDT source map reset, the
 * timestamps kept.  Errors, all before any launch: VGICP_ERR_INVALID_ARGUMENT (null or non-finite twist, a rotation beyond the
 * series), VGICP_ERR_BAD_STATE (no stored timestamps). */
VGICP_API int vgicp_deskew_source_stored(vgicp_handle h, const double twist[6]);
/* The data terms alone (no prior) at (T_eval, xi_eval) over the correspondences of (T_lin, xi_lin): H144 (12 x 12 column-major)
 * and b12, both given or both NULL (error only), and *err.  Errors as vgicp_align_ct's. */
VGICP_API int vgicp_compute_error_ct(vgicp_handle h, const double T_lin[16], const double xi_lin[6], const double T_eval[16], const double xi_eval[6], double* H144,
                                     double* b12, double* err);
typedef struct {
  double T[16];        /* final pose at t_ref */
  double twist[6];     /* final body twist [omega, v] */
  double H[144];       /* final 12 x 12 system matrix (prior included), column-major */
  int nr_iterations;
  int converged;       /* the last step moved both the pose and the sweep's end (Exp(S d_xi), S = max |s_i|) below the epsilons */
  int n_linearize;
  int n_compute_error;
  int lm_failed;
} vgicp_align_ct_result;
/* vgicp_align's optimiser (the same LM / GN state machine in 12 dimensions): lambda starts at lm_init_lambda_factor times the largest
 * of the 12 diagonal entries, the gain ratio's denominator runs over all 12; a trial whose rotation over the sweep |omega| S exceeds
 * pi/2 (outside the series) is a rejected step and launches nothing (with Gauss-Newton it ends the run with lm_failed = 1, the last
 * estimate kept).  params NULL: vgicp_lsq_default_params.  The handle's linearisation point and the rest of its single-pose state
 * are left as they were.  Errors, all returned before any launch: VGICP_ERR_INVALID_ARGUMENT (a null or non-finite input, a weight
 * <= 0, a twist guess or prior beyond the series bound), VGICP_ERR_BAD_STATE (no timestamps, or the preconditions of vgicp_align),
 * VGICP_ERR_UNSUPPORTED (an NDT problem, or a handle with source or stage-1 sharding or in a multi-GPU communicator). */
VGICP_API int vgicp_align_ct(vgicp_handle h, const double guess[16], const double twist_guess[6], const double twist_prior[6], const double twist_weight[6],
                             const vgicp_lsq_params* params, vgicp_align_ct_result* result);
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
/* Execution hint: how an evaluation hands its result to the host.  0 = latency (default: every evaluation writes its 43 doubles
 * straight into mapped host memory and the calling thread spins on a completion word), 1 = throughput / polite (evaluations are
 * read back with a copy and a stream wait, so the host thread sleeps instead of spinning).  The kernels, their launch shapes and
 * the results are the same under both.  bench.py uses the latency shape. */
VGICP_API int vgicp_set_execution_hint(vgicp_handle h, int hint);
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
