/* vgicp_prep_b200.h -- device-side input preparation for the VGICP path (SURVEY.md 8f-2): what the reference's callers do to a raw
 * scan on the host, serially, before setInputTarget / setInputSource:
 *   src/align.cpp:128-133          erase(remove_if(squaredNorm() < 1e-3))          near-origin filter (invalid returns)
 *   src/align.cpp:136-147, src/kitti.cpp:80-82, src/python/main.cpp:46-62,81-91   pcl::ApproximateVoxelGrid<PointXYZ>
 * A separate small library (lib/libvgicp_prep_b200.so): the registration library does not depend on it.
 *
 * The algorithm is pinned on the CPU side (oracle/vgicp_oracle.c: orc_approximate_voxel_grid reproduces the committed benchmark
 * fixture bit for bit); the CUDA implementation is compiled for sm_90a and checked against it by tests/test_input_prep.py.
 *
 * pcl::ApproximateVoxelGrid is a streaming filter: each point goes to entry (ix*7171 + iy*3079 + iz*4231) & 511 of a 512-entry
 * history; an entry holding another voxel is flushed (its centroid emitted) first; what is left is flushed in entry order at the
 * end.  The output therefore depends on the input ORDER -- but only within an entry: the 512 entries are 512 independent
 * sequential chains.  The device version runs them as 512 threads of one block, keeps the per-entry order, and places every
 * flushed centroid at the rank of the point that flushed it, so the output (points AND order) is the one the serial filter
 * produces, bit for bit (float sums in input order, IEEE division). */
#ifndef VGICP_PREP_B200_H
#define VGICP_PREP_B200_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif
#if defined(_WIN32)
#define VGICP_PREP_API
#else
#define VGICP_PREP_API __attribute__((visibility("default")))
#endif

typedef struct vgicp_prep_context* vgicp_prep_handle;

/* status codes as vgicp_b200.h: 0 ok, 1 invalid argument, 3 CUDA error, 5 no device */
VGICP_PREP_API int vgicp_prep_create(int device, vgicp_prep_handle* out);
VGICP_PREP_API void vgicp_prep_destroy(vgicp_prep_handle h);
VGICP_PREP_API const char* vgicp_prep_last_error(vgicp_prep_handle h);

/* xyz: n points, float32 x y z at stride_bytes (>= 12, multiple of 4), host memory (on_device = 0) or device memory (1).
 * remove_near_origin != 0 applies align.cpp:128-133 first (the filter is stable, so it is fused: filtered points simply never
 * reach the history).  leaf: the cubic leaf size (setLeafSize(l, l, l)).
 * out_xyz: packed float32 xyz, capacity `cap` points (n always suffices), host (out_on_device = 0) or device memory.
 * *n_out receives the number of points written.  Blocks until the result is in place. */
VGICP_PREP_API int vgicp_prep_approximate_voxel_grid(vgicp_prep_handle h, const float* xyz, size_t n, size_t stride_bytes, int on_device, float leaf, int remove_near_origin,
                                                     float* out_xyz, size_t cap, int out_on_device, size_t* n_out);
/* The same filter keeping per-point float fields, as pcl::ApproximateVoxelGrid<PointT> does by default (setDownsampleAllData(true)):
 * the time and intensity of a PointXYZIT-like point are averaged over the voxel next to x y z.
 *   points         n records stride_bytes apart (>= 12, a multiple of 4), host (on_device = 0) or device memory; x y z at byte
 *                  offsets 0, 4, 8 of each record.  A host input is copied up to the last byte of the last record the filter reads.
 *   field_offsets  n_fields (1 ... 8) byte offsets of float32 fields, each a multiple of 4, >= 12 and offset + 4 <= stride_bytes.
 *   out            m records of 3 + n_fields floats: x y z f_0 ... f_{F-1}, capacity `cap` records (n always suffices), host
 *                  (out_on_device = 0) or device memory.  A device output is the layout vgicp_set_source_cloud_device(out, m,
 *                  (3 + F) * 4) reads, and field j is read in place at out + 3 + j with the same stride (e.g. by
 *                  vgicp_set_source_timestamps_device).
 * Arithmetic: each field is summed in float in input order next to x y z and divided once by (float)count (IEEE division), at
 * the same flushes and in the same output order; x y z are vgicp_prep_approximate_voxel_grid's bytes for the same input.
 * Blocks until the result is in place. */
VGICP_PREP_API int vgicp_prep_approximate_voxel_grid_fields(vgicp_prep_handle h, const float* points, size_t n, size_t stride_bytes, int on_device, float leaf,
                                                            int remove_near_origin, const size_t* field_offsets, int n_fields, float* out, size_t cap, int out_on_device,
                                                            size_t* n_out);
/* pcl::VoxelGrid, the exact grid: one centroid per occupied voxel, x y z and n_fields per-point float fields (0 ... 8) averaged over
 * the voxel.  Unlike the approximate filter its output does not depend on the order of the input points.
 *   points, n, stride_bytes, on_device, remove_near_origin, field_offsets, out, cap, out_on_device, n_out: as for
 *                  vgicp_prep_approximate_voxel_grid_fields (field_offsets may be null when n_fields is 0); the output is m records of
 *                  3 + n_fields floats, the layout vgicp_set_source_cloud_device and vgicp_set_source_timestamps_device read in place.
 *   min_points_per_voxel  voxels with fewer points are dropped (pcl::VoxelGrid::setMinimumPointsNumberPerVoxel; 0 and 1 keep all).
 * Recipe (every float operation one IEEE single operation, no contraction):
 *   1. kept points: x, y and z finite (a non-dense pcl::VoxelGrid drops the others) and, when remove_near_origin is set, not
 *      ((x*x + y*y) + z*z) < 1e-3f.  Dropped points neither widen the box nor land in a voxel.
 *   2. cells: inv = 1.0f / leaf; per axis c = floorf(x * inv) (one multiplication).  A kept c outside [-2^31, 2^31) refuses the
 *      call; otherwise g = (int)c.
 *   3. box: min_b, max_b = per-axis min and max of g over the kept points; div = max_b - min_b + 1 in int64.  A cell product
 *      div_x * div_y * div_z > INT32_MAX refuses the call (pcl::VoxelGrid has the same guard but silently returns its input
 *      instead; refusing is deliberate).  x * inv is monotone in x, so min_b is PCL's floor(min_p * inv).
 *   4. voxel index: idx = (g_x - min_b_x) + (g_y - min_b_y) * div_x + (g_z - min_b_z) * div_x * div_y in integers.  PCL subtracts in
 *      float; the two differ only where |x / leaf| >= 2^24, where PCL's index can be wrong.
 *   5. a voxel is a run of equal idx; voxels with fewer than min_points_per_voxel points are dropped; the output is in ascending
 *      idx order (PCL's).
 *   6. centroids: for x, y, z and each field, s = 0.0f, then s = s + v over the voxel's points in ascending input index, then
 *      s / (float)count.  This is PCL's Vector4f accumulation with the order inside a voxel, which PCL's std::sort leaves
 *      unspecified, fixed to input order.  Non-finite field values propagate (a NaN result is a NaN; its payload is not pinned).
 *   7. no kept point, or no voxel with enough points: status 0 and *n_out = 0.
 * Status 1 with nothing written to out and *n_out = 0: a null handle, n_out or buffer, a bad stride, offset or field count, a leaf
 * that is not finite and positive, n > INT32_MAX - 4096, a cell outside the int range or a cell product above INT32_MAX.  Status 1
 * with *n_out = m (out untouched) when m > cap.  3 on a CUDA error.  Blocks until the result is in place. */
VGICP_PREP_API int vgicp_prep_voxel_grid(vgicp_prep_handle h, const float* points, size_t n, size_t stride_bytes, int on_device, float leaf,
                                         int remove_near_origin, const size_t* field_offsets, int n_fields, unsigned min_points_per_voxel,
                                         float* out, size_t cap, int out_on_device, size_t* n_out);
#ifdef __cplusplus
}
#endif
#endif
