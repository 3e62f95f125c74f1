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
#ifdef __cplusplus
}
#endif
#endif
