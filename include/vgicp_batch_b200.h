/* vgicp_batch_b200.h -- many registrations, one call: the reference's benchmark and odometry loops (src/align.cpp:72-81 "100times",
 * src/kitti.cpp:97-118) call clear + setInputTarget + setInputSource + align once per pair from one host thread.  A 17k-point
 * registration is a chain of ~30 small latency-bound launches and cannot fill an H100; the throughput configuration runs several
 * registrations concurrently, one vgicp handle (own CUDA streams) and one host thread each (DESIGN.md 5).  This small host-side
 * library (lib/libvgicp_batch_b200.so, plain C++ over the public C ABI of vgicp_b200.h, no CUDA code of its own) packages that:
 * a pool of handles on one device, worker threads pulling pairs from a shared counter.  Every pair goes through vgicp_register
 * on one handle exactly as a sequential caller would run it, so the results are those of the sequential loop, bit for bit,
 * whatever the interleaving.  (SURVEY.md 8b lists it as the `vgicp_batch_align` extension.)
 *
 * Checked by tests/test_batch.py (24 pairs over 6 handles against the sequential loop: same poses, counters and aligned clouds,
 * bit for bit).  A device-batched execution path (one launch per stage over all pairs) is not built: DESIGN.md 8. */
#ifndef VGICP_BATCH_B200_H
#define VGICP_BATCH_B200_H
#include <stddef.h>

#include "vgicp_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct vgicp_batch_context* vgicp_batch_handle;

/* n_streams handles on `device` (1..64); status codes as vgicp_b200.h */
VGICP_API int vgicp_batch_create(int device, int n_streams, vgicp_batch_handle* out);
VGICP_API void vgicp_batch_destroy(vgicp_batch_handle b);
VGICP_API const char* vgicp_batch_last_error(vgicp_batch_handle b);
VGICP_API int vgicp_batch_num_streams(vgicp_batch_handle b);
/* FastVGICPCuda::setResolution / setNeighborSearchMethod on every handle of the pool (fast_vgicp_cuda_impl.hpp:40-61) */
VGICP_API int vgicp_batch_configure(vgicp_batch_handle b, double resolution, int neighbor_search_method, double radius);
/* n_pairs registrations.  Pair i: target_xyz[i] (n_target[i] points) and source_xyz[i] (n_source[i] points), float32 xyz at
 * stride_bytes, host pointers or device pointers (on_device != 0); k, regularization_method as vgicp_register; guesses: 16 doubles
 * per pair (column-major) or NULL for identity; params NULL for the LsqRegistration defaults.  results[i] receives what
 * vgicp_align returns for pair i.  aligned_out: NULL, or per pair NULL / a HOST buffer of n_source[i] packed xyz floats that
 * receives the source transformed by the final pose (what align() hands back, lsq_registration_impl.hpp:78).
 * Returns the first error any worker met (its message in vgicp_batch_last_error); results of pairs not reached are left untouched. */
VGICP_API int vgicp_batch_register(vgicp_batch_handle b, size_t n_pairs, const float* const* target_xyz, const size_t* n_target, const float* const* source_xyz,
                                   const size_t* n_source, size_t stride_bytes, int on_device, int k, int regularization_method, const double* guesses,
                                   const vgicp_lsq_params* params, vgicp_align_result* results, float* const* aligned_out);
#ifdef __cplusplus
}
#endif
#endif
