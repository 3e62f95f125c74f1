// vgicp_devbuf.hpp -- the grow-only device array of both native libraries (libvgicp_b200.so and libvgicp_prep_b200.so).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace vgicp {

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
  // reserve that keeps the first `keep` elements: copied in stream order on `st`; the old array is freed once `st` has drained,
  // since work enqueued there may still read it
  cudaError_t grow(size_t n, size_t keep, cudaStream_t st) {
    if (n <= cap) return cudaSuccess;
    if (external) return cudaErrorMemoryAllocation;
    const size_t want = n + n / 4 + 16;
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (keep) e = cudaMemcpyAsync(q, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && p) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
      cudaFree(q);
      return e;
    }
    if (p) cudaFree(p);
    p = q;
    cap = want;
    return cudaSuccess;
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

}  // namespace vgicp
