// vgicp_devbuf.hpp -- the owners of the CUDA resources of both native libraries (libvgicp_b200.so and libvgicp_prep_b200.so).
// Every resource a handle allocates is held by one of these, so deleting the handle frees all of it.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <memory>
#include <type_traits>
#include <utility>

namespace vgicp {

template <typename T>
struct DevBuf {  // grow-only device array
  T* p = nullptr;
  size_t cap = 0;
  bool external = false;  // points into memory owned elsewhere (the multi-GPU exchange arena): fixed capacity, never freed here
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)), external(std::exchange(o.external, false)) {}
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      reset();
      p = std::exchange(o.p, nullptr);
      cap = std::exchange(o.cap, 0);
      external = std::exchange(o.external, false);
    }
    return *this;
  }
  ~DevBuf() { reset(); }
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
  void attach(T* q, size_t capacity) {  // switch to external storage
    reset();
    p = q;
    cap = capacity;
    external = true;
  }

 private:
  void reset() {
    if (p && !external) cudaFree(p);
    p = nullptr;
    cap = 0;
    external = false;
  }
};

// Owners of fixed-size resources: each frees its resource when it is destroyed or reset
struct DeviceFree { void operator()(void* p) const { cudaFree(p); } };
struct HostFree { void operator()(void* p) const { cudaFreeHost(p); } };
struct IpcClose { void operator()(void* p) const { cudaIpcCloseMemHandle(p); } };
struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct GraphExecDestroy { void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); } };
// (an array takes T[]: the owner then indexes like a pointer)
template <typename T>
using DevPtr = std::unique_ptr<T, DeviceFree>;  // device memory (cudaMalloc)
template <typename T>
using HostPtr = std::unique_ptr<T, HostFree>;  // pinned host memory (cudaHostAlloc, with the site's flags)
template <typename T>
using IpcPtr = std::unique_ptr<T, IpcClose>;  // a peer process's device memory mapped into this one (cudaIpcOpenMemHandle)
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy>;
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDestroy>;
using GraphExec = std::unique_ptr<std::remove_pointer_t<cudaGraphExec_t>, GraphExecDestroy>;

template <typename T>
constexpr bool kMoveOnly = !std::is_copy_constructible<T>::value && !std::is_copy_assignable<T>::value && std::is_nothrow_move_constructible<T>::value;
static_assert(kMoveOnly<DevBuf<int>> && kMoveOnly<DevPtr<int[]>> && kMoveOnly<HostPtr<int[]>> && kMoveOnly<IpcPtr<int[]>> && kMoveOnly<Event> &&
                  kMoveOnly<Stream> && kMoveOnly<GraphExec>,
              "an owner is never copied: the copy would free the resource a second time");

// The creation calls: on success the owner holds the new resource (and has freed what it held); on failure it is unchanged
template <typename T>
cudaError_t device_alloc(DevPtr<T>& o, size_t bytes) {
  void* p = nullptr;
  const cudaError_t e = cudaMalloc(&p, bytes);
  if (e == cudaSuccess) o.reset(static_cast<typename DevPtr<T>::pointer>(p));
  return e;
}
template <typename T>
cudaError_t host_alloc(HostPtr<T>& o, size_t bytes, unsigned flags) {
  void* p = nullptr;
  const cudaError_t e = cudaHostAlloc(&p, bytes, flags);
  if (e == cudaSuccess) o.reset(static_cast<typename HostPtr<T>::pointer>(p));
  return e;
}
inline cudaError_t event_create(Event& o, unsigned flags) {
  cudaEvent_t ev = nullptr;
  const cudaError_t e = cudaEventCreateWithFlags(&ev, flags);
  if (e == cudaSuccess) o.reset(ev);
  return e;
}
inline cudaError_t stream_create(Stream& o, unsigned flags) {
  cudaStream_t st = nullptr;
  const cudaError_t e = cudaStreamCreateWithFlags(&st, flags);
  if (e == cudaSuccess) o.reset(st);
  return e;
}

}  // namespace vgicp
