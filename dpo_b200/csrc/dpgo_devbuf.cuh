// dpgo_devbuf.cuh -- owners of the host side's CUDA resources.  Every device array, pinned buffer, event and graph exec
// the library keeps is held by one of these, so dropping or replacing it (a reset is the assignment of a fresh value)
// releases it, and no free list has to name it.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <memory>
#include <type_traits>

namespace dpgo {

struct CudaFree { void operator()(void *p) const { cudaFree(p); } };
struct CudaFreeHost { void operator()(void *p) const { cudaFreeHost(p); } };
struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct GraphExecDestroy { void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };

using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy>;
using GraphExec = std::unique_ptr<std::remove_pointer_t<cudaGraphExec_t>, GraphExecDestroy>;
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDestroy>;

// By default an event without timing (the fork / join events of the round calls).
inline cudaError_t create_event(Event &ev, unsigned flags = cudaEventDisableTiming) {
  cudaEvent_t e = nullptr;
  const cudaError_t rc = cudaEventCreateWithFlags(&e, flags);
  ev.reset(e);
  return rc;
}

// A device array of T, move-only, freed by its destructor.
template <class T> class DevBuf {
 public:
  T *get() const { return p_.get(); }
  explicit operator bool() const { return p_ != nullptr; }

  // Replaces the array by one of `count` elements (at least one, so that an empty table still has an address).
  cudaError_t alloc(size_t count) {
    p_.reset();
    T *q = nullptr;
    const cudaError_t e = cudaMalloc(&q, sizeof(T) * std::max<size_t>(count, 1));
    p_.reset(q);
    return e;
  }

  // Copies `count` elements from host memory, ordered on `stream` with the kernels that read them.  The host memory must
  // stay valid until the stream has reached the copy.
  cudaError_t upload(const T *host, size_t count, cudaStream_t stream) {
    if (!count) return cudaSuccess;
    return cudaMemcpyAsync(get(), host, sizeof(T) * count, cudaMemcpyHostToDevice, stream);
  }

  // alloc(count), then upload(host, count, stream).
  cudaError_t assign(const T *host, size_t count, cudaStream_t stream) {
    const cudaError_t e = alloc(count);
    return e == cudaSuccess ? upload(host, count, stream) : e;
  }

 private:
  std::unique_ptr<T, CudaFree> p_;
};

}  // namespace dpgo
