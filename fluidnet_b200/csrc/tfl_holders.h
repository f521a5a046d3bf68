// Owners of CUDA resources: std::unique_ptr with a stateless deleter, one owner per resource, released when the owner
// goes (on every error path too).  The helpers make one and return an empty holder when the CUDA call fails.
#pragma once
#include <cuda_runtime.h>
#include <memory>
#include <vector>

namespace tfl {

struct CudaFree { void operator()(void* p) const { cudaFree(p); } };
struct CudaFreeHost { void operator()(void* p) const { cudaFreeHost(p); } };
struct CudaStreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct CudaEventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct CudaGraphDestroy { void operator()(cudaGraph_t g) const { cudaGraphDestroy(g); } };
struct CudaGraphExecDestroy { void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); } };
struct CudaIpcClose { void operator()(void* p) const { cudaIpcCloseMemHandle(p); } };

template <typename T> using DevPtr = std::unique_ptr<T, CudaFree>;          // device memory
template <typename T> using PinnedPtr = std::unique_ptr<T, CudaFreeHost>;   // pinned host memory
template <typename T> using IpcPtr = std::unique_ptr<T, CudaIpcClose>;      // a peer's memory (ipc_map)
using StreamPtr = std::unique_ptr<CUstream_st, CudaStreamDestroy>;
using EventPtr = std::unique_ptr<CUevent_st, CudaEventDestroy>;
using GraphPtr = std::unique_ptr<CUgraph_st, CudaGraphDestroy>;
using GraphExecPtr = std::unique_ptr<CUgraphExec_st, CudaGraphExecDestroy>;

// n device values, uninitialised; empty if cudaMalloc fails.
template <typename T>
DevPtr<T> dev_alloc(size_t n) {
  T* p = nullptr;
  if (cudaMalloc((void**)&p, n * sizeof(T)) != cudaSuccess) return DevPtr<T>();
  return DevPtr<T>(p);
}
// n device values set to zero; empty if cudaMalloc or cudaMemset fails.
template <typename T>
DevPtr<T> dev_zeros(size_t n) {
  DevPtr<T> d = dev_alloc<T>(n);
  if (d && cudaMemset(d.get(), 0, n * sizeof(T)) != cudaSuccess) d.reset();
  return d;
}
// A device copy of host[0, n); empty if cudaMalloc or cudaMemcpy fails.
template <typename T>
DevPtr<T> upload(const T* host, size_t n) {
  DevPtr<T> d = dev_alloc<T>(n);
  if (d && cudaMemcpy(d.get(), host, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) d.reset();
  return d;
}
template <typename T>
DevPtr<T> upload(const std::vector<T>& host) { return upload(host.data(), host.size()); }
// n pinned host values, uninitialised; empty if cudaMallocHost fails.
template <typename T>
PinnedPtr<T> pinned_alloc(size_t n) {
  T* p = nullptr;
  if (cudaMallocHost((void**)&p, n * sizeof(T)) != cudaSuccess) return PinnedPtr<T>();
  return PinnedPtr<T>(p);
}
// A stream / event with these flags; empty if the creation fails.
inline StreamPtr new_stream(unsigned flags) {
  cudaStream_t s = nullptr;
  if (cudaStreamCreateWithFlags(&s, flags) != cudaSuccess) return StreamPtr();
  return StreamPtr(s);
}
inline EventPtr new_event(unsigned flags) {
  cudaEvent_t e = nullptr;
  if (cudaEventCreateWithFlags(&e, flags) != cudaSuccess) return EventPtr();
  return EventPtr(e);
}

}  // namespace tfl
