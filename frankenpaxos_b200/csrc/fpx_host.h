// fpx_host.h -- host-only helpers of fpx_engine.cu: the CUDA resources of a handle, the one CUDA check and the
// device check.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/fpx.h"

// Every device allocation, pinned allocation, stream and event one handle (or one call's temporaries) creates,
// released together when the owner goes: the device is set, the owner's streams are drained, device memory and
// then pinned memory is freed, events and then streams are destroyed.  It records allocations, not fields, so a
// handle may swap its buffers or regrow one (free_dev + alloc).
struct CudaResources {
  int device = 0;
  std::vector<void*> dev, pinned;
  std::vector<cudaEvent_t> events;
  std::vector<cudaStream_t> streams;

  explicit CudaResources(int d = 0) : device(d) {}
  CudaResources(const CudaResources&) = delete;
  CudaResources& operator=(const CudaResources&) = delete;
  ~CudaResources() {
    sync();
    for (void* p : dev) cudaFree(p);
    for (void* p : pinned) cudaFreeHost(p);
    for (cudaEvent_t ev : events) cudaEventDestroy(ev);
    for (cudaStream_t s : streams) cudaStreamDestroy(s);
  }
  // sets the device and waits for the owner's streams
  void sync() const {
    cudaSetDevice(device);
    for (cudaStream_t s : streams) cudaStreamSynchronize(s);
  }
  template <class T> cudaError_t alloc(T** p, size_t bytes) { return keep(dev, cudaMalloc(p, bytes), p); }
  template <class T> cudaError_t alloc_pinned(T** p, size_t bytes) { return keep(pinned, cudaMallocHost((void**)p, bytes), p); }
  cudaError_t stream(cudaStream_t* s) { return keep(streams, cudaStreamCreateWithFlags(s, cudaStreamNonBlocking), s); }
  cudaError_t event(cudaEvent_t* ev, unsigned flags) { return keep(events, cudaEventCreateWithFlags(ev, flags), ev); }
  void free_dev(void* p) {
    auto it = std::find(dev.begin(), dev.end(), p);
    if (it != dev.end()) { cudaFree(p); dev.erase(it); }
  }

 private:
  template <class V, class P> static cudaError_t keep(std::vector<V>& v, cudaError_t err, P* made) {
    if (err == cudaSuccess) v.push_back(*made);
    return err;
  }
};

// A failed CUDA call: "<call>: <error>" goes to stderr and, when there is a handle, to its last_error.
template <class H>
static int cuda_failed(const H& h, const char* call, cudaError_t err) {
  std::string msg = std::string(call) + ": " + cudaGetErrorString(err);
  fprintf(stderr, "fpx: %s\n", msg.c_str());
  if constexpr (!std::is_same<H, std::nullptr_t>::value) h->last_error = std::move(msg);
  return FPX_ERR_CUDA;
}
#define CK(h, call)                                                \
  do {                                                             \
    const cudaError_t _err = (call);                               \
    if (_err != cudaSuccess) return cuda_failed((h), #call, _err); \
  } while (0)

static bool device_exists(int device) {
  int n = 0;
  return cudaGetDeviceCount(&n) == cudaSuccess && device >= 0 && device < n;
}
