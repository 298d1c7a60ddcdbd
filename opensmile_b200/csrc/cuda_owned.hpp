// cuda_owned.hpp -- move-only owners of the CUDA resources of plans, functionals objects and sessions (host-only C++17, also built
// by g++ for host/front.cpp).  Each releases in its destructor, after its holder has selected the device; a null owner makes no
// CUDA call, so description-only objects never touch the runtime.  A moved owner keeps its address: raw views into it stay valid.
#pragma once
#include <cuda_runtime_api.h>

#include <cstdio>
#include <utility>

#include "plan.hpp"

namespace osm {

inline osm_b200_status cuda_fail(cudaError_t e, const char *what)
{
  char buf[512];
  snprintf(buf, sizeof buf, "CUDA error in %s: %s", what, cudaGetErrorString(e));
  return set_last_error(OSM_B200_ERR_CUDA, buf);
}

#define CU(call)                                                \
  do {                                                          \
    cudaError_t e_ = (call);                                    \
    if (e_ != cudaSuccess) return osm::cuda_fail(e_, #call);    \
  } while (0)

// array of T in device memory, or in page-locked host memory (Pinned)
template <typename T, bool Pinned>
struct CudaBuf {
  T *p = nullptr;
  size_t cap = 0;   // elements

  CudaBuf() = default;
  CudaBuf(CudaBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  ~CudaBuf() { release(); }

  // at least n elements; a buffer that grows gets headroom for later batches and loses its contents
  cudaError_t reserve(size_t n) { return n <= cap ? cudaSuccess : alloc(n + n / 8 + 64); }
  // at least n elements; a buffer that grows gets exactly n
  cudaError_t reserve_exact(size_t n) { return n <= cap ? cudaSuccess : alloc(n); }
  // exactly n elements holding a copy of the host array `src` (device memory)
  cudaError_t upload(const T *src, size_t n)
  {
    const cudaError_t e = alloc(n);
    return e != cudaSuccess ? e : cudaMemcpy(p, src, n * sizeof(T), cudaMemcpyHostToDevice);
  }

 private:
  void release()
  {
    if (p) { if (Pinned) cudaFreeHost(p); else cudaFree(p); }
    p = nullptr; cap = 0;
  }
  cudaError_t alloc(size_t n)
  {
    release();
    void *q = nullptr;
    const cudaError_t e = Pinned ? cudaMallocHost(&q, n * sizeof(T)) : cudaMalloc(&q, n * sizeof(T));
    if (e == cudaSuccess) { p = static_cast<T *>(q); cap = n; }
    return e;
  }
};
template <typename T> using DevBuf = CudaBuf<T, false>;
template <typename T> using PinBuf = CudaBuf<T, true>;

// a cudaStream_t or cudaEvent_t; converts to the raw handle for runtime calls
template <typename H, cudaError_t (*Create)(H *, unsigned), cudaError_t (*Destroy)(H)>
class CudaHandle {
 public:
  CudaHandle() = default;
  CudaHandle(CudaHandle &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  CudaHandle &operator=(CudaHandle o) noexcept { std::swap(h_, o.h_); return *this; }
  ~CudaHandle() { if (h_) Destroy(h_); }

  cudaError_t create(unsigned flags = 0) { *this = CudaHandle(); return Create(&h_, flags); }
  operator H() const { return h_; }

 private:
  H h_ = nullptr;
};
using CudaStream = CudaHandle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;
using CudaEvent = CudaHandle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;

}  // namespace osm
