// dev_buffer.h -- the one owner of the C ABI's HBM and pinned host memory: the only code in csrc/ that allocates or frees it
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include "../../include/openclaw_gov.h"
namespace cg {
int cuda_fail(cudaError_t e, const char* what);   // (capi.cu) records the error -> CG_ERR_CUDA

// n elements of T in HBM (pinned host memory when Pinned) behind Pad zeroed bytes, readable by the kernels, and before Pad more.
// Move-only; reset(), the next alloc() and the destructor free it with cudaFree / cudaFreeHost, which wait for the device.
template <typename T, bool Pinned = false, size_t Pad = 0>
class Buf {
 public:
  Buf() = default;
  Buf(Buf&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  Buf& operator=(Buf&& o) noexcept { if (this != &o) { reset(); p_ = o.p_; n_ = o.n_; o.p_ = nullptr; o.n_ = 0; } return *this; }
  ~Buf() { reset(); }
  T* get() const { return p_ ? reinterpret_cast<T*>(p_ + Pad) : nullptr; }
  size_t cap() const { return n_; }
  // exactly n elements, uninitialised; what was held is freed first (on failure the buffer is empty)
  int alloc(size_t n) {
    reset();
    const cudaError_t e = Pinned ? cudaMallocHost((void**)&p_, n * sizeof(T) + 2 * Pad) : cudaMalloc((void**)&p_, n * sizeof(T) + 2 * Pad);
    if (e != cudaSuccess) { p_ = nullptr; return cuda_fail(e, Pinned ? "cudaMallocHost" : "cudaMalloc"); }
    if (Pad) cudaMemset(p_, 0, Pad);
    n_ = n;
    return CG_OK;
  }
  // grow-only: at least `need` elements; a reallocation adds need / 4 + 64 elements of slack and keeps no contents
  int grow(size_t need) { return need <= n_ && p_ ? CG_OK : alloc(need + need / 4 + 64); }
  void reset() { if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); } p_ = nullptr; n_ = 0; }
 private:
  char* p_ = nullptr; size_t n_ = 0;
};
template <typename T> using DevBuf = Buf<T>;
template <typename T> using HostBuf = Buf<T, true>;
}  // namespace cg
