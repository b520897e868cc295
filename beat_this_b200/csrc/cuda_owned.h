// Move-only owners of the CUDA resources the C ABI allocates: device and pinned host buffers, events and the
// tensor-core plans.  Each releases what it holds when it is destroyed or assigned over, so a bt_ctx that holds them
// frees everything it allocated when it is deleted (with its device current).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <memory>
#include <utility>

#include "bt_kernels.h"

namespace bt {

// A block of bytes from Alloc, seen as T*.
template <class T, cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
class CudaBuffer {
 public:
  CudaBuffer() = default;
  CudaBuffer(CudaBuffer&& o) noexcept { *this = std::move(o); }
  CudaBuffer& operator=(CudaBuffer&& o) noexcept {
    p_ = std::move(o.p_);
    cap_ = std::exchange(o.cap_, 0);
    return *this;
  }

  // frees the block, then allocates `bytes` (empty on failure)
  cudaError_t alloc(size_t bytes) {
    p_.reset();
    cap_ = 0;
    void* p = nullptr;
    const cudaError_t e = Alloc(&p, bytes);
    if (e != cudaSuccess) return e;
    p_.reset(static_cast<T*>(p));
    cap_ = bytes;
    return cudaSuccess;
  }
  // grow-only: when `need` bytes do not fit, frees the block, then allocates `bytes`
  cudaError_t reserve(size_t need, size_t bytes) { return need <= cap_ ? cudaSuccess : alloc(bytes); }
  T* get() const { return p_.get(); }

 private:
  struct Release { void operator()(T* p) const { Free(p); } };
  std::unique_ptr<T, Release> p_;
  size_t cap_ = 0;
};

template <class T = void>
using DeviceBuffer = CudaBuffer<T, cudaMalloc, cudaFree>;
template <class T = void>
using PinnedBuffer = CudaBuffer<T, cudaMallocHost, cudaFreeHost>;

struct CudaDestroy {
  void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
  void operator()(TcGemmPlan* p) const { tc_gemm_plan_destroy(p); }
  void operator()(TcAttnPlan* p) const { tc_attn_plan_destroy(p); }
  void operator()(TcFreqPlan* p) const { tc_freq_plan_destroy(p); }
  void operator()(TcFfPlan* p) const { tc_ff_plan_destroy(p); }
  void operator()(TcQkvPlan* p) const { tc_qkv_plan_destroy(p); }
};

using Event = std::unique_ptr<CUevent_st, CudaDestroy>;
using GemmPlan = std::unique_ptr<TcGemmPlan, CudaDestroy>;
using AttnPlan = std::unique_ptr<TcAttnPlan, CudaDestroy>;
using FreqPlan = std::unique_ptr<TcFreqPlan, CudaDestroy>;
using FfPlan = std::unique_ptr<TcFfPlan, CudaDestroy>;
using QkvPlan = std::unique_ptr<TcQkvPlan, CudaDestroy>;

}  // namespace bt
