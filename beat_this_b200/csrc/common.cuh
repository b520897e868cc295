// Shared device helpers for the sm_90a kernels: mbarrier and TMA wrappers (inline PTX), small math helpers.
// No torch, no CUTLASS.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace bt {

// 16-bit operand type of the tensor-core path (BT_DTYPE_H16).  Default: IEEE fp16 -- the dtype the reference's
// float16=True autocasts to on CUDA (beat_this/inference.py:245-246); every operand on this path is RMS-normalised,
// a folded weight, a softmax probability <= 2^8 or a GELU output, all far inside fp16 range, and its 11-bit
// significand cuts the logit error of the bf16 build ~8x at the same tensor-core rate.  -DBT_ACT_BF16 builds bf16.
#if defined(BT_ACT_BF16)
typedef __nv_bfloat16 h16;
#define BT_H16_IS_F16 0
#define BT_H16_MMA_SYNC "bf16.bf16"
#else
typedef __half h16;
#define BT_H16_IS_F16 1
#define BT_H16_MMA_SYNC "f16.f16"
#endif

__host__ __device__ constexpr int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ constexpr int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// exact-erf GELU (nn.GELU() default; reference roformer.py:50, beat_tracker.py:124,166)
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

template <typename T>
__device__ __forceinline__ T to_out(float v);
template <>
__device__ __forceinline__ float to_out<float>(float v) { return v; }
#if BT_H16_IS_F16
template <>
__device__ __forceinline__ h16 to_out<h16>(float v) { return __float2half_rn(v); }
__device__ __forceinline__ float to_f32(h16 v) { return __half2float(v); }
__device__ __forceinline__ uint32_t pack_h16x2(float lo, float hi) {
  __half2 p = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&p);
}
__device__ __forceinline__ void unpack_h16x2(uint32_t w, float& lo, float& hi) {
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w));
  lo = f.x; hi = f.y;
}
#else
__device__ __forceinline__ void unpack_h16x2(uint32_t w, float& lo, float& hi) {  // bf16 = the top half of an fp32
  lo = __uint_as_float(w << 16); hi = __uint_as_float(w & 0xffff0000u);
}
template <>
__device__ __forceinline__ h16 to_out<h16>(float v) { return __float2bfloat16_rn(v); }
__device__ __forceinline__ float to_f32(h16 v) { return __bfloat162float(v); }
__device__ __forceinline__ uint32_t pack_h16x2(float lo, float hi) {
  __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&p);
}
#endif
__device__ __forceinline__ float to_f32(float v) { return v; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ----------------------------------------------------------------------------- PTX: misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- PTX: mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a broken pipeline traps (-> CUDA error) instead of hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) {
      printf("bt: mbarrier timeout block (%d,%d,%d) thread %d\n", blockIdx.x, blockIdx.y,
             blockIdx.z, threadIdx.x);
      __trap();
    }
  }
}

// --- variants taking a precomputed 32-bit shared-space address (hot loops: the generic->shared
// conversion of a pointer costs several instructions per use) ---
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded spin that traps without a printf: a call (printf is one) in a kernel that issues wgmma makes ptxas
// serialise every wgmma of that kernel (C7510).  The trap still ends a broken pipeline in a launch error.
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) break;
    if (++spins > (1u << 26)) __trap();
  }
}
__device__ __forceinline__ void tma_load_3d_a(uint32_t smem_dst, const void* tmap, uint32_t bar, int32_t c0, int32_t c1,
                                              int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_f32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ float4 ld_shared_v4_f32(uint32_t addr) {
  float4 q;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(q.x), "=f"(q.y), "=f"(q.z), "=f"(q.w) : "r"(addr) : "memory");
  return q;
}
__device__ __forceinline__ float ld_shared_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// ----------------------------------------------------------------------------- PTX: TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

}  // namespace bt
