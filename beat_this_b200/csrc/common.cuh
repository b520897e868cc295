// Shared device helpers for the sm_90a kernels: mbarrier and TMA wrappers (inline PTX), small math helpers.
// No torch, no CUTLASS.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

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
#else
template <>
__device__ __forceinline__ h16 to_out<h16>(float v) { return __float2bfloat16_rn(v); }
__device__ __forceinline__ float to_f32(h16 v) { return __bfloat162float(v); }
__device__ __forceinline__ uint32_t pack_h16x2(float lo, float hi) {
  __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&p);
}
#endif

// Counter-based Philox4x32-10 (Salmon et al., SC'11; the rounds of curand's curand_Philox4x32_10): ten rounds of the
// two 32 x 32 -> 64-bit products, the key bumped by the Weyl constants between rounds.  Dropout masks are regenerated
// from it in every kernel that needs them (include/beatthis.h, "dropout masks").
__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = uint64_t{0xD2511F53u} * c.x, p1 = uint64_t{0xCD9E8D57u} * c.z;
    const uint32_t hi0 = static_cast<uint32_t>(p0 >> 32), lo0 = static_cast<uint32_t>(p0);
    const uint32_t hi1 = static_cast<uint32_t>(p1 >> 32), lo1 = static_cast<uint32_t>(p1);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ----------------------------------------------------------------------------- PTX: misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------- PTX: mbarrier
// The mbarrier and TMA wrappers take 32-bit shared-space addresses, computed once by the kernel: converting a generic
// pointer to one costs several instructions per use in the hot loops.
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded spin that traps without a printf: a call (printf is one) in a kernel that issues wgmma makes ptxas
// serialise every wgmma of that kernel (C7510).  The trap still ends a broken pipeline in a launch error.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
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

// ----------------------------------------------------------------------------- PTX: TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tmap, uint32_t bar, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const void* tmap, uint32_t bar, int32_t c0, int32_t c1,
                                            int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

}  // namespace bt
