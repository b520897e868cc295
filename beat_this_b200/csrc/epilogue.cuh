// GEMM epilogues of the fp32 CUDA-core GEMM and the h16 wgmma GEMM.
// epilogue_apply (fp32 GEMM): a thread hands over four consecutive accumulator columns [n0, n0+4) of output row m;
// epi_bias_gelu / epi_resid / epi_rope / epi_gates_pair: two adjacent columns [n, n+1) (the wgmma accumulator fragment).
#pragma once
#include "bt_kernels.h"
#include <cuda_fp16.h>

#include "common.cuh"

namespace bt {

// erf by Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7) on the MUFU/FMA pipes: the tensor-core
// epilogue evaluates GELU for every FFN hidden element and erff()'s ~35 instructions made it
// issue-bound.  gelu(x) = 0.5 x (1 + erf(x / sqrt 2)).
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  p *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * z * -1.4426950408889634f));
  const float erf_abs = fmaf(-p, e, 1.0f);            // erf(|x|/sqrt2)
  return 0.5f * x + 0.5f * fabsf(x) * erf_abs;         // 0.5x(1 + sign(x) erf_abs)
}
// tanh-form GELU on one MUFU op: 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))).  Differs from
// the exact erf form by <= 5e-4 absolute (and tanh.approx adds ~5e-4): a quarter of a h16 ulp
// of the values it produces.  Used only by the h16 tensor-core path, whose FFN epilogues were
// issue/MUFU-bound on the 16-instruction + 2-MUFU erf evaluation above.
__device__ __forceinline__ float gelu_tanh_fast(float x) {
  const float u = x * fmaf(0.0356774081f, x * x, 0.7978845608f);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  const float hx = 0.5f * x;
  return fmaf(hx, t, hx);
}
template <typename TAct>
__device__ __forceinline__ float gelu_for(float x) {
  if constexpr (sizeof(TAct) == 2) return gelu_tanh_fast(x);
  else return gelu_erf(x);
}

__device__ __forceinline__ void store_f32x4(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
// n0 % 4 == 0; for kind 1 a head (32 columns) is never split across a q/k/v boundary because C % 32 == 0.
__device__ __forceinline__ void epilogue_apply(const EpiParams& e, int L, int64_t m, int n0, float (&v)[4]) {
  if (e.kind == 0) {
    if (e.bias) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(e.bias + n0));
      v[0] += q.x; v[1] += q.y; v[2] += q.z; v[3] += q.w;
    }
    if (e.gelu) {
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = gelu_erf(v[i]);
    }
    if (e.resid) {
      const float4 q = *reinterpret_cast<const float4*>(e.resid + m * e.ldr + n0);
      v[0] += q.x; v[1] += q.y; v[2] += q.z; v[3] += q.w;
    }
    if (e.out_f32) store_f32x4(e.out_f32 + m * e.ldo_f32 + n0, v);
    if (e.out_act) store_f32x4(reinterpret_cast<float*>(e.out_act) + m * e.ldo_act + n0, v);
  } else if (e.kind == 2) {
    // attention gates (reference roformer.py:127-128): sigmoid(to_gates(x_normed)), N padded to 32
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (n0 + i < e.heads) e.out_f32[m * e.heads + n0 + i] = sigmoidf_(v[i] + __ldg(e.bias + n0 + i));
  } else {
    // qkv: RoPE on interleaved pairs (rotary_embedding_torch semantics, reference
    // roformer.py:121-123): out[2i] = x[2i] cos - x[2i+1] sin ; out[2i+1] = x[2i+1] cos + x[2i] sin
    const int which = n0 / e.C;          // 0 q, 1 k, 2 v
    float* dst = reinterpret_cast<float*>(e.out_act) + m * e.ldo_act + n0;
    // the store sits in both branches: hoisted after them, it changes ptxas's register allocation of the whole GEMM
    if (which < 2) {
      const float sc = which == 0 ? e.qscale : 1.0f;
      const int c = n0 - which * e.C;
      const int pos = e.posmode == 0 ? static_cast<int>(m % L) : static_cast<int>((m / L) % e.F);
      const float* cs = e.rope_cos + pos * 16 + ((c & 31) >> 1);
      const float* sn = e.rope_sin + pos * 16 + ((c & 31) >> 1);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float co = __ldg(cs + i), si = __ldg(sn + i);
        const float x0 = v[2 * i], x1 = v[2 * i + 1];
        v[2 * i] = (x0 * co - x1 * si) * sc;
        v[2 * i + 1] = (x1 * co + x0 * si) * sc;
      }
      store_f32x4(dst, v);
    } else {
      store_f32x4(dst, v);
    }
  }
}

// The same operations for the column pair (n, n + 1), n even, the pair a thread of a wgmma accumulator fragment holds.
// The 16-bit GEMM applies them to its accumulators in place; kinds 0 and 1 then stage the values through shared memory
// (fp32 as they are, 16-bit through pack_h16x2), the gates (kind 2) store straight from registers.
// Kind 0, in this order: bias, GELU, then the fp32 residual (epi_resid).
template <typename TAct>
__device__ __forceinline__ void epi_bias_gelu(const EpiParams& e, int n, float& v0, float& v1) {
  if (e.bias) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(e.bias + n));
    v0 += b.x; v1 += b.y;
  }
  if (e.gelu) { v0 = gelu_for<TAct>(v0); v1 = gelu_for<TAct>(v1); }
}
__device__ __forceinline__ void epi_resid(float& v0, float& v1, float2 r) { v0 += r.x; v1 += r.y; }
// Kind 1: the pair is one interleaved RoPE pair and (co, si) its rotation at the row's position, read once per row by
// the caller; q columns are also scaled by qscale, v columns pass unchanged.
__device__ __forceinline__ void epi_rope(const EpiParams& e, int n, float& v0, float& v1, float co, float si) {
  const int which = n / e.C;  // 0 q, 1 k, 2 v
  if (which < 2) {
    const float sc = which == 0 ? e.qscale : 1.0f;
    const float x0 = v0, x1 = v1;
    // (x0 co - x1 si) sc and (x1 co + x0 si) sc with the fused multiply-adds written out: left to the compiler, which
    // product gets fused changes with the surrounding code, and with it the last bit of q and k
    v0 = fmaf(x0, co, -__fmul_rn(x1, si)) * sc;
    v1 = fmaf(x1, co, __fmul_rn(x0, si)) * sc;
  }
}
// Kind 2 (attention gates) of output row m, stored from registers.  Only the gates instantiation contains the IEEE
// division of sigmoidf_, whose slow path is a function call.
__device__ __forceinline__ void epi_gates_pair(const EpiParams& e, int64_t m, int n, float v0, float v1) {
  if (n < e.heads) e.out_f32[m * e.heads + n] = sigmoidf_(v0 + __ldg(e.bias + n));
  if (n + 1 < e.heads) e.out_f32[m * e.heads + n + 1] = sigmoidf_(v1 + __ldg(e.bias + n + 1));
}

}  // namespace bt
