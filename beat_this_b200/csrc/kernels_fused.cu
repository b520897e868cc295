// Persistent fused kernels for the narrow frontend sub-blocks (C = 32 / 64): [out-projection +] RMSNorm + FFN +
// residual (fused_ff_kernel) and RMSNorm + gates + QKV + RoPE (fused_qkv_kernel); reference
// roformer.py:38-61,114-128 as called by PartialFTTransformer, beat_tracker.py:290-301.
//
// Every weight matrix of the block is staged once per CTA into shared memory (rows padded by 16 bytes, so that the
// eight row addresses of each ldmatrix hit different bank groups).  A warp then owns 16 token rows at a time and does
// the whole block in registers with mma.sync m16n8k16 (16-bit operands, fp32 accumulate): each thread reads the fp32
// values of its two rows in the order of the MMA fragments, so the row it normalises is also the A operand, and for
// C <= 64 the accumulator of an N = C product holds exactly the columns the thread read.  The rows come from a
// per-warp stage in shared memory that cp.async fills with the warp's next 16 rows while it computes the current ones.
// Unfused, the FFN streams 32 bytes per element through HBM (norm 6 + ff1 10 + ff2 16); fused it is 8 (+2 for the out-projection input, +2 for the 16-bit copy).
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "tc_common.cuh"

namespace bt {

constexpr int FU_WARPS = 8;
constexpr int FU_THREADS = 32 * FU_WARPS;

// W [rows][cols] 16-bit row-major (global) -> shared memory with row stride cols + 8 elements
__device__ __forceinline__ void stage_weight(h16* dst, const h16* __restrict__ src, int rows, int cols) {
  const int vpr = cols / 8;  // 16-byte vectors per row
  for (int i = threadIdx.x; i < rows * vpr; i += blockDim.x) {
    const int r = i / vpr, v = i - r * vpr;
    *reinterpret_cast<uint4*>(dst + r * (cols + 8) + v * 8) = __ldg(reinterpret_cast<const uint4*>(src + static_cast<int64_t>(r) * cols) + v);
  }
}
// B fragments of out = A W^T, W staged at shared address sW with row stride LD elements.  b_frag_k2: output columns
// [8 nb, 8 nb + 8) at the k-steps ks (b[0], b[1]) and ks + 1 (b[2], b[3]); b_frag_n2: the column blocks nb (b[0], b[1])
// and nb + 1 (b[2], b[3]) at the k-step ks.  Lanes 8 i .. 8 i + 7 address the rows of 8 x 8 matrix i.
template <int LD>
__device__ __forceinline__ void b_frag_k2(uint32_t sW, int nb, int ks, int lane, uint32_t (&b)[4]) {
  ldmatrix_x4(sW + 2 * ((nb * 8 + (lane & 7)) * LD + ks * 16 + 8 * (lane >> 3)), b);
}
template <int LD>
__device__ __forceinline__ void b_frag_n2(uint32_t sW, int nb, int ks, int lane, uint32_t (&b)[4]) {
  ldmatrix_x4(sW + 2 * ((nb * 8 + (lane & 7) + 8 * (lane >> 4)) * LD + ks * 16 + 8 * ((lane >> 3) & 1)), b);
}

// Two 16-bit pairs of one row, lo at columns 8 nb + 2 q (+1) and hi at 8 (nb + 1) + 2 q (+1), spread over the lanes
// q = 0..3 of a quad: after one exchange with lane q ^ 1, lane q holds the 4 consecutive columns from
// 8 nb + quad_col(q), so the quad writes the row's 32 bytes of both blocks as one whole 32-byte sector, 8 bytes per
// lane.  Stored block by block, each warp store covered half of every sector it touched, and the QKV kernels ran at
// under half the HBM rate of the FFN kernels, whose fp32 stores cover whole sectors.
__device__ __forceinline__ int quad_col(int q) { return 8 * (q & 1) + 2 * (q & 2); }
__device__ __forceinline__ uint2 quad_pair(uint32_t lo, uint32_t hi, int q) {
  const uint32_t other = __shfl_xor_sync(0xffffffffu, (q & 1) ? lo : hi, 1);
  return (q & 1) ? make_uint2(other, hi) : make_uint2(lo, other);
}

// ---------------------------------------------------------------- per-warp row stage
// The 16 fp32 rows [16 g, 16 g + 16) of X [M][C], 8 floats of padding after every row but each fourth: the 4 rows of
// a half warp's float2 fragment read (8 consecutive floats each) start 8 banks apart, so the read hits 32 different
// banks.  Every index is the lane's own offset plus a constant, and the stage is 384 bytes smaller than with 8 floats
// after every row, which is what lets two CTAs of fused_ff_kernel<64, true> fit on an SM.
template <int C> __host__ __device__ constexpr int stage_floats() { return 16 * C + 96; }
template <int C>
__device__ __forceinline__ int stage_idx(int r, int col) { return r * C + 8 * (r & 3) + 24 * (r >> 2) + col; }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool ok) {  // !ok: 16 zero bytes, src unread
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
// Start loading group g into the stage at shared address st (rows >= M zero-filled; nothing for g past the last group).
// One commit group per call, so cp_async_wait_all waits for exactly this load.
template <int C>
__device__ __forceinline__ void stage_rows(uint32_t st, const float* __restrict__ X, int64_t g, int64_t ngroups,
                                           int64_t M, int lane) {
  constexpr int CPR = C / 4;  // 16-byte chunks per row
  if (g < ngroups) {
#pragma unroll
    for (int t = 0; t < 16 * CPR / 32; ++t) {
      const int r = (lane >> 3) + 4 * (t / (CPR / 8)), k = (lane & 7) + 8 * (t % (CPR / 8));
      cp_async16(st + 4 * stage_idx<C>(r, 4 * k), X + (g * 16 + r) * C + 4 * k, g * 16 + r < M);  // M <= row: no read
    }
  }
  cp_async_commit();
}
// the fragment-order float2 of row r (0..15) at column col (even) from the stage at shared address st
template <int C>
__device__ __forceinline__ float2 stage_f2(uint32_t st, int r, int col) {
  return ld_shared_v2_f32(st + 4 * stage_idx<C>(r, col));
}

// ==================================================================== fused frontend QKV projection
// gates = sigmoid(wg . rmsnorm(x) + bg) in fp32, qkv = RoPE(rmsnorm(x) Wqkv^T) (q also scaled) -> 16-bit.  HBM: 4 bytes
// in, 6 bytes out per element.
template <int C>
__global__ void __launch_bounds__(FU_THREADS, C == 32 ? 4 : 2)
fused_qkv_kernel(const h16* __restrict__ wqkv, const float* __restrict__ X, const float* __restrict__ wg,
                 const float* __restrict__ bg, const float* __restrict__ rope_cos, const float* __restrict__ rope_sin,
                 h16* __restrict__ qkv, float* __restrict__ gates, int64_t M, int L, int F, int posmode, float qscale) {
  constexpr int LD = C + 8, KS = C / 16, heads = C / 32;
  extern __shared__ uint4 fu_smem[];
  h16* sW = reinterpret_cast<h16*>(fu_smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q = lane & 3;
  const uint32_t sw = smem_u32(sW), st = sw + 2 * 3 * C * LD + 4 * warp * stage_floats<C>();  // st: this warp's row stage
  const int64_t ngroups = (M + 15) / 16;
  int64_t g = static_cast<int64_t>(blockIdx.x) * FU_WARPS + warp;
  stage_rows<C>(st, X, g, ngroups, M, lane);
  stage_weight(sW, wqkv, 3 * C, C);
  __syncthreads();
  for (; g < ngroups; g += static_cast<int64_t>(gridDim.x) * FU_WARPS) {
    int64_t m[2];
    bool ok[2];
    float xs[2][C / 4];  // xs[r][4 ks + 2 h + e] = x[row r][16 ks + 8 h + 2 q + e]
    cp_async_wait_all();
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      m[r] = g * 16 + (lane >> 2) + 8 * r;
      ok[r] = m[r] < M;
#pragma unroll
      for (int j = 0; j < C / 4; j += 2) {
        const float2 v = stage_f2<C>(st, (lane >> 2) + 8 * r, 16 * (j >> 2) + 8 * ((j >> 1) & 1) + 2 * q);
        xs[r][j] = v.x;
        xs[r][j + 1] = v.y;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {  // RMSNorm without gamma (folded into the weights); the quad holds the whole row
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < C / 4; ++j) ss = fmaf(xs[r][j], xs[r][j], ss);
      ss += __shfl_xor_sync(0xffffffffu, ss, 1);
      ss += __shfl_xor_sync(0xffffffffu, ss, 2);
      const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
      for (int j = 0; j < C / 4; ++j) xs[r][j] *= inv;
    }
#pragma unroll
    for (int h = 0; h < heads; ++h) {  // gates = sigmoid(to_gates(x_normed)) (gamma * sqrt(C) folded into wg)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float a = 0.f;
#pragma unroll
        for (int j = 0; j < C / 4; j += 2) {
          const float2 w = __ldg(reinterpret_cast<const float2*>(wg + h * C + 16 * (j >> 2) + 8 * ((j >> 1) & 1) + 2 * q));
          a = fmaf(xs[r][j], w.x, fmaf(xs[r][j + 1], w.y, a));
        }
        a += __shfl_xor_sync(0xffffffffu, a, 1);
        a += __shfl_xor_sync(0xffffffffu, a, 2);
        if (q == 0 && ok[r]) gates[m[r] * heads + h] = sigmoidf_(a + __ldg(bg + h));
      }
    }
    uint32_t a[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      a[ks][0] = pack_h16x2(xs[0][4 * ks], xs[0][4 * ks + 1]);
      a[ks][1] = pack_h16x2(xs[1][4 * ks], xs[1][4 * ks + 1]);
      a[ks][2] = pack_h16x2(xs[0][4 * ks + 2], xs[0][4 * ks + 3]);
      a[ks][3] = pack_h16x2(xs[1][4 * ks + 2], xs[1][4 * ks + 3]);
    }
    __syncwarp();  // every lane has read the stage: refill it with the next group while this one computes
    stage_rows<C>(st, X, g + static_cast<int64_t>(gridDim.x) * FU_WARPS, ngroups, M, lane);
    const float* cs[2];
    const float* sn[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {  // RoPE position of the row (interleaved pairs, rotary_embedding_torch semantics)
      const int pos = ok[r] ? (posmode == 0 ? static_cast<int>(m[r] % L) : static_cast<int>((m[r] / L) % F)) : 0;
      cs[r] = rope_cos + pos * 16;
      sn[r] = rope_sin + pos * 16;
    }
    // 0 q, 1 k, 2 v, C / 8 column blocks each, two at a time; not unrolled, so that the B fragments of all 3 C columns
    // are not loaded ahead at once (at C = 64 that spilled at the 128 registers of 2 CTAs per SM)
#pragma unroll 1
    for (int which = 0; which < 3; ++which)
#pragma unroll
    for (int nb = which * (C / 8); nb < (which + 1) * (C / 8); nb += 2) {
      float acc[2][4] = {};
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int ks = 0; ks < KS; ks += 2) {
          uint32_t b[4];
          b_frag_k2<LD>(sw, nb + u, ks, lane, b);
          mma_16816(acc[u], a[ks], b[0], b[1]);
          mma_16816(acc[u], a[ks + 1], b[2], b[3]);
        }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        uint32_t p[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int n = (nb + u) * 8 + 2 * q;
          float v0 = acc[u][2 * r], v1 = acc[u][2 * r + 1];
          if (which < 2) {
            const float sc = which == 0 ? qscale : 1.0f;
            const int i = ((n - which * C) & 31) >> 1;
            const float co = __ldg(cs[r] + i), si = __ldg(sn[r] + i);
            const float x0 = v0, x1 = v1;
            v0 = (x0 * co - x1 * si) * sc;
            v1 = (x1 * co + x0 * si) * sc;
          }
          p[u] = pack_h16x2(v0, v1);
        }
        const uint2 w = quad_pair(p[0], p[1], q);
        if (ok[r]) *reinterpret_cast<uint2*>(qkv + m[r] * (3 * C) + nb * 8 + quad_col(q)) = w;
      }
    }
  }
}

// ==================================================================== fused frontend FFN
// x += W2 gelu(W1 rmsnorm(x) + b1) + b2; with OP the preceding attention's out-projection runs in front
// (x' = x + O Wo^T, reference roformer.py:134-140, then the FFN on x').  The accumulator of the N = C products starts
// from the residual row, so the tensor core adds it.  Hidden units go 16 at a time: two 8-column blocks of
// rmsnorm(x') W1^T -> bias + GELU -> packed straight from the accumulator layout into the A operand of the W2
// product: the hidden activations never leave the registers.
template <int C, bool OP>
__global__ void __launch_bounds__(FU_THREADS, C == 32 ? 3 : 2)
fused_ff_kernel(const h16* __restrict__ w1, const h16* __restrict__ w2, const h16* __restrict__ wo,
                const h16* __restrict__ O, float* __restrict__ X, const float* __restrict__ b1,
                const float* __restrict__ b2, h16* __restrict__ xb_out, int64_t M) {
  constexpr int HID = 4 * C, LD1 = C + 8, LD2 = HID + 8, KS = C / 16, NB = C / 8, HS = HID / 16;
  extern __shared__ uint4 fu_smem[];
  h16* sW1 = reinterpret_cast<h16*>(fu_smem);  // [4C][C + 8]
  h16* sW2 = sW1 + HID * LD1;                   // [C][4C + 8]
  h16* sWo = sW2 + C * LD2;                     // [C][C + 8] (OP)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q = lane & 3;
  const uint32_t sw1 = smem_u32(sW1), sw2 = smem_u32(sW2), swo = smem_u32(sWo);
  const uint32_t st = swo + 2 * (OP ? C * LD1 : 0) + 4 * warp * stage_floats<C>();  // this warp's row stage
  const int64_t ngroups = (M + 15) / 16;
  int64_t g = static_cast<int64_t>(blockIdx.x) * FU_WARPS + warp;
  // O is not staged (at C = 64 the weights and the X stages leave no room for it): its rows go to L2 one group ahead
  auto prefetch_o = [&](int64_t gg) {
    if (OP && lane == 0 && gg < ngroups) {
      const int64_t rows = M - gg * 16 < 16 ? M - gg * 16 : 16;
      asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(O + gg * 16 * C), "r"(static_cast<uint32_t>(rows * C * 2))
                   : "memory");
    }
  };
  stage_rows<C>(st, X, g, ngroups, M, lane);
  prefetch_o(g);
  stage_weight(sW1, w1, HID, C);
  stage_weight(sW2, w2, C, HID);
  if constexpr (OP) stage_weight(sWo, wo, C, C);
  __syncthreads();
  for (; g < ngroups; g += static_cast<int64_t>(gridDim.x) * FU_WARPS) {
    int64_t m[2];
    bool ok[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      m[r] = g * 16 + (lane >> 2) + 8 * r;
      ok[r] = m[r] < M;
    }
    float acc[NB][4];  // columns 8 nb + 2 q + {0, 1} of rows r0 (acc[nb][0..1]) and r0 + 8 (acc[nb][2..3])
    cp_async_wait_all();
    __syncwarp();
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float2 v = stage_f2<C>(st, (lane >> 2) + 8 * r, nb * 8 + 2 * q);
        acc[nb][2 * r] = v.x;
        acc[nb][2 * r + 1] = v.y;
      }
    __syncwarp();  // every lane has read the stage: refill it with the next group while this one computes
    stage_rows<C>(st, X, g + static_cast<int64_t>(gridDim.x) * FU_WARPS, ngroups, M, lane);
    prefetch_o(g + static_cast<int64_t>(gridDim.x) * FU_WARPS);
    if constexpr (OP) {  // x' = x + O Wo^T, O (gated attention output, 16-bit) loaded in A-fragment order
      uint32_t ao[KS][4];
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = i & 1;
          ao[ks][i] = ok[r] ? *reinterpret_cast<const uint32_t*>(O + m[r] * C + ks * 16 + 8 * (i >> 1) + 2 * q) : 0u;
        }
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int ks = 0; ks < KS; ks += 2) {
          uint32_t b[4];
          b_frag_k2<LD1>(swo, nb, ks, lane, b);
          mma_16816(acc[nb], ao[ks], b[0], b[1]);
          mma_16816(acc[nb], ao[ks + 1], b[2], b[3]);
        }
    }
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float ss = 0.f;
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) ss = fmaf(acc[nb][2 * r], acc[nb][2 * r], fmaf(acc[nb][2 * r + 1], acc[nb][2 * r + 1], ss));
      ss += __shfl_xor_sync(0xffffffffu, ss, 1);
      ss += __shfl_xor_sync(0xffffffffu, ss, 2);
      inv[r] = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
    }
    uint32_t a[KS][4];  // rmsnorm(x') as the A operand: k-step ks covers accumulator blocks 2 ks and 2 ks + 1
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      a[ks][0] = pack_h16x2(acc[2 * ks][0] * inv[0], acc[2 * ks][1] * inv[0]);
      a[ks][1] = pack_h16x2(acc[2 * ks][2] * inv[1], acc[2 * ks][3] * inv[1]);
      a[ks][2] = pack_h16x2(acc[2 * ks + 1][0] * inv[0], acc[2 * ks + 1][1] * inv[0]);
      a[ks][3] = pack_h16x2(acc[2 * ks + 1][2] * inv[1], acc[2 * ks + 1][3] * inv[1]);
    }
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {  // + b2: the result accumulates on top of x' + b2
      const float2 b = __ldg(reinterpret_cast<const float2*>(b2 + nb * 8 + 2 * q));
      acc[nb][0] += b.x; acc[nb][1] += b.y;
      acc[nb][2] += b.x; acc[nb][3] += b.y;
    }
#pragma unroll 2
    for (int j = 0; j < HS; ++j) {  // hidden units [16 j, 16 j + 16)
      float hh[2][4];
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        hh[t][0] = hh[t][1] = hh[t][2] = hh[t][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < KS; ks += 2) {
          uint32_t b[4];
          b_frag_k2<LD1>(sw1, 2 * j + t, ks, lane, b);
          mma_16816(hh[t], a[ks], b[0], b[1]);
          mma_16816(hh[t], a[ks + 1], b[2], b[3]);
        }
        const float2 b = __ldg(reinterpret_cast<const float2*>(b1 + (2 * j + t) * 8 + 2 * q));
        hh[t][0] = gelu_tanh_fast(hh[t][0] + b.x); hh[t][1] = gelu_tanh_fast(hh[t][1] + b.y);
        hh[t][2] = gelu_tanh_fast(hh[t][2] + b.x); hh[t][3] = gelu_tanh_fast(hh[t][3] + b.y);
      }
      const uint32_t ah[4] = {pack_h16x2(hh[0][0], hh[0][1]), pack_h16x2(hh[0][2], hh[0][3]), pack_h16x2(hh[1][0], hh[1][1]),
                              pack_h16x2(hh[1][2], hh[1][3])};
#pragma unroll
      for (int nb = 0; nb < NB; nb += 2) {
        uint32_t b[4];
        b_frag_n2<LD2>(sw2, nb, j, lane, b);
        mma_16816(acc[nb], ah, b[0], b[1]);
        mma_16816(acc[nb + 1], ah, b[2], b[3]);
      }
    }
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (!ok[r]) continue;
        const int64_t o = m[r] * C + nb * 8 + 2 * q;
        *reinterpret_cast<float2*>(X + o) = make_float2(acc[nb][2 * r], acc[nb][2 * r + 1]);
        if (xb_out) *reinterpret_cast<uint32_t*>(xb_out + o) = pack_h16x2(acc[nb][2 * r], acc[nb][2 * r + 1]);
      }
  }
}

// weights, then one 16-row fp32 stage per warp
template <int C> constexpr int ff_smem(bool op) {
  return (4 * C * (C + 8) + C * (4 * C + 8) + (op ? C * (C + 8) : 0)) * 2 + FU_WARPS * stage_floats<C>() * 4;
}
template <int C> constexpr int qkv_smem() { return 3 * C * (C + 8) * 2 + FU_WARPS * stage_floats<C>() * 4; }
template <int C> constexpr int ff_ctas() { return C == 32 ? 3 : 2; }
template <int C> constexpr int qkv_ctas() { return C == 32 ? 4 : 2; }

struct TcFfPlan {
  const void *w1, *w2, *o, *wo;
  int C;
  int64_t M;
  bool outproj;
};

// o_h16 / wout_h16 != nullptr: plan for the variant with the attention out-projection fused in front
// (o_h16: gated attention output [M, C], wout_h16: [C, C]).
TcFfPlan* tc_ff_plan_create(const void* w1_h16, const void* w2_h16, int C, int64_t M, const void* o_h16,
                            const void* wout_h16, char* err, int errlen) {
  if (C != 32 && C != 64) { snprintf(err, errlen, "fused ff: C must be 32 or 64"); return nullptr; }
  TcFfPlan* p = new TcFfPlan();
  p->w1 = w1_h16; p->w2 = w2_h16; p->o = o_h16; p->wo = wout_h16;
  p->C = C; p->M = M; p->outproj = o_h16 != nullptr && wout_h16 != nullptr;
  return p;
}
void tc_ff_plan_destroy(TcFfPlan* p) { delete p; }

static unsigned fused_grid(int64_t M, int ctas_per_sm) {
  const int64_t ctas = ((M + 15) / 16 + FU_WARPS - 1) / FU_WARPS;
  const int64_t slots = static_cast<int64_t>(g_num_sms) * ctas_per_sm;  // persistent CTAs: weights staged once each
  return static_cast<unsigned>(ctas < slots ? ctas : slots);
}

void launch_fused_ff(const TcFfPlan* p, float* X, const float* b1, const float* b2, void* xb_out, cudaStream_t st) {
  const h16* w1 = static_cast<const h16*>(p->w1);
  const h16* w2 = static_cast<const h16*>(p->w2);
  const h16* wo = static_cast<const h16*>(p->wo);
  const h16* o = static_cast<const h16*>(p->o);
  h16* xb = static_cast<h16*>(xb_out);
#define BT_FF_L(CC, OPP)                                                                                            \
  fused_ff_kernel<CC, OPP><<<fused_grid(p->M, ff_ctas<CC>()), FU_THREADS, ff_smem<CC>(OPP), st>>>(w1, w2, wo, o, X, b1, \
                                                                                                  b2, xb, p->M)
  if (p->C == 32) { if (p->outproj) BT_FF_L(32, true); else BT_FF_L(32, false); }
  else { if (p->outproj) BT_FF_L(64, true); else BT_FF_L(64, false); }
#undef BT_FF_L
}

struct TcQkvPlan {
  const void* w;
  int C;
  int64_t M;
};
TcQkvPlan* tc_qkv_plan_create(const void* wqkv_h16, int C, int64_t M, char* err, int errlen) {
  if (C != 32 && C != 64) { snprintf(err, errlen, "fused qkv: C must be 32 or 64"); return nullptr; }
  TcQkvPlan* p = new TcQkvPlan();
  p->w = wqkv_h16; p->C = C; p->M = M;
  return p;
}
void tc_qkv_plan_destroy(TcQkvPlan* p) { delete p; }
void launch_fused_qkv(const TcQkvPlan* p, const float* X, const float* wg, const float* bg, const float* rope_cos,
                      const float* rope_sin, void* qkv, float* gates, int L, int F, int posmode, float qscale,
                      cudaStream_t st) {
  const h16* w = static_cast<const h16*>(p->w);
  h16* out = static_cast<h16*>(qkv);
  if (p->C == 32)
    fused_qkv_kernel<32><<<fused_grid(p->M, qkv_ctas<32>()), FU_THREADS, qkv_smem<32>(), st>>>(w, X, wg, bg, rope_cos, rope_sin, out,
                                                                                             gates, p->M, L, F, posmode, qscale);
  else
    fused_qkv_kernel<64><<<fused_grid(p->M, qkv_ctas<64>()), FU_THREADS, qkv_smem<64>(), st>>>(w, X, wg, bg, rope_cos, rope_sin, out,
                                                                                             gates, p->M, L, F, posmode, qscale);
}

// fused_ff_kernel<64, OP> needs the largest shared-memory carveout for its 2 CTAs per SM (2 x 113 KB + 1 KB reserved
// per CTA = 228 KB with OP); the others keep the default, which leaves L1 room for the RoPE tables and biases.
template <typename K>
static cudaError_t fused_attrs(K* kernel, int smem, bool max_carveout = false) {
  cudaError_t r = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (r == cudaSuccess && max_carveout)
    r = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  return r;
}

int tc_init_fused(char* err, int errlen) {
  cudaError_t r = fused_attrs(fused_ff_kernel<32, false>, ff_smem<32>(false));
  if (r == cudaSuccess) r = fused_attrs(fused_ff_kernel<64, false>, ff_smem<64>(false), true);
  if (r == cudaSuccess) r = fused_attrs(fused_ff_kernel<32, true>, ff_smem<32>(true));
  if (r == cudaSuccess) r = fused_attrs(fused_ff_kernel<64, true>, ff_smem<64>(true), true);
  if (r == cudaSuccess) r = fused_attrs(fused_qkv_kernel<32>, qkv_smem<32>());
  if (r == cudaSuccess) r = fused_attrs(fused_qkv_kernel<64>, qkv_smem<64>());
  if (r != cudaSuccess) {
    snprintf(err, errlen, "cudaFuncSetAttribute(fused_ff_kernel / fused_qkv_kernel) failed: %s", cudaGetErrorString(r));
    return -1;
  }
  return 0;
}

}  // namespace bt
