// The model's HBM-bound row kernels (stem conv, zero tail, RMSNorm(+gates)), both frequency-direction attentions,
// head + aggregation scatter, peak picking, the f32 <-> 16-bit conversions and the QKV packing of the test hooks.
#include <cuda_fp16.h>
#include <cstdio>
#include <cstdlib>

#include "bt_kernels.h"
#include "common.cuh"
#include "tc_common.cuh"

namespace bt {

// ------------------------------------------------------------------------------------------
// stem: BN1d(128) -> Conv2d(1->32, k(4,3), s(4,1), p(0,1), no bias) -> BN2d -> GELU
// (reference beat_tracker.py:108-126).  BN2d is folded into w/bias on the host; BN1d cannot
// be folded (the conv's time padding is zero *after* BN1d) and is applied to each tap.
// Chunks are gathered straight from the per-clip spectrograms (split_piece/zeropad,
// inference.py:90-135): frames outside the clip are zero *before* BN1d.
// out: [B, 32 f, L, 32 c] fp32.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
stem_kernel(const float* __restrict__ spect, const ChunkSrc* __restrict__ chunks, int L,
            const float* __restrict__ bn1_scale, const float* __restrict__ bn1_shift,
            const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ out) {
  __shared__ float ws[32 * 12];
  __shared__ float bs[32];
  for (int i = threadIdx.x; i < 32 * 12; i += 128) ws[i] = w[i];
  if (threadIdx.x < 32) bs[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int t = blockIdx.x * 128 + threadIdx.x;  // frames t and t ^ 1 are neighbouring lanes
  const int f = blockIdx.y;
  const int b = blockIdx.z;
  const ChunkSrc cs = chunks[b];  // t >= L: computed (its loads stay inside the clip) but not stored
  float in[4][3];
#pragma unroll
  for (int dt = 0; dt < 3; ++dt) {
    const int tl = t + dt - 1;
    const bool conv_ok = tl >= 0 && tl < cs.len;  // zero padding of the convolution at the ends of THIS chunk
    const int64_t fr = static_cast<int64_t>(cs.start) + tl;
    const bool clip_ok = fr >= 0 && fr < cs.T;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (conv_ok && clip_ok)
      v = *reinterpret_cast<const float4*>(spect + (cs.frame_base + fr) * 128 + 4 * f);
    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int df = 0; df < 4; ++df)
      in[df][dt] = conv_ok ? fmaf(vv[df], bn1_scale[4 * f + df], bn1_shift[4 * f + df]) : 0.f;
  }
  // Channels go 8 at a time, one 32-byte sector of the frame's row.  The lanes of frames t and t ^ 1 swap half of their
  // 8 values, then each store of the pair writes one whole sector: first frame t & ~1's, then frame t | 1's, the even
  // lane channels 8 c8 .. + 3 and the odd lane 8 c8 + 4 .. + 7.  (A lane's own 16-byte stores would cover half of
  // every sector they touch, which makes L2 read the sector from HBM before it merges the write.)
  const bool odd = t & 1;
  float* op = out + ((static_cast<int64_t>(b) * 32 + f) * L + (t & ~1)) * 32 + (odd ? 4 : 0);
#pragma unroll
  for (int c8 = 0; c8 < 4; ++c8) {
    float r[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int co = c8 * 8 + i;
      float a = bs[co];
#pragma unroll
      for (int df = 0; df < 4; ++df)
#pragma unroll
        for (int dt = 0; dt < 3; ++dt) a = fmaf(in[df][dt], ws[co * 12 + df * 3 + dt], a);
      r[i] = gelu_fast(a);  // erf to 1.5e-7 on rcp + ex2 (erff: ~35 instructions, 32 of them per thread here)
    }
    float x[4];  // the partner's values: the even lane gets channels 8 c8 .. + 3 of frame t | 1, the odd lane
                 // 8 c8 + 4 .. + 7 of frame t & ~1
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = __shfl_xor_sync(0xffffffffu, odd ? r[i] : r[4 + i], 1);
    const float4 lo = odd ? make_float4(x[0], x[1], x[2], x[3]) : make_float4(r[0], r[1], r[2], r[3]);
    const float4 hi = odd ? make_float4(r[4], r[5], r[6], r[7]) : make_float4(x[0], x[1], x[2], x[3]);
    if ((t & ~1) < L) reinterpret_cast<float4*>(op + 8 * c8)[0] = lo;
    if ((t | 1) < L) reinterpret_cast<float4*>(op + 32 + 8 * c8)[0] = hi;
  }
}

__global__ void __launch_bounds__(256)
zero_tail_kernel(uint4* __restrict__ buf, const ChunkSrc* __restrict__ chunks, int F, int L, int row_vec) {
  const int plane = blockIdx.x;
  const int len = chunks[plane / F].len;
  const int64_t n = static_cast<int64_t>(L - len) * row_vec;  // 16-byte vectors to clear
  uint4* p = buf + (static_cast<int64_t>(plane) * L + len) * row_vec;
  for (int64_t i = threadIdx.x; i < n; i += 256) p[i] = make_uint4(0u, 0u, 0u, 0u);
}
void launch_zero_tail(void* buf, int elem_bytes, const ChunkSrc* chunks, int nchunks, int F, int L, int C, cudaStream_t st) {
  zero_tail_kernel<<<nchunks * F, 256, 0, st>>>(reinterpret_cast<uint4*>(buf), chunks, F, L, C * elem_bytes / 16);
}

void launch_stem(const float* spect, const ChunkSrc* chunks, int nchunks, int L, const float* bn1_scale,
                 const float* bn1_shift, const float* w, const float* bias, float* out,
                 cudaStream_t st) {
  dim3 grid(ceil_div(L, 128), 32, nchunks);
  stem_kernel<<<grid, 128, 0, st>>>(spect, chunks, L, bn1_scale, bn1_shift, w, bias, out);
}

// ------------------------------------------------------------------------------------------
// RMSNorm (reference roformer.py:22-32: x / max(||x||, 1e-12) * sqrt(dim) * gamma; the
// sqrt(dim)*gamma factor is folded into the consuming weights).  Pure HBM streaming:
// 4 B read + sizeof(TAct) B written per element.  A row is handled by C/4 (<= 32) lanes with
// float4 loads; several rows share a warp when C < 128.
// ------------------------------------------------------------------------------------------
template <typename TAct, int C>
__global__ void __launch_bounds__(256)
norm_kernel(const float* __restrict__ x, TAct* __restrict__ xn, int64_t M, float* __restrict__ gates,
            const float* __restrict__ wg, const float* __restrict__ bg, int heads) {
  constexpr int LPR = C / 4 < 32 ? C / 4 : 32;  // lanes per row
  constexpr int RPW = 32 / LPR;                 // rows per warp
  constexpr int VPL = C / 4 / LPR;              // float4 per lane
  const int lane = threadIdx.x & 31;
  const int64_t warp = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int64_t row = warp * RPW + lane / LPR;
  const int li = lane % LPR;
  const bool ok = row < M;
  const float4* xr = reinterpret_cast<const float4*>(x + (ok ? row : 0) * C);
  float4 v[VPL];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    v[i] = xr[li + LPR * i];
    ss = fmaf(v[i].x, v[i].x, ss); ss = fmaf(v[i].y, v[i].y, ss);
    ss = fmaf(v[i].z, v[i].z, ss); ss = fmaf(v[i].w, v[i].w, ss);
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
  for (int i = 0; i < VPL; ++i) { v[i].x *= inv; v[i].y *= inv; v[i].z *= inv; v[i].w *= inv; }
  if (gates) {
    // attention gates sigmoid(to_gates(x_normed)) (reference roformer.py:127-128) for the few-head
    // frontend attentions (1, 2 or 4 heads): a handful of FMAs per row inside this HBM-bound kernel
    // instead of a separate padded-N GEMM launch over the same rows.
    for (int h = 0; h < heads; ++h) {
      const float4* w4 = reinterpret_cast<const float4*>(wg + h * C);
      float a = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const float4 w = __ldg(w4 + li + LPR * i);
        a = fmaf(v[i].x, w.x, a); a = fmaf(v[i].y, w.y, a); a = fmaf(v[i].z, w.z, a); a = fmaf(v[i].w, w.w, a);
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (ok && li == 0) gates[row * heads + h] = sigmoidf_(a + __ldg(bg + h));
    }
  }
  if (!ok) return;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    TAct* dst = xn + row * C + 4 * (li + LPR * i);
    if constexpr (sizeof(TAct) == 4) {
      *reinterpret_cast<float4*>(dst) = v[i];
    } else {
      uint2 u;
      u.x = pack_h16x2(v[i].x, v[i].y);
      u.y = pack_h16x2(v[i].z, v[i].w);
      *reinterpret_cast<uint2*>(dst) = u;
    }
  }
}

template <typename TAct>
static void norm_dispatch(const float* x, void* xn, int64_t M, int C, float* gates, const float* wg, const float* bg,
                          int heads, cudaStream_t st) {
  TAct* o = reinterpret_cast<TAct*>(xn);
#define BT_NORM_CASE(c)                                                                                   \
  case c: {                                                                                               \
    constexpr int rpw = (c / 4 < 32) ? 32 / (c / 4) : 1;                                                  \
    norm_kernel<TAct, c><<<static_cast<unsigned>(ceil_div64(M, 8 * rpw)), 256, 0, st>>>(x, o, M, gates, wg, \
                                                                                          bg, heads);     \
  } break;
  switch (C) {
    BT_NORM_CASE(32) BT_NORM_CASE(64) BT_NORM_CASE(128) BT_NORM_CASE(256) BT_NORM_CASE(512) BT_NORM_CASE(1024)
    default: break;  // validated in bt_create
  }
#undef BT_NORM_CASE
}

void launch_norm(const float* x, void* xn, int64_t M, int C, int act_h16, cudaStream_t st, float* gates,
                 const float* wg, const float* bg, int heads) {
  if (act_h16) norm_dispatch<h16>(x, xn, M, C, gates, wg, bg, heads, st);
  else norm_dispatch<float>(x, xn, M, C, gates, wg, bg, heads, st);
}

// ------------------------------------------------------------------------------------------
// frequency-direction attention (PartialFTTransformer attnF, reference
// beat_tracker.py:292-294): sequences of F in {32,16,8} tokens over the frequency axis for
// every (chunk, frame, head).  Token m = (b*F + f)*L + t.  A warp handles 32/F groups
// (b,t,h) at once: lane -> (group g = lane / F, token f = lane % F).  Each lane loads its own
// q/k/v rows with 16-byte loads, K/V are shared through padded shared memory (float4
// broadcast reads).  HBM bytes: 3C in + C out per token (fp32).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_row32(const float* p, float (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 q = reinterpret_cast<const float4*>(p)[i];
    v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w;
  }
}

template <int F>
__global__ void __launch_bounds__(128, 4)
attn_freq_kernel(const float* __restrict__ qkv, const float* __restrict__ gates, float* __restrict__ out,
                 int B, int L, int heads, float scale) {
  constexpr int GPW = 32 / F;
  constexpr int RS = 36;               // padded row stride (floats)
  constexpr int GS = F * RS + 4;       // group stride: skews groups onto different banks
  __shared__ __align__(16) float Ks[4][GPW * GS];
  __shared__ __align__(16) float Vs[4][GPW * GS];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / F, f = lane % F;
  const int64_t ngrp = static_cast<int64_t>(B) * L * heads;
  const int64_t grp0 = (static_cast<int64_t>(blockIdx.x) * 4 + wib) * GPW;
  if (grp0 >= ngrp) return;  // warp-uniform
  const int64_t grp = grp0 + g;
  const bool act = grp < ngrp;
  const int64_t gg = act ? grp : grp0;
  const int h = static_cast<int>(gg % heads);
  const int64_t bt_ = gg / heads;
  const int t = static_cast<int>(bt_ % L);
  const int b = static_cast<int>(bt_ / L);
  const int C = heads * 32;
  const int64_t m = (static_cast<int64_t>(b) * F + f) * L + t;
  const float* rp = qkv + m * 3 * C + h * 32;
  float q[32];
  {
    float kv[32];
    load_row32(rp + C, kv);
    float* kd = &Ks[wib][g * GS + f * RS];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      reinterpret_cast<float4*>(kd)[i] = make_float4(kv[4 * i], kv[4 * i + 1], kv[4 * i + 2], kv[4 * i + 3]);
    load_row32(rp + 2 * C, kv);
    float* vd = &Vs[wib][g * GS + f * RS];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      reinterpret_cast<float4*>(vd)[i] = make_float4(kv[4 * i], kv[4 * i + 1], kv[4 * i + 2], kv[4 * i + 3]);
    load_row32(rp, q);
#pragma unroll
    for (int d = 0; d < 32; ++d) q[d] *= scale;
  }
  __syncwarp();
  const float* kb = &Ks[wib][g * GS];
  const float* vb = &Vs[wib][g * GS];
  float s[F];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < F; ++j) {
    float a = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 k4 = reinterpret_cast<const float4*>(kb + j * RS)[i];
      a = fmaf(q[4 * i], k4.x, a); a = fmaf(q[4 * i + 1], k4.y, a);
      a = fmaf(q[4 * i + 2], k4.z, a); a = fmaf(q[4 * i + 3], k4.w, a);
    }
    s[j] = a;
    mx = fmaxf(mx, a);
    asm volatile("" ::: "memory");  // keep ptxas from hoisting every K row into registers (spills)
  }
  float l = 0.f;
#pragma unroll
  for (int j = 0; j < F; ++j) {
    s[j] = __expf(s[j] - mx);
    l += s[j];
  }
  float o[32];
#pragma unroll
  for (int d = 0; d < 32; ++d) o[d] = 0.f;
#pragma unroll
  for (int j = 0; j < F; ++j) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 v4 = reinterpret_cast<const float4*>(vb + j * RS)[i];
      o[4 * i] = fmaf(s[j], v4.x, o[4 * i]); o[4 * i + 1] = fmaf(s[j], v4.y, o[4 * i + 1]);
      o[4 * i + 2] = fmaf(s[j], v4.z, o[4 * i + 2]); o[4 * i + 3] = fmaf(s[j], v4.w, o[4 * i + 3]);
    }
    asm volatile("" ::: "memory");
  }
  if (act) {
    const float gsc = gates[m * heads + h] / l;
    float* op = out + m * C + h * 32;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      reinterpret_cast<float4*>(op)[i] = make_float4(o[4 * i] * gsc, o[4 * i + 1] * gsc, o[4 * i + 2] * gsc, o[4 * i + 3] * gsc);
  }
}

// h16 path: the same attention on warp-level tensor-core MMAs (mma.sync m16n8k16, fp32 accumulate).
// A warp stages 32 rows (32/F groups: q | k | v, 64 bytes each) in shared memory with the coalesced
// row-per-lane loads of the SIMT kernel, then works on two 16-row query tiles: S = Q K^T from
// ldmatrix fragments, softmax in the accumulator layout (row reductions over the 4 lanes of a quad),
// P re-packed in registers as the A operand of P V (V through ldmatrix.trans).  F = 32: a tile sees
// all 32 keys; F = 16: a tile is one group; F = 8: a tile holds two groups, the cross blocks are
// masked.  ~40 tensor instructions per warp instead of ~4000 FMAs per lane.

// Tile = FT_TT consecutive frames of one chunk, all F frequency planes, all heads: ONE TMA box per (q|k|v, head)
// brings [TT][F][32] fp16 into shared memory (SWIZZLE_64B; the tensor map lists the plane dimension before the frame
// dimension, so the F rows one attention group reads are CONSECUTIVE 64-byte rows and ldmatrix is conflict free --
// with [F][TT] order the eight rows of an ldmatrix phase were 256 B apart: 4-way conflicts, L1 data pipe 82 % in
// ncu) and one box stores the [TT][F][C] output tile.  (Before: every lane fetched its own
// row, L * 3C elements away from its neighbour's -- 32 lines per ld.global, L1 wavefronts 73-87 % in ncu.)
constexpr int FT_TT = 4;

template <int F>
__global__ void __launch_bounds__(128)
attn_freq_mma_kernel(const __grid_constant__ CUtensorMap tmIn, const __grid_constant__ CUtensorMap tmOut,
                     const float* __restrict__ gates, int L, int heads, float scale_log2) {
  constexpr int GPW = 32 / F;             // groups (frame, head) per warp
  constexpr int NT = F == 32 ? 4 : 2;     // 8-key tiles a query tile attends to
  constexpr int HEADS = 4 * GPW / FT_TT;  // 1, 2, 4 for F = 32, 16, 8: the four warps cover TT frames x HEADS heads
  constexpr int C = HEADS * 32;
  constexpr int PH_BYTES = F * FT_TT * 64;  // one (part, head) box
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sIn = sbase;                                  // [3 parts][HEADS][F * TT rows][64 B]
  const uint32_t sOut = sIn + 3 * HEADS * PH_BYTES;            // [F * TT rows][C * 2 B], dense
  const uint32_t bar = sOut + F * FT_TT * C * 2;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t0 = blockIdx.x * FT_TT, b = blockIdx.y;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
    mbar_expect_tx(bar, 3 * HEADS * PH_BYTES);
    for (int part = 0; part < 3; ++part)
      for (int h = 0; h < HEADS; ++h)
        tma_load_3d(sIn + (part * HEADS + h) * PH_BYTES, &tmIn, bar, part * C + h * 32, b * F, t0);
  }
  __syncthreads();
  mbar_wait(bar, 0);
  // this warp's groups: head h, frames tt_base .. tt_base + GPW - 1; "staged row" r = gl * F + f as before
  const int h = (wib * GPW) / FT_TT;
  const int tt_base = (wib * GPW) % FT_TT;
  auto row_addr = [&](uint32_t base, int r, int chunk) -> uint32_t {  // 16-byte chunk `chunk` of staged row r
    const int row = tt_base * F + r;  // = (tt_base + r / F) * F + r % F
    return base + row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4);
  };
  const uint32_t sQ = sIn + (0 * HEADS + h) * PH_BYTES, sK = sIn + (1 * HEADS + h) * PH_BYTES, sV = sIn + (2 * HEADS + h) * PH_BYTES;
  const int g = lane >> 2, c = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
    const int key_base = F == 32 ? 0 : 16 * mt;
    uint32_t qa[2][4];
#pragma unroll
    for (int kk = 0; kk < 2; ++kk)
      ldmatrix_x4(row_addr(sQ, 16 * mt + (lane & 7) + ((lane >> 3) & 1) * 8, kk * 2 + (lane >> 4)), qa[kk]);
    float sc[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.f;
      uint32_t kb[4];
      ldmatrix_x4(row_addr(sK, key_base + 8 * j + (lane & 7), lane >> 3), kb);
      mma_16816(sc[j], qa[0], kb[0], kb[1]);
      mma_16816(sc[j], qa[1], kb[2], kb[3]);
    }
    if (F == 8) {  // rows 0-7 belong to the tile's first group (keys of tile 0), rows 8-15 to the second
      sc[1][0] = sc[1][1] = -INFINITY;
      sc[0][2] = sc[0][3] = -INFINITY;
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      mx0 = fmaxf(mx0, fmaxf(sc[j][0], sc[j][1]));
      mx1 = fmaxf(mx1, fmaxf(sc[j][2], sc[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      sc[j][0] = exp2f((sc[j][0] - mx0) * scale_log2); sc[j][1] = exp2f((sc[j][1] - mx0) * scale_log2);
      sc[j][2] = exp2f((sc[j][2] - mx1) * scale_log2); sc[j][3] = exp2f((sc[j][3] - mx1) * scale_log2);
      l0 += sc[j][0] + sc[j][1];
      l1 += sc[j][2] + sc[j][3];
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    float o[4][4];
#pragma unroll
    for (int jd = 0; jd < 4; ++jd) o[jd][0] = o[jd][1] = o[jd][2] = o[jd][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < NT / 2; ++kk) {
      uint32_t pa[4];
      pa[0] = pack_h16x2(sc[2 * kk][0], sc[2 * kk][1]);
      pa[1] = pack_h16x2(sc[2 * kk][2], sc[2 * kk][3]);
      pa[2] = pack_h16x2(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
      pa[3] = pack_h16x2(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
#pragma unroll
      for (int jd = 0; jd < 4; jd += 2) {
        uint32_t vb[4];
        const int q4 = lane >> 3;
        ldmatrix_x4_trans(row_addr(sV, key_base + 16 * kk + (q4 & 1) * 8 + (lane & 7), jd + (q4 >> 1)), vb);
        mma_16816(o[jd], pa, vb[0], vb[1]);
        mma_16816(o[jd + 1], pa, vb[2], vb[3]);
      }
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int r = 16 * mt + g + 8 * half;
      const int f = r % F, tt = tt_base + r / F;
      const int t = t0 + tt;
      const int64_t m = (static_cast<int64_t>(b) * F + f) * L + (t < L ? t : L - 1);
      const float gsc = gates[m * HEADS + h] / (half == 0 ? l0 : l1);
      const uint32_t orow = sOut + (tt * F + f) * (C * 2) + h * 64;
#pragma unroll
      for (int jd = 0; jd < 4; ++jd)
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(orow + (4 * jd + c) * 4), "r"(pack_h16x2(o[jd][2 * half] * gsc, o[jd][2 * half + 1] * gsc)) : "memory");
    }
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (threadIdx.x == 0) {
    tma_store_3d(&tmOut, sOut, 0, b * F, t0);  // frames beyond L are clipped
    bulk_commit();
    bulk_wait_read<0>();
  }
}

// The (F, heads) pairs of the frontend blocks: the four warps of a CTA cover FT_TT frames x 32 / F heads.
#define BT_FREQ_TC_INSTANCES(X) X(32) X(16) X(8)
template <int F> constexpr int freq_tc_heads() { return 4 * (32 / F) / FT_TT; }
template <int F> constexpr int freq_tc_smem() {
  return 3 * freq_tc_heads<F>() * F * FT_TT * 64 + F * FT_TT * freq_tc_heads<F>() * 32 * 2 + 1024 + 64;
}

struct TcFreqPlan {
  CUtensorMap tmIn;   // qkv [B * F planes, L, 3C], boxes of FT_TT frames x F planes x one head
  CUtensorMap tmOut;  // out [B * F planes, L, C], boxes of FT_TT frames x F planes x C
  int B, F, L;
};

TcFreqPlan* tc_freq_plan_create(const void* qkv, void* out, int B, int F, int L, int heads, char* err, int errlen) {
  bool ok = false;
#define BT_FREQ_OK(FF) ok = ok || (F == FF && heads == freq_tc_heads<FF>());
  BT_FREQ_TC_INSTANCES(BT_FREQ_OK)
#undef BT_FREQ_OK
  if (!ok) {
    snprintf(err, errlen, "frequency attention: no tensor-core kernel for F = %d with %d heads (F = 32, 16, 8 take 1, 2, 4 "
             "heads)", F, heads);
    return nullptr;
  }
  TcFreqPlan* p = new TcFreqPlan();
  p->B = B; p->F = F; p->L = L;
  const int C = heads * 32;
  // dimension order (channels, planes, frames): the plane stride is the larger one
  const uint64_t din[3] = {static_cast<uint64_t>(3 * C), static_cast<uint64_t>(B) * F, static_cast<uint64_t>(L)};
  const uint64_t sin_[2] = {static_cast<uint64_t>(L) * 3 * C * 2, static_cast<uint64_t>(3 * C) * 2};
  const uint32_t bin[3] = {32, static_cast<uint32_t>(F), FT_TT};
  const uint64_t dout[3] = {static_cast<uint64_t>(C), static_cast<uint64_t>(B) * F, static_cast<uint64_t>(L)};
  const uint64_t sout[2] = {static_cast<uint64_t>(L) * C * 2, static_cast<uint64_t>(C) * 2};
  const uint32_t bout[3] = {static_cast<uint32_t>(C), static_cast<uint32_t>(F), FT_TT};
  if (!make_tmap(&p->tmIn, qkv, 3, din, sin_, bin, 64, err, errlen) || !make_tmap(&p->tmOut, out, 3, dout, sout, bout, 0, err, errlen)) {
    delete p;
    return nullptr;
  }
  return p;
}
void tc_freq_plan_destroy(TcFreqPlan* p) { delete p; }

void launch_attn_freq_tc(const TcFreqPlan* p, const float* gates, float scale, cudaStream_t st) {
  const float sl2 = scale * 1.4426950408889634f;
  const dim3 grid(ceil_div(p->L, FT_TT), p->B);
#define BT_FREQ_LAUNCH(FF)                                                                                             \
  if (p->F == FF)                                                                                                      \
    attn_freq_mma_kernel<FF><<<grid, 128, freq_tc_smem<FF>(), st>>>(p->tmIn, p->tmOut, gates, p->L, freq_tc_heads<FF>(), sl2);
  BT_FREQ_TC_INSTANCES(BT_FREQ_LAUNCH)
#undef BT_FREQ_LAUNCH
}

int tc_init_attn_freq(char* err, int errlen) {
  cudaError_t r = cudaSuccess;
#define BT_FREQ_ATTR(FF) \
  if (r == cudaSuccess) r = cudaFuncSetAttribute(attn_freq_mma_kernel<FF>, cudaFuncAttributeMaxDynamicSharedMemorySize, freq_tc_smem<FF>());
  BT_FREQ_TC_INSTANCES(BT_FREQ_ATTR)
#undef BT_FREQ_ATTR
  if (r != cudaSuccess) {
    snprintf(err, errlen, "cudaFuncSetAttribute(attn_freq_mma_kernel) failed: %s", cudaGetErrorString(r));
    return -1;
  }
  return 0;
}

void launch_attn_freq_simt(const float* qkv, const float* gates, float* out, int B, int F, int L, int heads, float scale,
                           cudaStream_t st) {
  const int64_t ngrp = static_cast<int64_t>(B) * L * heads;
  const unsigned grid = static_cast<unsigned>(ceil_div64(ngrp, 4 * (32 / F)));
  if (F == 32) attn_freq_kernel<32><<<grid, 128, 0, st>>>(qkv, gates, out, B, L, heads, scale);
  else if (F == 16) attn_freq_kernel<16><<<grid, 128, 0, st>>>(qkv, gates, out, B, L, heads, scale);
  else attn_freq_kernel<8><<<grid, 128, 0, st>>>(qkv, gates, out, B, L, heads, scale);
}

// ------------------------------------------------------------------------------------------
// head: final RMSNorm (roformer.py:174,180; gamma*sqrt(D) folded into w) -> Linear(D->2) ->
// SumHead (beat = o0 + o1 in fp32, downbeat = o1; beat_tracker.py:315-330) -> scatter into
// the per-clip frame arrays with aggregate_prediction's keep_first rule
// (inference.py:138-185): each chunk owns the chunk-local frames [write_lo, write_hi).
// One warp per token.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
head_kernel(const float* __restrict__ x, int D, const float* __restrict__ w, const float* __restrict__ bias,
            const ChunkSrc* __restrict__ chunks, int nchunks, int L, float* __restrict__ beat,
            float* __restrict__ down, int sum_head) {
  const int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= static_cast<int64_t>(nchunks) * L) return;
  const int b = static_cast<int>(row / L), t = static_cast<int>(row % L);
  const ChunkSrc cs = chunks[b];
  if (t < cs.write_lo || t >= cs.write_hi) return;  // warp-uniform
  const float* xr = x + row * D;
  float ss = 0.f, a0 = 0.f, a1 = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float v = xr[i];
    ss = fmaf(v, v, ss);
    a0 = fmaf(v, __ldg(w + i), a0);
    a1 = fmaf(v, __ldg(w + D + i), a1);
  }
  ss = warp_sum(ss); a0 = warp_sum(a0); a1 = warp_sum(a1);
  if (lane == 0) {
    const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
    const float o0 = a0 * inv + bias[0], o1 = a1 * inv + bias[1];
    const int64_t fr = cs.out_base + cs.start + t;
    beat[fr] = sum_head ? o0 + o1 : o0;  // SumHead (beat_tracker.py:315-330) / Head (beat_tracker.py:333-346)
    down[fr] = o1;
  }
}

void launch_head(const float* x, int D, const float* w, const float* b, const ChunkSrc* chunks,
                 int nchunks, int L, float* beat, float* down, int sum_head, cudaStream_t st) {
  const int64_t rows = static_cast<int64_t>(nchunks) * L;
  head_kernel<<<static_cast<unsigned>(ceil_div64(rows, 8)), 256, 0, st>>>(x, D, w, b, chunks, nchunks, L,
                                                                           beat, down, sum_head);
}

// ------------------------------------------------------------------------------------------
// minimal postprocessor (reference model/postprocessor.py:85-136, deduplicate_peaks
// :176-197): peak <=> x[t] == max(x[t-3..t+3]) and x[t] > 0; runs of peaks at most one
// frame from the running mean are merged into the running mean (float64, like the Python
// loop); times = frame / fps, one correctly rounded float64 division as numpy's; every downbeat snaps to the
// nearest beat (first argmin); unique.
// One CTA per clip: ordered compaction by ballot/prefix, then the short sequential part.
// ------------------------------------------------------------------------------------------
__device__ int compact_peaks(const float* __restrict__ x, int T, double* __restrict__ frames, int cap,
                             int* s_warp, int* s_base) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) *s_base = 0;
  __syncthreads();
  for (int t0 = 0; t0 < T; t0 += 256) {
    const int t = t0 + tid;
    bool pk = false;
    if (t < T) {
      const float v = x[t];
      float mx = v;
#pragma unroll
      for (int d = -3; d <= 3; ++d) {
        const int u = t + d;
        if (u >= 0 && u < T) mx = fmaxf(mx, x[u]);
      }
      pk = (v == mx) && (v > 0.f);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, pk);
    if (lane == 0) s_warp[wid] = __popc(bal);
    __syncthreads();
    int off = *s_base;
    for (int w = 0; w < wid; ++w) off += s_warp[w];
    if (pk) {
      const int idx = off + __popc(bal & ((1u << lane) - 1));
      if (idx < cap) frames[idx] = static_cast<double>(t);
    }
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < 8; ++w) tot += s_warp[w];
      *s_base += tot;
    }
    __syncthreads();
  }
  return *s_base;
}

__device__ int dedup_to_times(double* p, int n, double fps) {
  // deduplicate_peaks(width=1) followed by / fps; in place (output index <= input index)
  if (n == 0) return 0;
  int out = 0;
  double cur = p[0];
  double c = 1.0;
  for (int i = 1; i < n; ++i) {
    const double p2 = p[i];
    if (p2 - cur <= 1.0) {
      c += 1.0;
      cur += (p2 - cur) / c;
    } else {
      p[out++] = cur / fps;
      cur = p2;
      c = 1.0;
    }
  }
  p[out++] = cur / fps;
  return out;
}

__global__ void __launch_bounds__(256)
peakpick_kernel(const float* __restrict__ beat, const float* __restrict__ down,
                const int64_t* __restrict__ frame_off, double* __restrict__ beat_t, int32_t* __restrict__ n_beat,
                double* __restrict__ down_t, int32_t* __restrict__ n_down, int max_peaks, double fps) {
  __shared__ int s_warp[8];
  __shared__ int s_base;
  const int clip = blockIdx.x;
  const int64_t f0 = frame_off[clip];
  const int T = static_cast<int>(frame_off[clip + 1] - f0);
  double* bt_ = beat_t + static_cast<int64_t>(clip) * max_peaks;
  double* dt_ = down_t + static_cast<int64_t>(clip) * max_peaks;
  const int nb_raw = compact_peaks(beat + f0, T, bt_, max_peaks, s_warp, &s_base);
  __syncthreads();
  const int nd_raw = compact_peaks(down + f0, T, dt_, max_peaks, s_warp, &s_base);
  __syncthreads();
  __shared__ int s_nb, s_nd;
  if (threadIdx.x == 0) {
    if (nb_raw > max_peaks || nd_raw > max_peaks) {  // overflow: report the true counts, keep the first max_peaks
      n_beat[clip] = nb_raw;
      n_down[clip] = nd_raw;
      s_nb = -1;
    } else {
      s_nb = dedup_to_times(bt_, nb_raw, fps);
      s_nd = dedup_to_times(dt_, nd_raw, fps);
    }
  }
  __syncthreads();
  const int nb = s_nb;
  if (nb < 0) return;
  int nd = s_nd;
  // every downbeat moves to the nearest beat time (first minimum, postprocessor.py:128-134): one downbeat per thread
  if (nb > 0) {
    for (int i = threadIdx.x; i < nd; i += blockDim.x) {
      const double d = dt_[i];
      int best = 0;
      double bd = fabs(bt_[0] - d);
      for (int j = 1; j < nb; ++j) {
        const double dd = fabs(bt_[j] - d);
        if (dd < bd) { bd = dd; best = j; }
      }
      dt_[i] = bt_[best];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // np.unique: sort + drop duplicates (snapped downbeats are non-decreasing; insertion sort is a no-op then)
    for (int i = 1; i < nd; ++i) {
      const double v = dt_[i];
      int j = i - 1;
      while (j >= 0 && dt_[j] > v) { dt_[j + 1] = dt_[j]; --j; }
      dt_[j + 1] = v;
    }
    int o = 0;
    for (int i = 0; i < nd; ++i)
      if (o == 0 || dt_[i] != dt_[o - 1]) dt_[o++] = dt_[i];
    nd = o;
    n_beat[clip] = nb;
    n_down[clip] = nd;
  }
}

void launch_peakpick(const float* beat, const float* down, const int64_t* frame_off_dev, int n_clips,
                     double* beat_t, int32_t* n_beat, double* down_t, int32_t* n_down, int max_peaks,
                     double fps, cudaStream_t st) {
  if (n_clips <= 0) return;
  peakpick_kernel<<<n_clips, 256, 0, st>>>(beat, down, frame_off_dev, beat_t, n_beat, down_t, n_down,
                                           max_peaks, fps);
}

// ------------------------------------------------------------------------------------------ utils
__global__ void f32_to_h16_kernel(const float* __restrict__ in, h16* __restrict__ out, int64_t n) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = to_out<h16>(in[i]);
}
__global__ void h16_to_f32_kernel(const h16* __restrict__ in, float* __restrict__ out, int64_t n) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = to_f32(in[i]);
}
void launch_f32_to_h16(const float* in, void* out, int64_t n, cudaStream_t st) {
  if (n <= 0) return;
  f32_to_h16_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(in, reinterpret_cast<h16*>(out), n);
}
void launch_h16_to_f32(const void* in, float* out, int64_t n, cudaStream_t st) {
  if (n <= 0) return;
  h16_to_f32_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(reinterpret_cast<const h16*>(in), out, n);
}

template <typename TAct>
__global__ void pack_qkv_test_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                     const float* __restrict__ v, TAct* __restrict__ qkv, int seqs, int L,
                                     int heads, float qscale) {
  const int C = heads * 32;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t n = static_cast<int64_t>(seqs) * L * C;
  if (i >= n) return;
  const int c = static_cast<int>(i % C);
  const int64_t m = i / C;
  qkv[m * 3 * C + c] = to_out<TAct>(q[i] * qscale);
  qkv[m * 3 * C + C + c] = to_out<TAct>(k[i]);
  qkv[m * 3 * C + 2 * C + c] = to_out<TAct>(v[i]);
}
void launch_pack_qkv_test(const float* q, const float* k, const float* v, void* qkv, int seqs, int L, int heads,
                          float qscale, int act_h16, cudaStream_t st) {
  const int64_t n = static_cast<int64_t>(seqs) * L * heads * 32;
  const unsigned grid = static_cast<unsigned>(ceil_div64(n, 256));
  if (act_h16)
    pack_qkv_test_kernel<h16><<<grid, 256, 0, st>>>(q, k, v, reinterpret_cast<h16*>(qkv), seqs, L, heads, qscale);
  else
    pack_qkv_test_kernel<float><<<grid, 256, 0, st>>>(q, k, v, reinterpret_cast<float*>(qkv), seqs, L, heads, qscale);
}

}  // namespace bt
