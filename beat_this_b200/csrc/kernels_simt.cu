// fp32 CUDA-core path (BT_DTYPE_F32): tiled GEMM with the shared epilogues and a
// flash-style time-direction attention.  This is the exact-numerics path (the reference's
// float16=False behaviour); the 16-bit tensor-core path lives in kernels_gemm.cu, kernels_attn.cu, kernels_fused.cu.
#include "epilogue.cuh"

namespace bt {

// ------------------------------------------------------------------------------------ GEMM
constexpr int SG_BM = 64, SG_BN = 64, SG_BK = 16;

__global__ void __launch_bounds__(256)
gemm_simt_kernel(const float* __restrict__ A, const float* __restrict__ W, GemmShape g, EpiParams e) {
  __shared__ float As[SG_BK][SG_BM + 4];
  __shared__ float Ws[SG_BK][SG_BN + 4];
  const int t_tiles = ceil_div(g.L, SG_BM);
  const int p_out = blockIdx.x / t_tiles;
  const int t0 = (blockIdx.x % t_tiles) * SG_BM;
  const int n0 = blockIdx.y * SG_BN;
  const int tid = threadIdx.x;
  const int ty = tid / 16, tx = tid % 16;
  const int lr = tid / 4, lk = (tid % 4) * 4;  // loader: row / k offset
  const int Ktot = g.Kslab * g.nslab;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int kb = 0; kb < Ktot; kb += SG_BK) {
    const int s = kb / g.Kslab;
    const int k0 = kb - s * g.Kslab;
    {
      const int t = t0 + lr + g.t_shift[s];
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t >= 0 && t < g.L && (t0 + lr) < g.L) {
        const int64_t plane = static_cast<int64_t>(p_out) * g.plane_mul + g.plane_add[s];
        a = *reinterpret_cast<const float4*>(A + (plane * g.L + t) * g.lda + k0 + lk);
      }
      As[lk + 0][lr] = a.x; As[lk + 1][lr] = a.y; As[lk + 2][lr] = a.z; As[lk + 3][lr] = a.w;
      float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n0 + lr < g.N)
        w = *reinterpret_cast<const float4*>(W + static_cast<int64_t>(n0 + lr) * Ktot + kb + lk);
      Ws[lk + 0][lr] = w.x; Ws[lk + 1][lr] = w.y; Ws[lk + 2][lr] = w.z; Ws[lk + 3][lr] = w.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SG_BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 w = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
  const int n = n0 + tx * 4;
  if (n < g.N) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int t = t0 + ty * 4 + i;
      if (t < g.L) {
        const int64_t m = static_cast<int64_t>(p_out) * g.L + t;
        epilogue_apply(e, g.L, m, n, acc[i]);
      }
    }
  }
}

void launch_gemm_simt(const float* A, const float* W, const GemmShape& g, const EpiParams& e,
                      cudaStream_t st) {
  dim3 grid(ceil_div(g.L, SG_BM) * g.planes_out, ceil_div(g.N, SG_BN));
  gemm_simt_kernel<<<grid, 256, 0, st>>>(A, W, g, e);
}

// ------------------------------------------------------------------- time-direction attention
// One thread per query row, K/V tiles staged in shared memory, online softmax over blocks
// of 8 keys.  qkv: [seqs*L, 3C] (q | k | v), head h uses columns h*32..h*32+31 of each part.
constexpr int SA_BQ = 128, SA_BK = 64;

__global__ void __launch_bounds__(SA_BQ)
attn_time_simt_kernel(const float* __restrict__ qkv, const float* __restrict__ gates,
                      float* __restrict__ out, int L, int heads, float scale, const ChunkSrc* __restrict__ chunks,
                      int seqs_per_chunk) {
  __shared__ __align__(16) float Ks[SA_BK][32];
  __shared__ __align__(16) float Vs[SA_BK][32];
  const int C = heads * 32;
  const int seq = blockIdx.z, h = blockIdx.y;
  const int q_idx = blockIdx.x * SA_BQ + threadIdx.x;
  const bool q_ok = q_idx < L;
  const float* base = qkv + static_cast<int64_t>(seq) * L * 3 * C;
  float q[32], o[32];
  {
    const float* qp = base + static_cast<int64_t>(q_ok ? q_idx : 0) * 3 * C + h * 32;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float4 v = reinterpret_cast<const float4*>(qp)[i];
      q[4 * i] = v.x * scale; q[4 * i + 1] = v.y * scale; q[4 * i + 2] = v.z * scale; q[4 * i + 3] = v.w * scale;
    }
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float mx = -INFINITY, l = 0.f;

  const int Lk = chunks ? chunks[seq / seqs_per_chunk].len : L;  // keys that exist (the rest of the plane is padding)
  for (int k0 = 0; k0 < Lk; k0 += SA_BK) {
    __syncthreads();
    for (int i = threadIdx.x; i < SA_BK * 8; i += SA_BQ) {
      const int r = i / 8, c4 = i % 8;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (k0 + r < Lk) {
        const float* rp = base + static_cast<int64_t>(k0 + r) * 3 * C + h * 32;
        kv = reinterpret_cast<const float4*>(rp + C)[c4];
        vv = reinterpret_cast<const float4*>(rp + 2 * C)[c4];
      }
      reinterpret_cast<float4*>(&Ks[r][0])[c4] = kv;
      reinterpret_cast<float4*>(&Vs[r][0])[c4] = vv;
    }
    __syncthreads();
    const int kn = min(SA_BK, Lk - k0);
    for (int j0 = 0; j0 < kn; j0 += 8) {
      float s[8];
      float bm = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float a = 0.f;
#pragma unroll
        for (int d = 0; d < 32; ++d) a = fmaf(q[d], Ks[j0 + j][d], a);
        s[j] = (j0 + j < kn) ? a : -INFINITY;
        bm = fmaxf(bm, s[j]);
      }
      const float mn = fmaxf(mx, bm);
      const float corr = expf(mx - mn);  // mx = -inf on the first block -> 0
      l *= corr;
#pragma unroll
      for (int d = 0; d < 32; ++d) o[d] *= corr;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float p = expf(s[j] - mn);
        l += p;
#pragma unroll
        for (int d = 0; d < 32; ++d) o[d] = fmaf(p, Vs[j0 + j][d], o[d]);
      }
      mx = mn;
    }
  }
  if (q_ok) {
    const int64_t m = static_cast<int64_t>(seq) * L + q_idx;
    const float g = gates[m * heads + h] / l;
    float* op = out + m * C + h * 32;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      reinterpret_cast<float4*>(op)[i] =
          make_float4(o[4 * i] * g, o[4 * i + 1] * g, o[4 * i + 2] * g, o[4 * i + 3] * g);
  }
}

void launch_attn_time_simt(const float* qkv, const float* gates, float* out, int seqs, int L,
                           int heads, cudaStream_t st, const ChunkSrc* chunks, int seqs_per_chunk) {
  dim3 grid(ceil_div(L, SA_BQ), heads, seqs);
  attn_time_simt_kernel<<<grid, SA_BQ, 0, st>>>(qkv, gates, out, L, heads, 0.17677669529663687f, chunks, seqs_per_chunk);
}

}  // namespace bt
