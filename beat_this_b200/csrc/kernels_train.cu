// fp32 CUDA-core kernels of the training forward and backward (bt_train_forward / bt_train_backward): a strided GEMM
// with split-K partials, fixed-order reductions, RMSNorm, BatchNorm + GELU, the convolutions' im2col and col2im, RoPE,
// and flash-style attention forward and backward over strided sequences (head_dim 32).  No kernel uses atomics, so
// every result is bitwise repeatable.  Dropout masks (training mode) are regenerated from Philox4x32-10 wherever they
// are needed and never stored.
#include <cmath>

#include "bt_train.h"
#include "common.cuh"

namespace bt {

TrDrop tr_drop(uint64_t seed, uint32_t site, double p, int64_t e0) {
  const uint32_t thresh = p > 0.0 ? static_cast<uint32_t>(std::floor(p * 4294967296.0)) : 0u;
  return TrDrop{seed, site, thresh, thresh ? static_cast<float>(1.0 / (1.0 - p)) : 1.f, e0};
}

// ------------------------------------------------------------------------------------ dropout masks
// the four Philox words of elements 4 g .. 4 g + 3 of a site
__device__ __forceinline__ uint4 tr_drop_words(const TrDrop& d, int64_t g) {
  const uint64_t u = static_cast<uint64_t>(g);
  return philox4x32_10(make_uint4(static_cast<uint32_t>(u), static_cast<uint32_t>(u >> 32), d.site, 0u),
                       make_uint2(static_cast<uint32_t>(d.seed), static_cast<uint32_t>(d.seed >> 32)));
}
// element e of the site kept
__device__ __forceinline__ bool tr_keep(const TrDrop& d, int64_t e) {
  const uint4 w = tr_drop_words(d, e >> 2);
  const int k = static_cast<int>(e & 3);
  return (k == 0 ? w.x : k == 1 ? w.y : k == 2 ? w.z : w.w) >= d.thresh;
}
// bit k (k < cnt <= 32): element e + k of the site kept; one Philox call per four elements
__device__ __forceinline__ uint32_t tr_keep32(const TrDrop& d, int64_t e, int cnt) {
  uint32_t bits = 0;
  for (int64_t g = e >> 2; g <= (e + cnt - 1) >> 2; ++g) {
    const uint4 w = tr_drop_words(d, g);
    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int64_t k = 4 * g + q - e;
      if (k >= 0 && k < cnt && ws[q] >= d.thresh) bits |= 1u << k;
    }
  }
  return bits;
}

// ------------------------------------------------------------------------------------ GEMM
// C[z][m, n] = sum_{k in split z} A(m, k) B(n, k) (+ bias[n]) (+ resid[m, n]); with gelu_out also gelu_out = GELU(C).
constexpr int TG_BM = 64, TG_BN = 64, TG_BK = 16;

__device__ __forceinline__ void tg_load(float (*S)[TG_BM + 4], const TrMat& X, int rows, int r0, int k0, int k1,
                                        int tid) {
  // consecutive threads walk the operand's unit-stride dimension
  const bool k_inner = X.cs == 1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = tid + 256 * i;
    const int r = k_inner ? e / TG_BK : e % TG_BM;
    const int k = k_inner ? e % TG_BK : e / TG_BM;
    float v = 0.f;
    if (r0 + r < rows && k0 + k < k1) v = X.p[static_cast<int64_t>(r0 + r) * X.rs + static_cast<int64_t>(k0 + k) * X.cs];
    S[k][r] = v;
  }
}

__global__ void __launch_bounds__(256)
tr_gemm_kernel(TrMat A, TrMat B, TrGemmOut o, int M, int N, int K, int kc) {
  __shared__ float As[TG_BK][TG_BM + 4];
  __shared__ float Bs[TG_BK][TG_BN + 4];
  const int m0 = blockIdx.x * TG_BM, n0 = blockIdx.y * TG_BN, z = blockIdx.z;
  const int kb = z * kc, ke = min(K, kb + kc);
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  float acc[4][4] = {};
  for (int k0 = kb; k0 < ke; k0 += TG_BK) {
    tg_load(As, A, M, m0, k0, ke, tid);
    tg_load(Bs, B, N, n0, k0, ke, tid);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TG_BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* C = o.C + static_cast<int64_t>(z) * o.zs;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const uint32_t keep =
        o.drop.thresh ? tr_keep32(o.drop, o.drop.e0 + static_cast<int64_t>(m) * N + n0 + tx * 4, 4) : 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (o.bias) v += o.bias[n];
      if (o.drop.thresh) {
        const bool kept = (keep >> j) & 1u;
        if (o.gelu_out) {  // the FFN hidden: C keeps the pre-GELU value, gelu_out the dropped GELU output
          C[static_cast<int64_t>(m) * o.ldc + n] = v;
          o.gelu_out[static_cast<int64_t>(m) * o.ldc + n] = kept ? gelu_erf(v) * o.drop.scale : 0.f;
          continue;
        }
        v = kept ? v * o.drop.scale : 0.f;
      }
      if (o.resid) v += o.resid[static_cast<int64_t>(m) * o.ldr + n];
      C[static_cast<int64_t>(m) * o.ldc + n] = v;
      if (o.gelu_out) o.gelu_out[static_cast<int64_t>(m) * o.ldc + n] = gelu_erf(v);
    }
  }
}

void launch_tr_gemm(const TrMat& A, const TrMat& B, const TrGemmOut& o, int M, int N, int K, int splits, cudaStream_t st) {
  const int kc = tr_gemm_kc(K, splits);
  dim3 grid(ceil_div(M, TG_BM), ceil_div(N, TG_BN), ceil_div(K, kc));
  tr_gemm_kernel<<<grid, 256, 0, st>>>(A, B, o, M, N, K, kc);
}

// out[i] = scale * sum_{z < Z} part[z * n + i], z ascending; then masked (drop) and added to beta out[i] (beta != 0)
__global__ void tr_reduce_kernel(const float* __restrict__ part, int Z, int64_t n, float scale, float* __restrict__ out,
                                 float beta, TrDrop drop) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int z = 0; z < Z; ++z) s += part[z * n + i];
  float v = s * scale;
  if (drop.thresh) v = tr_keep(drop, drop.e0 + i) ? v * drop.scale : 0.f;
  if (beta != 0.f) v = fmaf(beta, out[i], v);
  out[i] = v;
}

void launch_tr_reduce(const float* part, int Z, int64_t n, float scale, float* out, cudaStream_t st, float beta,
                      const TrDrop& drop) {
  tr_reduce_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(part, Z, n, scale, out, beta, drop);
}

// part[z][n] = sum over rows m of split z of a (* B[m, n]) (* rs[m]), a = A[m, n] - shift[n] (SHIFT) or A[m, n], a * a
// with SHIFT and no B: 32 columns x 8 row lanes per CTA, the lanes summed in a fixed order through shared memory.
template <bool SHIFT>
__global__ void __launch_bounds__(256)
tr_colsum_kernel(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ rs, int64_t M, int N,
                 int64_t rows_per_split, float* __restrict__ part, const float* __restrict__ shift) {
  __shared__ float red[8][33];
  const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;
  const int n = blockIdx.x * 32 + tx;
  const int64_t r0 = blockIdx.y * rows_per_split, r1 = min(M, r0 + rows_per_split);
  const float sh = SHIFT && n < N ? shift[n] : 0.f;
  float s = 0.f;
  if (n < N)
    for (int64_t m = r0 + ty; m < r1; m += 8) {
      float v = A[m * N + n];
      if (SHIFT) v -= sh;
      if (B) v *= B[m * N + n];
      else if (SHIFT) v *= v;
      if (rs) v *= rs[m];
      s += v;
    }
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][tx];
    part[static_cast<int64_t>(blockIdx.y) * N + n] = t;
  }
}

int launch_tr_colsum(const float* A, const float* B, const float* rs, int64_t M, int N, int splits, float* part,
                     cudaStream_t st, const float* shift) {
  const int64_t rps = ceil_div64(M, splits);
  const int parts = static_cast<int>(ceil_div64(M, rps));
  const dim3 grid(ceil_div(N, 32), parts);
  if (shift) tr_colsum_kernel<true><<<grid, 256, 0, st>>>(A, B, rs, M, N, rps, part, shift);
  else tr_colsum_kernel<false><<<grid, 256, 0, st>>>(A, B, rs, M, N, rps, part, shift);
  return parts;
}

// ------------------------------------------------------------------------------------ RMSNorm
// One warp per row: inv = 1 / max(||x||, 1e-12) (F.normalize), xn = x inv sqrt(C) gamma.
__global__ void tr_rms_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, int64_t M, int C,
                                  float* __restrict__ xn, float* __restrict__ inv) {
  const int64_t m = static_cast<int64_t>(blockIdx.x) * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (m >= M) return;
  const float* xr = x + m * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s = fmaf(xr[c], xr[c], s);
  s = warp_sum(s);
  const float iv = 1.f / fmaxf(sqrtf(s), 1e-12f);
  const float sc = sqrtf(static_cast<float>(C));
  for (int c = lane; c < C; c += 32) xn[m * C + c] = xr[c] * iv * sc * gamma[c];
  if (lane == 0) inv[m] = iv;
}

void launch_tr_rms_fwd(const float* x, const float* gamma, int64_t M, int C, float* xn, float* inv, cudaStream_t st) {
  tr_rms_fwd_kernel<<<static_cast<unsigned>(ceil_div64(M, 8)), 256, 0, st>>>(x, gamma, M, C, xn, inv);
}

// du = dxn sqrt(C) gamma, u = x inv; dx = inv (du - u (u . du)), or du inv where the norm was clamped to 1e-12.
// dres[m] = (add ? dres[m] : 0) + dx.
__global__ void tr_rms_bwd_kernel(const float* __restrict__ dxn, const float* __restrict__ x,
                                  const float* __restrict__ inv, const float* __restrict__ gamma, int64_t M, int C,
                                  int add, float* dres) {
  const int64_t m = static_cast<int64_t>(blockIdx.x) * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (m >= M) return;
  const float sc = sqrtf(static_cast<float>(C));
  const float iv = inv[m];
  float ss = 0.f, dot = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float xv = x[m * C + c];
    ss = fmaf(xv, xv, ss);
    dot = fmaf(xv * iv, dxn[m * C + c] * sc * gamma[c], dot);
  }
  ss = warp_sum(ss);
  dot = warp_sum(dot);
  const bool clamped = sqrtf(ss) < 1e-12f;
  for (int c = lane; c < C; c += 32) {
    const float du = dxn[m * C + c] * sc * gamma[c];
    const float dx = clamped ? du * iv : iv * (du - x[m * C + c] * iv * dot);
    dres[m * C + c] = add ? dres[m * C + c] + dx : dx;
  }
}

void launch_tr_rms_bwd(const float* dxn, const float* x, const float* inv, const float* gamma, int64_t M, int C, bool add,
                       float* dres, cudaStream_t st) {
  tr_rms_bwd_kernel<<<static_cast<unsigned>(ceil_div64(M, 8)), 256, 0, st>>>(dxn, x, inv, gamma, M, C, add, dres);
}

// ------------------------------------------------------------------------------------ BatchNorm + GELU
// rm / rv: the running statistics (eval mode) or the batch mean and biased variance (training mode)
__device__ __forceinline__ float bn_scale(const TrBn& b, int c) { return b.w[c] / sqrtf(b.rv[c] + 1e-5f); }

// y = GELU(z scale + shift), channel = index % C
__global__ void tr_bn_gelu_fwd_kernel(const float* __restrict__ z, TrBn b, int64_t n, int C, float* __restrict__ y) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = static_cast<int>(i % C);
  const float s = bn_scale(b, c);
  y[i] = gelu_erf(z[i] * s + (b.b[c] - b.rm[c] * s));
}

__device__ __forceinline__ float gelu_grad(float x) {
  const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752440f));
  const float pdf = 0.3989422804014327f * expf(-0.5f * x * x);
  return cdf + x * pdf;
}

// dbn = dy GELU'(z scale + shift) (the gradient at the BatchNorm's output), dz = dbn scale
__global__ void tr_bn_gelu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ z, TrBn b, int64_t n, int C,
                                      float* __restrict__ dbn, float* __restrict__ dz) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = static_cast<int>(i % C);
  const float s = bn_scale(b, c);
  const float g = dy[i] * gelu_grad(z[i] * s + (b.b[c] - b.rm[c] * s));
  dbn[i] = g;
  dz[i] = g * s;
}

// From the column sums S_gz = sum dbn z and S_g = sum dbn: dweight = (S_gz - rm S_g) / sqrt(rv + eps), dbias = S_g.
__global__ void tr_bn_grads_kernel(const float* __restrict__ s_gz, const float* __restrict__ s_g, TrBn b, int C,
                                   float* dw, float* db) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (dw) dw[c] = (s_gz[c] - b.rm[c] * s_g[c]) / sqrtf(b.rv[c] + 1e-5f);
  if (db) db[c] = s_g[c];
}

// dx = g scale: the gradient at a BatchNorm's input in eval mode.  With batch statistics (bb.x set), xhat = (x - mean)
// rstd: dx = scale (g - S_g / N - xhat sum(g xhat) / N), sum(g xhat) = rstd (S_gz - mean S_g).
__global__ void tr_bn_scale_kernel(const float* __restrict__ g, TrBn b, int64_t n, int C, float* __restrict__ dx,
                                   TrBnBatch bb) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = static_cast<int>(i % C);
  if (!bb.x) {
    dx[i] = g[i] * bn_scale(b, c);
    return;
  }
  const float mean = b.rm[c], ivar = 1.f / (b.rv[c] + 1e-5f);
  const float t = (bb.s_gz[c] - mean * bb.s_g[c]) * ivar;
  dx[i] = bn_scale(b, c) * (g[i] - bb.s_g[c] * bb.inv_n - (bb.x[i] - mean) * t * bb.inv_n);
}

void launch_tr_bn_gelu_fwd(const float* z, const TrBn& b, int64_t n, int C, float* y, cudaStream_t st) {
  tr_bn_gelu_fwd_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(z, b, n, C, y);
}
void launch_tr_bn_gelu_bwd(const float* dy, const float* z, const TrBn& b, int64_t n, int C, float* dbn, float* dz,
                           cudaStream_t st) {
  tr_bn_gelu_bwd_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(dy, z, b, n, C, dbn, dz);
}
void launch_tr_bn_grads(const float* s_gz, const float* s_g, const TrBn& b, int C, float* dw, float* db, cudaStream_t st) {
  tr_bn_grads_kernel<<<ceil_div(C, 128), 128, 0, st>>>(s_gz, s_g, b, C, dw, db);
}
void launch_tr_bn_scale(const float* g, const TrBn& b, int64_t n, int C, float* dx, cudaStream_t st,
                        const TrBnBatch* batch) {
  tr_bn_scale_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(g, b, n, C, dx,
                                                                                batch ? *batch : TrBnBatch{});
}

// dh = da GELU'(h), da masked and scaled first under drop (element i); in place when dh == da
__global__ void tr_gelu_bwd_kernel(const float* da, const float* __restrict__ h, int64_t n, float* dh, TrDrop drop) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float d = da[i];
  if (drop.thresh) d = tr_keep(drop, drop.e0 + i) ? d * drop.scale : 0.f;
  dh[i] = d * gelu_grad(h[i]);
}
void launch_tr_gelu_bwd(const float* da, const float* h, int64_t n, float* dh, cudaStream_t st, const TrDrop& drop) {
  tr_gelu_bwd_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(da, h, n, dh, drop);
}

// ------------------------------------------------------------------------------------ convolution slabs
// Kernel (S, 3), stride (S, 1), padding (0, 1) over an input of Fo * S frequencies: col row (b * Fo + fo) * L + t,
// column (c * S + df) * 3 + dt (the order of a [Cout, Cin, S, 3] weight) = in(b, fo S + df, t + dt - 1, c), 0 outside
// [0, L).  With bn, in-range values pass through the 1-d BatchNorm of frequency fo S + df first (the stem).
__global__ void tr_im2col_kernel(const float* __restrict__ in, TrImg g, TrBn bn, int use_bn, float* __restrict__ col) {
  const int K = g.C * g.S * 3;
  const int64_t n = static_cast<int64_t>(g.B) * g.Fo * g.L * K;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = static_cast<int>(i % K);
  const int64_t r = i / K;
  const int t = static_cast<int>(r % g.L);
  const int64_t bf = r / g.L;
  const int fo = static_cast<int>(bf % g.Fo), b = static_cast<int>(bf / g.Fo);
  const int dt = k % 3, df = (k / 3) % g.S, c = k / (3 * g.S);
  const int f = fo * g.S + df, ti = t + dt - 1;
  float v = 0.f;
  if (ti >= 0 && ti < g.L) {
    v = in[b * g.sb + f * g.sf + static_cast<int64_t>(ti) * g.st + c * g.sc];
    if (use_bn) {
      const float s = bn_scale(bn, f);
      v = v * s + (bn.b[f] - bn.rm[f] * s);
    }
  }
  col[i] = v;
}

// The adjoint of im2col (without the BatchNorm): din(b, f, t, c) = sum_dt dcol[row (b, f / S, t - dt + 1), column
// (c, f % S, dt)], dt ascending.  One thread per input element; nothing is accumulated across threads.
__global__ void tr_col2im_kernel(const float* __restrict__ dcol, TrImg g, float* __restrict__ din) {
  const int64_t n = static_cast<int64_t>(g.B) * g.Fo * g.S * g.L * g.C;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int K = g.C * g.S * 3;
  const int c = static_cast<int>(i % g.C);
  int64_t r = i / g.C;
  const int t = static_cast<int>(r % g.L);
  r /= g.L;
  const int F = g.Fo * g.S;
  const int f = static_cast<int>(r % F), b = static_cast<int>(r / F);
  const int fo = f / g.S, df = f % g.S;
  float s = 0.f;
#pragma unroll
  for (int dt = 0; dt < 3; ++dt) {
    const int to = t - dt + 1;
    if (to >= 0 && to < g.L)
      s += dcol[((static_cast<int64_t>(b) * g.Fo + fo) * g.L + to) * K + (c * g.S + df) * 3 + dt];
  }
  din[b * g.sb + f * g.sf + static_cast<int64_t>(t) * g.st + c * g.sc] = s;
}

void launch_tr_im2col(const float* in, const TrImg& g, const TrBn* bn, float* col, cudaStream_t st) {
  const int64_t n = static_cast<int64_t>(g.B) * g.Fo * g.L * g.C * g.S * 3;
  tr_im2col_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(in, g, bn ? *bn : TrBn{}, bn != nullptr,
                                                                               col);
}
void launch_tr_col2im(const float* dcol, const TrImg& g, float* din, cudaStream_t st) {
  const int64_t n = static_cast<int64_t>(g.B) * g.Fo * g.S * g.L * g.C;
  tr_col2im_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(dcol, g, din);
}

// "b c f t -> b t (c f)" between tokens [B, F, L, C] and rows [B * L, C * F]: forward gathers the rows, backward
// scatters their gradient back (a permutation both ways).
__global__ void tr_concat_kernel(const float* __restrict__ src, int B, int F, int L, int C, int backward,
                                 float* __restrict__ dst) {
  const int64_t n = static_cast<int64_t>(B) * F * L * C;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = static_cast<int>(i % (C * F));  // row layout index
  const int64_t bt = i / (C * F);
  const int t = static_cast<int>(bt % L), b = static_cast<int>(bt / L);
  const int c = k / F, f = k % F;
  const int64_t tok = ((static_cast<int64_t>(b) * F + f) * L + t) * C + c;
  if (backward) dst[tok] = src[i];
  else dst[i] = src[tok];
}
void launch_tr_concat(const float* src, int B, int F, int L, int C, bool backward, float* dst, cudaStream_t st) {
  const int64_t n = static_cast<int64_t>(B) * F * L * C;
  tr_concat_kernel<<<static_cast<unsigned>(ceil_div64(n, 256)), 256, 0, st>>>(src, B, F, L, C, backward, dst);
}

// ------------------------------------------------------------------------------------ RoPE, gates, head
// Rotates the q and k columns of qkv [M, 3C] in place by pos * freqs[i] for the interleaved pair i of each head
// (rotary_embedding_torch); inverse: by -pos * freqs[i] (the gradient of the rotation).  pos = m % L (posmode 0) or
// (m / L) % F (posmode 1).
__global__ void tr_rope_kernel(float* qkv, const float* __restrict__ freqs, int64_t M, int C, int L, int F, int posmode,
                               int inverse) {
  const int pairs = C;  // C / 2 pairs in each of q and k
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= M * pairs) return;
  const int64_t m = i / pairs;
  const int p = static_cast<int>(i % pairs);
  const int col = (p < C / 2) ? 2 * p : C + 2 * (p - C / 2);
  const int pos = posmode == 0 ? static_cast<int>(m % L) : static_cast<int>((m / L) % F);
  const float ang = static_cast<float>(pos) * freqs[(col % 32) / 2];
  const float co = cosf(ang), si = inverse ? -sinf(ang) : sinf(ang);
  float* v = qkv + m * 3 * C + col;
  const float x0 = v[0], x1 = v[1];
  v[0] = x0 * co - x1 * si;
  v[1] = x1 * co + x0 * si;
}
void launch_tr_rope(float* qkv, const float* freqs, int64_t M, int C, int L, int F, int posmode, bool inverse,
                    cudaStream_t st) {
  tr_rope_kernel<<<static_cast<unsigned>(ceil_div64(M * C, 256)), 256, 0, st>>>(qkv, freqs, M, C, L, F, posmode, inverse);
}

// G = O sigmoid(g) per head: O [M, C], g [M, heads]
__global__ void tr_gate_fwd_kernel(const float* __restrict__ O, const float* __restrict__ g, int64_t M, int C,
                                   float* __restrict__ G) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const int64_t m = i / C;
  const int h = static_cast<int>(i % C) / 32;
  G[i] = O[i] * sigmoidf_(g[m * (C / 32) + h]);
}
void launch_tr_gate_fwd(const float* O, const float* g, int64_t M, int C, float* G, cudaStream_t st) {
  tr_gate_fwd_kernel<<<static_cast<unsigned>(ceil_div64(M * C, 256)), 256, 0, st>>>(O, g, M, C, G);
}

// From dG (the gradient at the gated output, overwritten by dO = dG sigmoid(g)): dg = sigmoid'(g) sum_d dG O and the
// flash-backward row term delta = sum_d dO O, per (row, head).
__global__ void tr_gate_bwd_kernel(float* dG, const float* __restrict__ O, const float* __restrict__ g, int64_t M, int C,
                                   float* __restrict__ dg, float* __restrict__ delta) {
  const int heads = C / 32;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= M * heads) return;
  const float sg = sigmoidf_(g[i]);
  float* d = dG + i * 32;  // row m = i / heads, head h = i % heads: columns (m * C + h * 32)
  const float* o = O + i * 32;
  float s = 0.f, t = 0.f;
#pragma unroll 8
  for (int j = 0; j < 32; ++j) {
    const float dv = d[j], ov = o[j];
    s = fmaf(dv, ov, s);
    const float dov = dv * sg;
    t = fmaf(dov, ov, t);
    d[j] = dov;
  }
  dg[i] = s * sg * (1.f - sg);
  delta[i] = t;
}
void launch_tr_gate_bwd(float* dG, const float* O, const float* g, int64_t M, int C, float* dg, float* delta,
                        cudaStream_t st) {
  tr_gate_bwd_kernel<<<static_cast<unsigned>(ceil_div64(M * (C / 32), 128)), 128, 0, st>>>(dG, O, g, M, C, dg, delta);
}

// beat = o0 + o1 (sum head) or o0, down = o1
__global__ void tr_head_fwd_kernel(const float* __restrict__ o, int64_t M, int sum_head, float* __restrict__ beat,
                                   float* __restrict__ down) {
  const int64_t m = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float o0 = o[2 * m], o1 = o[2 * m + 1];
  beat[m] = sum_head ? o0 + o1 : o0;
  down[m] = o1;
}
// do0 = dbeat, do1 = ddown (+ dbeat for the sum head)
__global__ void tr_head_bwd_kernel(const float* __restrict__ dbeat, const float* __restrict__ ddown, int64_t M,
                                   int sum_head, float* __restrict__ dout) {
  const int64_t m = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float db = dbeat[m], dd = ddown[m];
  dout[2 * m] = db;
  dout[2 * m + 1] = sum_head ? dd + db : dd;
}
void launch_tr_head_fwd(const float* o, int64_t M, bool sum_head, float* beat, float* down, cudaStream_t st) {
  tr_head_fwd_kernel<<<static_cast<unsigned>(ceil_div64(M, 256)), 256, 0, st>>>(o, M, sum_head, beat, down);
}
void launch_tr_head_bwd(const float* dbeat, const float* ddown, int64_t M, bool sum_head, float* dout, cudaStream_t st) {
  tr_head_bwd_kernel<<<static_cast<unsigned>(ceil_div64(M, 256)), 256, 0, st>>>(dbeat, ddown, M, sum_head, dout);
}

// ------------------------------------------------------------------------------------ attention
// Sequence s, position i: token row = (s / seq_in) * s_out + (s % seq_in) * s_in + i * s_pos.  q, k, v of head h at
// qkv[row * 3C + {0, C, 2C} + 32 h] (q, k roped, q not scaled).  One thread per query (or key) row; the other side in
// shared-memory tiles of TA_T rows.
constexpr int TA_Q = 64, TA_T = 32;

__device__ __forceinline__ int64_t ta_row(const TrSeqs& q, int s, int i) {
  return static_cast<int64_t>(s / q.seq_in) * q.s_out + static_cast<int64_t>(s % q.seq_in) * q.s_in +
         static_cast<int64_t>(i) * q.s_pos;
}
__device__ __forceinline__ void ta_load32(float (&r)[32], const float* p, float sc = 1.f) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = reinterpret_cast<const float4*>(p)[i];
    r[4 * i] = v.x * sc; r[4 * i + 1] = v.y * sc; r[4 * i + 2] = v.z * sc; r[4 * i + 3] = v.w * sc;
  }
}
__device__ __forceinline__ void ta_store32(float* p, const float (&r)[32], float sc = 1.f) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
    reinterpret_cast<float4*>(p)[i] = make_float4(r[4 * i] * sc, r[4 * i + 1] * sc, r[4 * i + 2] * sc, r[4 * i + 3] * sc);
}
// rows [j0, j0 + TA_T) of sequence s, columns `off` + 32 h of a [*, ld] array, into T (zeros past n)
__device__ __forceinline__ void ta_tile(float (*T)[32], const float* base, int64_t ld, int off, const TrSeqs& q, int s,
                                        int j0) {
  for (int e = threadIdx.x; e < TA_T * 8; e += TA_Q) {
    const int r = e / 8, c4 = e % 8;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (j0 + r < q.n) v = reinterpret_cast<const float4*>(base + ta_row(q, s, j0 + r) * ld + off)[c4];
    reinterpret_cast<float4*>(&T[r][0])[c4] = v;
  }
}

// element ((s heads + h) n + i) n of the probability dropout site: the first of query row i
__device__ __forceinline__ int64_t ta_drop_row(const TrSeqs& q, int s, int h, int i) {
  return ((static_cast<int64_t>(s) * q.heads + h) * q.n + i) * q.n;
}

// O = softmax(q k^T / sqrt 32) v, lse = log-sum-exp of the scaled scores (natural log).  DROP: O = (mask P / (1 - p)) v
// with the mask of drop (lse unchanged).
template <bool DROP>
__global__ void __launch_bounds__(TA_Q)
tr_attn_fwd_kernel(const float* __restrict__ qkv, TrSeqs q, float* __restrict__ O, float* __restrict__ lse,
                   TrDrop drop) {
  __shared__ __align__(16) float Ks[TA_T][32];
  __shared__ __align__(16) float Vs[TA_T][32];
  const int C = q.heads * 32, h = blockIdx.y;
  const int qt = ceil_div(q.n, TA_Q);
  const int s = blockIdx.x / qt, i = (blockIdx.x % qt) * TA_Q + threadIdx.x;
  const bool ok = i < q.n;
  const int64_t row = ta_row(q, s, ok ? i : 0);
  float qv[32], o[32];
  ta_load32(qv, qkv + row * 3 * C + h * 32, 0.17677669529663687f);
#pragma unroll
  for (int d = 0; d < 32; ++d) o[d] = 0.f;
  float mx = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < q.n; j0 += TA_T) {
    __syncthreads();
    ta_tile(Ks, qkv, 3 * C, C + h * 32, q, s, j0);
    ta_tile(Vs, qkv, 3 * C, 2 * C + h * 32, q, s, j0);
    __syncthreads();
    const int kn = min(TA_T, q.n - j0);
    const uint32_t keep = DROP ? tr_keep32(drop, drop.e0 + ta_drop_row(q, s, h, ok ? i : 0) + j0, kn) : 0u;
    for (int j = 0; j < kn; ++j) {
      float a = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) a = fmaf(qv[d], Ks[j][d], a);
      const float mn = fmaxf(mx, a);
      const float corr = expf(mx - mn), p = expf(a - mn);
      l = l * corr + p;
      const float pv = DROP && !((keep >> j) & 1u) ? 0.f : p;
#pragma unroll
      for (int d = 0; d < 32; ++d) o[d] = fmaf(pv, Vs[j][d], o[d] * corr);
      mx = mn;
    }
  }
  if (ok) {
    ta_store32(O + row * C + h * 32, o, DROP ? drop.scale / l : 1.f / l);
    lse[row * q.heads + h] = mx + logf(l);
  }
}

// dq = sum_j p_ij (dO_i . v_j - delta_i) k_j / sqrt 32, with p_ij = exp(q_i . k_j / sqrt 32 - lse_i); into the q columns
// of dqkv.  DROP: dO_i . v_j is masked and scaled as the forward's P was.
template <bool DROP>
__global__ void __launch_bounds__(TA_Q)
tr_attn_dq_kernel(const float* __restrict__ qkv, const float* __restrict__ dO, const float* __restrict__ lse,
                  const float* __restrict__ delta, TrSeqs q, float* __restrict__ dqkv, TrDrop drop) {
  __shared__ __align__(16) float Ks[TA_T][32];
  __shared__ __align__(16) float Vs[TA_T][32];
  const int C = q.heads * 32, h = blockIdx.y;
  const int qt = ceil_div(q.n, TA_Q);
  const int s = blockIdx.x / qt, i = (blockIdx.x % qt) * TA_Q + threadIdx.x;
  const bool ok = i < q.n;
  const int64_t row = ta_row(q, s, ok ? i : 0);
  const float sc = 0.17677669529663687f;
  float qv[32], dov[32], dq[32];
  ta_load32(qv, qkv + row * 3 * C + h * 32, sc);
  ta_load32(dov, dO + row * C + h * 32);
  const float L_i = lse[row * q.heads + h], D_i = delta[row * q.heads + h];
#pragma unroll
  for (int d = 0; d < 32; ++d) dq[d] = 0.f;
  for (int j0 = 0; j0 < q.n; j0 += TA_T) {
    __syncthreads();
    ta_tile(Ks, qkv, 3 * C, C + h * 32, q, s, j0);
    ta_tile(Vs, qkv, 3 * C, 2 * C + h * 32, q, s, j0);
    __syncthreads();
    const int kn = min(TA_T, q.n - j0);
    const uint32_t keep = DROP ? tr_keep32(drop, drop.e0 + ta_drop_row(q, s, h, ok ? i : 0) + j0, kn) : 0u;
    for (int j = 0; j < kn; ++j) {
      float a = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        a = fmaf(qv[d], Ks[j][d], a);
        dp = fmaf(dov[d], Vs[j][d], dp);
      }
      if (DROP) dp = (keep >> j) & 1u ? dp * drop.scale : 0.f;
      const float ds = expf(a - L_i) * (dp - D_i);
#pragma unroll
      for (int d = 0; d < 32; ++d) dq[d] = fmaf(ds, Ks[j][d], dq[d]);
    }
  }
  if (ok) ta_store32(dqkv + row * 3 * C + h * 32, dq, sc);
}

// dk_j = sum_i ds_ij q_i / sqrt 32, dv_j = sum_i p_ij dO_i; into the k and v columns of dqkv.  DROP: dv takes the
// masked, scaled p_ij and ds_ij the masked, scaled dO_i . v_j; each query tile's mask bits for the CTA's 64 keys are
// expanded once into shared memory (two words per query row, one word per thread).
template <bool DROP>
__global__ void __launch_bounds__(TA_Q)
tr_attn_dkv_kernel(const float* __restrict__ qkv, const float* __restrict__ dO, const float* __restrict__ lse,
                   const float* __restrict__ delta, TrSeqs q, float* __restrict__ dqkv, TrDrop drop) {
  static_assert(TA_Q == 2 * TA_T, "one mask word of 32 keys per thread and query row");
  __shared__ __align__(16) float Qs[TA_T][32];
  __shared__ __align__(16) float Ds[TA_T][32];
  __shared__ float Ls[TA_T], Dl[TA_T];
  __shared__ uint32_t Ms[DROP ? TA_T : 1][2];
  const int C = q.heads * 32, h = blockIdx.y;
  const int kt = ceil_div(q.n, TA_Q);
  const int s = blockIdx.x / kt, j = (blockIdx.x % kt) * TA_Q + threadIdx.x;
  const bool ok = j < q.n;
  const int64_t row = ta_row(q, s, ok ? j : 0);
  const float sc = 0.17677669529663687f;
  float kv[32], vv[32], dk[32], dv[32];
  ta_load32(kv, qkv + row * 3 * C + C + h * 32);
  ta_load32(vv, qkv + row * 3 * C + 2 * C + h * 32);
#pragma unroll
  for (int d = 0; d < 32; ++d) dk[d] = dv[d] = 0.f;
  for (int i0 = 0; i0 < q.n; i0 += TA_T) {
    __syncthreads();
    ta_tile(Qs, qkv, 3 * C, h * 32, q, s, i0);
    ta_tile(Ds, dO, C, h * 32, q, s, i0);
    if (threadIdx.x < TA_T) {
      const int i = i0 + threadIdx.x;
      const int64_t r = ta_row(q, s, i < q.n ? i : 0);
      Ls[threadIdx.x] = lse[r * q.heads + h];
      Dl[threadIdx.x] = delta[r * q.heads + h];
    }
    if (DROP) {
      const int i = i0 + threadIdx.x / 2, jb = (blockIdx.x % kt) * TA_Q + (threadIdx.x % 2) * 32;
      Ms[threadIdx.x / 2][threadIdx.x % 2] =
          i < q.n && jb < q.n ? tr_keep32(drop, drop.e0 + ta_drop_row(q, s, h, i) + jb, min(32, q.n - jb)) : 0u;
    }
    __syncthreads();
    const int qn = min(TA_T, q.n - i0);
    for (int i = 0; i < qn; ++i) {
      float a = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        a = fmaf(Qs[i][d], kv[d], a);
        dp = fmaf(Ds[i][d], vv[d], dp);
      }
      const float p = expf(a * sc - Ls[i]);
      float pv = p;
      if (DROP) {
        const bool kept = (Ms[i][threadIdx.x / 32] >> (threadIdx.x % 32)) & 1u;
        pv = kept ? p * drop.scale : 0.f;
        dp = kept ? dp * drop.scale : 0.f;
      }
      const float ds = p * (dp - Dl[i]);
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        dv[d] = fmaf(pv, Ds[i][d], dv[d]);
        dk[d] = fmaf(ds, Qs[i][d], dk[d]);
      }
    }
  }
  if (ok) {
    ta_store32(dqkv + row * 3 * C + C + h * 32, dk, sc);
    ta_store32(dqkv + row * 3 * C + 2 * C + h * 32, dv);
  }
}

// a rate of 0 runs the eval-mode instantiation
void launch_tr_attn_fwd(const float* qkv, const TrSeqs& q, float* O, float* lse, cudaStream_t st, const TrDrop& drop) {
  dim3 grid(q.seqs * ceil_div(q.n, TA_Q), q.heads);
  if (drop.thresh) tr_attn_fwd_kernel<true><<<grid, TA_Q, 0, st>>>(qkv, q, O, lse, drop);
  else tr_attn_fwd_kernel<false><<<grid, TA_Q, 0, st>>>(qkv, q, O, lse, drop);
}
void launch_tr_attn_dq(const float* qkv, const float* dO, const float* lse, const float* delta, const TrSeqs& q,
                       float* dqkv, cudaStream_t st, const TrDrop& drop) {
  dim3 grid(q.seqs * ceil_div(q.n, TA_Q), q.heads);
  if (drop.thresh) tr_attn_dq_kernel<true><<<grid, TA_Q, 0, st>>>(qkv, dO, lse, delta, q, dqkv, drop);
  else tr_attn_dq_kernel<false><<<grid, TA_Q, 0, st>>>(qkv, dO, lse, delta, q, dqkv, drop);
}
void launch_tr_attn_dkv(const float* qkv, const float* dO, const float* lse, const float* delta, const TrSeqs& q,
                        float* dqkv, cudaStream_t st, const TrDrop& drop) {
  dim3 grid(q.seqs * ceil_div(q.n, TA_Q), q.heads);
  if (drop.thresh) tr_attn_dkv_kernel<true><<<grid, TA_Q, 0, st>>>(qkv, dO, lse, delta, q, dqkv, drop);
  else tr_attn_dkv_kernel<false><<<grid, TA_Q, 0, st>>>(qkv, dO, lse, delta, q, dqkv, drop);
}

}  // namespace bt
