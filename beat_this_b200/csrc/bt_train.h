// Launchers of kernels_train.cu, the fp32 training forward and backward (api_train.cu drives them).
#pragma once
#include <algorithm>

#include "bt_kernels.h"

namespace bt {

// element (r, c) at p[r * rs + c * cs]
struct TrMat {
  const float* p;
  int64_t rs, cs;
};
// One dropout site (include/beatthis.h, "dropout masks"): element e (e0 + the site's own index) is kept iff word e % 4 of
// Philox4x32-10(counter (lo32(e / 4), hi32(e / 4), site, 0), key (lo32(seed), hi32(seed))) >= thresh, and kept values
// are multiplied by scale.  thresh 0 (a rate of 0, or a zero-initialised TrDrop) is no dropout: the kernels take their
// eval-mode path.
struct TrDrop {
  uint64_t seed;
  uint32_t site, thresh;
  float scale;
  int64_t e0;
};
// The site's mask for rate p in [0, 1) (thresh floor(p 2^32), scale 1 / (1 - p)).
TrDrop tr_drop(uint64_t seed, uint32_t site, double p, int64_t e0 = 0);

// C[z * zs + m * ldc + n] = A(m, :) . B(n, :) over split z of K, + bias[n] + resid[m * ldr + n] (null: none); gelu_out
// (null: none) gets GELU of the result at the same index.  drop (unsplit GEMMs only), element m N + n: with gelu_out the
// mask applies to gelu_out alone (C keeps the pre-GELU value); without, to the result before resid is added.
struct TrGemmOut {
  float* C;
  int64_t ldc, zs;
  const float* bias;
  const float* resid;
  int64_t ldr;
  float* gelu_out;
  TrDrop drop;
};
// eval-mode BatchNorm: scale = w / sqrt(rv + 1e-5), shift = b - rm scale
struct TrBn {
  const float *w, *b, *rm, *rv;
};
// the input of a (S, 3) convolution with stride (S, 1) and padding (0, 1): element (b, f, t, c) of B x (Fo S) x L x C
// at b sb + f sf + t st + c sc
struct TrImg {
  int B, Fo, S, L, C;
  int64_t sb, sf, st, sc;
};
// `seqs` attention sequences of n positions and `heads` heads of 32: position i of sequence s is token row
// (s / seq_in) s_out + (s % seq_in) s_in + i s_pos
struct TrSeqs {
  int seqs, n, heads, seq_in;
  int64_t s_out, s_in, s_pos;
};

// splits > 1: partial products of consecutive K ranges of tr_gemm_kc columns at C + z * zs, z < tr_gemm_parts, for
// launch_tr_reduce
inline int tr_gemm_kc(int K, int splits) { return ((K + splits - 1) / splits + 15) / 16 * 16; }
inline int tr_gemm_parts(int K, int splits) { return (K + tr_gemm_kc(K, splits) - 1) / tr_gemm_kc(K, splits); }

// Floats of the training pass's split-K / column-sum partials (its scratch holds one such block).
constexpr int64_t kTrPartFloats = int64_t{8} << 20;
// The split policy of a weight gradient dW[N, K] = dY[M, N]^T X[M, K] (a tr_gemm of N x K outputs over M): enough
// parts to give two CTAs per SM of 132, at least 256 rows each, and all parts inside kTrPartFloats.
inline int tr_dw_splits(int64_t M, int N, int K) {
  const int64_t tiles = int64_t{(N + 63) / 64} * ((K + 63) / 64);
  int64_t splits = std::min<int64_t>((2 * 132 + tiles - 1) / tiles, std::max<int64_t>(1, M / 256));
  return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(splits, kTrPartFloats / (int64_t{N} * K))));
}
// The split policy of a column sum over M rows of N columns: 512 rows per part, all parts inside kTrPartFloats.
inline int tr_colsum_splits(int64_t M, int N) {
  return static_cast<int>(std::min<int64_t>((M + 511) / 512, kTrPartFloats / N));
}
void launch_tr_gemm(const TrMat& A, const TrMat& B, const TrGemmOut& o, int M, int N, int K, int splits, cudaStream_t st);
// out[i] = scale sum_z part[z n + i] (+ beta out[i] when beta != 0: the running-statistics update); with drop, out[i] is
// the mask's drop.scale times that, or 0 where element i is dropped (one part: a masked copy of a [M, N] gradient)
void launch_tr_reduce(const float* part, int Z, int64_t n, float scale, float* out, cudaStream_t st, float beta = 0.f,
                      const TrDrop& drop = {});
// column sums of [M, N] A (times B, times rs[m], where given) over up to `splits` row ranges: returns the parts written.
// shift (null: none) centres column n of A by shift[n]; without B the centred value is squared (a centred variance).
int launch_tr_colsum(const float* A, const float* B, const float* rs, int64_t M, int N, int splits, float* part,
                     cudaStream_t st, const float* shift = nullptr);
void launch_tr_rms_fwd(const float* x, const float* gamma, int64_t M, int C, float* xn, float* inv, cudaStream_t st);
void launch_tr_rms_bwd(const float* dxn, const float* x, const float* inv, const float* gamma, int64_t M, int C, bool add,
                       float* dres, cudaStream_t st);
void launch_tr_bn_gelu_fwd(const float* z, const TrBn& b, int64_t n, int C, float* y, cudaStream_t st);
void launch_tr_bn_gelu_bwd(const float* dy, const float* z, const TrBn& b, int64_t n, int C, float* dbn, float* dz,
                           cudaStream_t st);
void launch_tr_bn_grads(const float* s_gz, const float* s_g, const TrBn& b, int C, float* dw, float* db, cudaStream_t st);
// The batch-statistics terms of a BatchNorm's input gradient: its input x, the column sums s_gz = sum g x and s_g = sum g
// of the gradient g at its output, and 1 / N (N positions per channel).  b's rm / rv are then the batch mean and biased
// variance.
struct TrBnBatch {
  const float *x, *s_gz, *s_g;
  float inv_n;
};
// dx = g scale (eval mode, batch null) or scale (g - s_g / N - xhat sum(g xhat) / N) (batch statistics)
void launch_tr_bn_scale(const float* g, const TrBn& b, int64_t n, int C, float* dx, cudaStream_t st,
                        const TrBnBatch* batch = nullptr);
// dh = GELU'(h) da, times drop's mask and scale at element i
void launch_tr_gelu_bwd(const float* da, const float* h, int64_t n, float* dh, cudaStream_t st, const TrDrop& drop = {});
// bn (null: none) is the 1-d BatchNorm over the input's frequencies (the stem)
void launch_tr_im2col(const float* in, const TrImg& g, const TrBn* bn, float* col, cudaStream_t st);
void launch_tr_col2im(const float* dcol, const TrImg& g, float* din, cudaStream_t st);
void launch_tr_concat(const float* src, int B, int F, int L, int C, bool backward, float* dst, cudaStream_t st);
void launch_tr_rope(float* qkv, const float* freqs, int64_t M, int C, int L, int F, int posmode, bool inverse,
                    cudaStream_t st);
void launch_tr_gate_fwd(const float* O, const float* g, int64_t M, int C, float* G, cudaStream_t st);
void launch_tr_gate_bwd(float* dG, const float* O, const float* g, int64_t M, int C, float* dg, float* delta,
                        cudaStream_t st);
// head: o [M, 2] -> beat, down [M]; backward: the logits' gradients -> dout [M, 2]
void launch_tr_head_fwd(const float* o, int64_t M, bool sum_head, float* beat, float* down, cudaStream_t st);
void launch_tr_head_bwd(const float* dbeat, const float* ddown, int64_t M, bool sum_head, float* dout, cudaStream_t st);
// drop: dropout on the probabilities P after the softmax, element ((s heads + h) n + i) n + j (lse stays that of the
// undropped scores; O is the dropped output, so delta = rowsum(dO O) stays the flash-backward row term)
void launch_tr_attn_fwd(const float* qkv, const TrSeqs& q, float* O, float* lse, cudaStream_t st,
                        const TrDrop& drop = {});
void launch_tr_attn_dq(const float* qkv, const float* dO, const float* lse, const float* delta, const TrSeqs& q,
                       float* dqkv, cudaStream_t st, const TrDrop& drop = {});
void launch_tr_attn_dkv(const float* qkv, const float* dO, const float* lse, const float* delta, const TrSeqs& q,
                        float* dqkv, cudaStream_t st, const TrDrop& drop = {});

}  // namespace bt
