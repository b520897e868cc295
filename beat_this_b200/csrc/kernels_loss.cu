// Training losses of the reference (model/loss.py: MaskedBCELoss, ShiftTolerantBCELoss, SplittedShiftTolerantBCELoss)
// over ragged rows of frames, forward and backward.  The contract is written out in include/beatthis.h (bt_beat_loss)
// and DESIGN.md section 9; tests/loss_reference.py restates it in numpy.
//
// Every CTA owns kLossTile consecutive frames of one row, one per thread, and stages the row around them in shared
// memory with the halo the max-pools need.  Element arithmetic is fp32 (torch's); sums are float64.  The forward writes
// one partial per CTA and a one-CTA launch reduces the partials in a fixed order, so results are bitwise repeatable.
// The backward gathers: each frame visits the 2t + 1 windows that cover it and adds the gradient of those it wins.
#include <cuda_runtime.h>

#include <cstdint>

#include "bt_kernels.h"

namespace bt {

namespace {

constexpr int kMasked = 0, kShift = 1;  // BT_LOSS_* of include/beatthis.h; 2 is the split kind
constexpr int kReduceThreads = 512;

// first frame scored by the kind (the scored range is [lo, len - lo))
__host__ __device__ __forceinline__ int64_t scored_lo(const LossParams& p) {
  return p.kind == kMasked ? 0 : 2 * static_cast<int64_t>(p.tolerance);
}

// the row that CTA b belongs to: last i with tile_first[i] <= b
__device__ __forceinline__ int find_row(const int64_t* tile_first, int n_rows, int64_t b) {
  int lo = 0, hi = n_rows - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tile_first[mid] <= b) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ float softplus(float z) { return log1pf(expf(-fabsf(z))) + fmaxf(z, 0.f); }

// binary_cross_entropy_with_logits with pos_weight p, one element
__device__ __forceinline__ float bce(float x, float y, float p) {
  return (1.f - y) * x + (1.f + (p - 1.f) * y) * softplus(-x);
}

// its derivative in x (torch's form)
__device__ __forceinline__ float bce_grad(float x, float y, float p) {
  const float py = p * y;
  return (py + 1.f - y) * (1.f / (1.f + expf(-x))) - py;
}

__device__ __forceinline__ double block_sum(double v, double* s_warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < nwarps; ++w) s += s_warp[w];
  return s;  // valid in thread 0
}

// Forward: CTA b sums the terms of kLossTile scored frames c0 + tid of its row.  sx holds x[c0 - t, c0 + kLossTile + t),
// sy holds y[c0 - 2t, c0 + kLossTile + 2t) (clipped to the row; a scored frame never reads past it).
__global__ void __launch_bounds__(kLossTile)
beat_loss_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ m,
                 const int64_t* __restrict__ row_off, const int64_t* __restrict__ tile_first, int n_rows, LossParams p,
                 double* __restrict__ partials) {
  __shared__ float sx[kLossTile + 2 * kLossMaxTolerance];
  __shared__ float sy[kLossTile + 4 * kLossMaxTolerance];
  __shared__ double s_warp[kLossTile / 32];
  const int64_t b = blockIdx.x;
  const int row = find_row(tile_first, n_rows, b);
  const int64_t base = row_off[row], len = row_off[row + 1] - base;
  const int t = p.kind == kMasked ? 0 : p.tolerance;
  const int64_t lo = scored_lo(p), c0 = lo + (b - tile_first[row]) * kLossTile;
  for (int i = threadIdx.x; i < kLossTile + 2 * t; i += kLossTile) {
    const int64_t j = c0 - t + i;
    sx[i] = j < len ? x[base + j] : 0.f;
  }
  for (int i = threadIdx.x; i < kLossTile + 4 * t; i += kLossTile) {
    const int64_t j = c0 - 2 * t + i;
    sy[i] = j < len ? y[base + j] : 0.f;
  }
  __syncthreads();
  const int64_t c = c0 + threadIdx.x;
  double term = 0.0;
  if (c < len - lo) {
    const int k = threadIdx.x;
    const float yc = sy[k + 2 * t], mc = m ? m[base + c] : 1.f;
    if (p.kind == kMasked) {
      term = mc * bce(sx[k], yc, p.pos_weight);
    } else {
      float xs = sx[k], ys = sy[k];
      for (int d = 1; d <= 2 * t; ++d) xs = fmaxf(xs, sx[k + d]);
      for (int d = 1; d <= 4 * t; ++d) ys = fmaxf(ys, sy[k + d]);
      if (p.kind == kShift) {
        const float w = (yc + (1.f - ys)) * mc;
        term = w * bce(xs, yc, p.pos_weight);
      } else {
        term = static_cast<double>(yc * mc * bce(xs, yc, p.pos_weight)) +
               static_cast<double>((1.f - ys) * mc * bce(xs, ys, p.pos_weight));
      }
    }
  }
  const double s = block_sum(term, s_warp);
  if (threadIdx.x == 0) partials[b] = s;
}

// Second forward launch, one CTA: row i's loss is its partials summed in order over its scored frames; the mean is the
// partials summed per thread in a fixed stride, then over the threads in a fixed order, over all scored frames.
__global__ void __launch_bounds__(kReduceThreads)
beat_loss_reduce_kernel(const double* __restrict__ partials, const int64_t* __restrict__ row_off,
                        const int64_t* __restrict__ tile_first, int n_rows, int64_t n_tiles, double n_scored,
                        LossParams p, double* __restrict__ row_loss, float* __restrict__ mean) {
  __shared__ double s_warp[kReduceThreads / 32];
  const int64_t lo = scored_lo(p);
  for (int i = threadIdx.x; i < n_rows; i += kReduceThreads) {
    double s = 0.0;
    for (int64_t k = tile_first[i]; k < tile_first[i + 1]; ++k) s += partials[k];
    row_loss[i] = s / static_cast<double>(row_off[i + 1] - row_off[i] - 2 * lo);
  }
  double s = 0.0;
  for (int64_t k = threadIdx.x; k < n_tiles; k += kReduceThreads) s += partials[k];
  s = block_sum(s, s_warp);
  if (threadIdx.x == 0) *mean = static_cast<float>(s / n_scored);
}

// Backward: CTA b writes the gradient of frames j0 + tid of its row.  The windows covering them have centres
// c in [j0 - t, j0 + kLossTile + t); sx holds x[j0 - 2t, ..+ kLossTile + 4t), sy holds y[j0 - 3t, ..+ kLossTile + 6t).
// Per centre i = c - (j0 - t): gc[i] = its gradient, ga[i] = the row-local frame that wins its window (-1: not scored).
__global__ void __launch_bounds__(kLossTile)
beat_loss_backward_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ m,
                          const int64_t* __restrict__ row_off, const int64_t* __restrict__ tile_first, int n_rows,
                          double n_scored, LossParams p, const float* __restrict__ grad_mean, float* __restrict__ grad) {
  __shared__ float sx[kLossTile + 4 * kLossMaxTolerance];
  __shared__ float sy[kLossTile + 6 * kLossMaxTolerance];
  __shared__ float gc[kLossTile + 2 * kLossMaxTolerance];
  __shared__ int32_t ga[kLossTile + 2 * kLossMaxTolerance];
  const int64_t b = blockIdx.x;
  const int row = find_row(tile_first, n_rows, b);
  const int64_t base = row_off[row], len = row_off[row + 1] - base;
  const int t = p.kind == kMasked ? 0 : p.tolerance;
  const int64_t lo = scored_lo(p), j0 = (b - tile_first[row]) * kLossTile;
  for (int i = threadIdx.x; i < kLossTile + 4 * t; i += kLossTile) {
    const int64_t j = j0 - 2 * t + i;
    sx[i] = j >= 0 && j < len ? x[base + j] : 0.f;
  }
  for (int i = threadIdx.x; i < kLossTile + 6 * t; i += kLossTile) {
    const int64_t j = j0 - 3 * t + i;
    sy[i] = j >= 0 && j < len ? y[base + j] : 0.f;
  }
  __syncthreads();
  const float scale = static_cast<float>(static_cast<double>(*grad_mean) / n_scored);
  for (int i = threadIdx.x; i < kLossTile + 2 * t; i += kLossTile) {
    const int64_t c = j0 - t + i;
    int32_t win = -1;
    float g = 0.f;
    if (c >= lo && c < len - lo) {
      const float yc = sy[i + 2 * t], mc = m ? m[base + c] : 1.f;
      // sx[i .. i + 2t] is x[c - t .. c + t]: the first maximum wins, as max_pool1d_with_indices picks it
      float xs = sx[i];
      int arg = 0;
      for (int d = 1; d <= 2 * t; ++d)
        if (sx[i + d] > xs) xs = sx[i + d], arg = d;
      win = static_cast<int32_t>(c - t + arg);
      if (p.kind == kMasked) {
        g = bce_grad(xs, yc, p.pos_weight) * mc * scale;
      } else {
        float ys = sy[i];
        for (int d = 1; d <= 4 * t; ++d) ys = fmaxf(ys, sy[i + d]);
        if (p.kind == kShift) {
          g = bce_grad(xs, yc, p.pos_weight) * ((yc + (1.f - ys)) * mc) * scale;
        } else {
          g = bce_grad(xs, yc, p.pos_weight) * (yc * mc) * scale + bce_grad(xs, ys, p.pos_weight) * ((1.f - ys) * mc) * scale;
        }
      }
    }
    gc[i] = g;
    ga[i] = win;
  }
  __syncthreads();
  const int64_t j = j0 + threadIdx.x;
  if (j < len) {
    float acc = 0.f;
    for (int i = threadIdx.x; i <= threadIdx.x + 2 * t; ++i)  // centres j - t .. j + t, ascending
      if (ga[i] == j) acc += gc[i];
    grad[base + j] = acc;
  }
}

}  // namespace

int64_t loss_tiles(int64_t len, const LossParams& p, bool backward) {
  const int64_t n = backward ? len : len - 2 * scored_lo(p);
  return (n + kLossTile - 1) / kLossTile;
}

void launch_beat_loss(const float* x, const float* y, const float* m, const int64_t* row_off_dev,
                      const int64_t* tile_first_dev, int n_rows, int64_t n_tiles, const LossParams& p, double* partials,
                      cudaStream_t st) {
  beat_loss_kernel<<<static_cast<unsigned>(n_tiles), kLossTile, 0, st>>>(x, y, m, row_off_dev, tile_first_dev, n_rows, p,
                                                                         partials);
}

void launch_beat_loss_reduce(const double* partials, const int64_t* row_off_dev, const int64_t* tile_first_dev,
                             int n_rows, int64_t n_tiles, int64_t n_scored, const LossParams& p, double* row_loss,
                             float* mean, cudaStream_t st) {
  beat_loss_reduce_kernel<<<1, kReduceThreads, 0, st>>>(partials, row_off_dev, tile_first_dev, n_rows, n_tiles,
                                                        static_cast<double>(n_scored), p, row_loss, mean);
}

void launch_beat_loss_backward(const float* x, const float* y, const float* m, const int64_t* row_off_dev,
                               const int64_t* tile_first_dev, int n_rows, int64_t n_tiles, int64_t n_scored,
                               const LossParams& p, const float* grad_mean, float* grad, cudaStream_t st) {
  beat_loss_backward_kernel<<<static_cast<unsigned>(n_tiles), kLossTile, 0, st>>>(
      x, y, m, row_off_dev, tile_first_dev, n_rows, static_cast<double>(n_scored), p, grad_mean, grad);
}

}  // namespace bt
