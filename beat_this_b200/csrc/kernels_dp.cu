// The gradient exchange of data-parallel training (bt_grad_pack, bt_grad_ordered_sum; include/beatthis.h): one launch
// each over every entry of a gradient table, found per block as adamw_kernel finds its entry (chunk_table.cuh).
//
// Memory-bound copies and sums.  Entry e's numel elements sit at e.off of a packed row, densely in table order, so an
// entry's elements are in general not 16-byte aligned there: every element moves as one float, kPer of them per thread
// in flight.  The ordered sum is ((g_0 + g_1) + g_2) + ... over the rows in the order given, one rounded fp32 add per
// step (__fadd_rn: never contracted or reassociated), the first row stored as it is: what autograd's AccumulateGrad
// builds from the same gradients, so results are bitwise those of one process summing them in place, signed zeros and
// NaNs included.  Each element is written by one thread, without atomics.
#include <cuda_runtime.h>

#include <cstdint>

#include "bt_kernels.h"
#include "chunk_table.cuh"

namespace bt {

namespace {

constexpr int kThreads = 256;
constexpr int kPer = 8;                             // elements per thread and chunk
constexpr int64_t kChunk = int64_t{kThreads} * kPer;  // elements per block

__global__ void __launch_bounds__(kThreads) grad_pack_kernel(const GradEntry* __restrict__ entries, int n_entries,
                                                             float* __restrict__ row) {
  const int64_t chunk = blockIdx.x;
  const GradEntry e = entries[entry_of_chunk(entries, n_entries, chunk)];
  const int64_t begin = (chunk - e.chunk0) * kChunk + threadIdx.x;
  float v[kPer];
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const int64_t i = begin + q * kThreads;
    v[q] = i < e.n ? __ldg(e.grad + i) : 0.f;
  }
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const int64_t i = begin + q * kThreads;
    if (i < e.n) row[e.off + i] = v[q];
  }
}

__global__ void __launch_bounds__(kThreads) grad_ordered_sum_kernel(const GradEntry* __restrict__ entries, int n_entries,
                                                                    const float* const* __restrict__ rows, int k) {
  const int64_t chunk = blockIdx.x;
  const GradEntry e = entries[entry_of_chunk(entries, n_entries, chunk)];
  const int64_t begin = (chunk - e.chunk0) * kChunk + threadIdx.x;
  float acc[kPer];
  const float* r0 = rows[0] + e.off;
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const int64_t i = begin + q * kThreads;
    acc[q] = i < e.n ? __ldg(r0 + i) : 0.f;
  }
  for (int j = 1; j < k; ++j) {
    const float* r = rows[j] + e.off;
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int64_t i = begin + q * kThreads;
      if (i < e.n) acc[q] = __fadd_rn(acc[q], __ldg(r + i));
    }
  }
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const int64_t i = begin + q * kThreads;
    if (i < e.n) e.grad[i] = acc[q];
  }
}

}  // namespace

int64_t grad_chunks(int64_t n) { return (n + kChunk - 1) / kChunk; }

void launch_grad_pack(const GradEntry* entries_dev, int n_entries, int64_t chunks, float* row, cudaStream_t st) {
  grad_pack_kernel<<<static_cast<unsigned>(chunks), kThreads, 0, st>>>(entries_dev, n_entries, row);
}

void launch_grad_ordered_sum(const GradEntry* entries_dev, int n_entries, int64_t chunks, const float* const* rows_dev,
                             int k, cudaStream_t st) {
  grad_ordered_sum_kernel<<<static_cast<unsigned>(chunks), kThreads, 0, st>>>(entries_dev, n_entries, rows_dev, k);
}

}  // namespace bt
