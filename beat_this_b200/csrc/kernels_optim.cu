// The AdamW update of bt_adamw_step (include/beatthis.h): one launch over every entry of a parameter table.
//
// Memory-bound: each element reads param, grad, exp_avg and exp_avg_sq and writes three of them back, 28 bytes, with a
// few dozen flops.  The table's entries are cut into chunks of kChunk elements; block b takes chunk b of the whole table
// and finds its entry by a binary search of the per-entry first chunks (prefix sums of the chunk counts the host
// computed), so one grid covers entries of any sizes without a block per entry.  An entry whose four pointers are
// 16-byte aligned moves float4s, the elements past its last whole float4 and every element of a misaligned entry go
// one float at a time.  Each element is read and written by one thread, without atomics, so results repeat bitwise.
//
// The arithmetic is torch's foreach AdamW (torch/optim/adam.py, _multi_tensor_adam with decoupled weight decay), op by
// op in fp32 on scalars the host rounded to fp32: the decay multiply, lerp (torch's two-sided formula), the second
// moment's multiply and addcmul, sqrt, division by sqrt(1 - beta2^t), + eps, and addcdiv with -lr / (1 - beta1^t).
#include <cuda_runtime.h>

#include <cstdint>

#include "bt_kernels.h"
#include "chunk_table.cuh"

namespace bt {

namespace {

constexpr int kThreads = 256;
constexpr int kVecPerThread = 4;                           // float4s per thread and chunk
constexpr int64_t kChunk = kThreads * kVecPerThread * 4;  // elements per block

__device__ __forceinline__ void adamw_element(float& p, float g, float& m, float& v, const AdamwEntry& e) {
  if (e.decay_on) p = p * e.decay;
  const float d = g - m;
  m = fabsf(e.w1) < 0.5f ? m + e.w1 * d : g - d * (1.f - e.w1);  // at::lerp(m, g, 1 - beta1)
  v = v * e.beta2;
  v = v + e.w2 * (g * g);
  const float den = sqrtf(v) / e.bc2_sqrt + e.eps;
  p = p + e.step_size * (m / den);
}

__global__ void __launch_bounds__(kThreads) adamw_kernel(const AdamwEntry* __restrict__ entries, int n_entries) {
  const int64_t chunk = blockIdx.x;
  const AdamwEntry e = entries[entry_of_chunk(entries, n_entries, chunk)];
  const int64_t begin = (chunk - e.chunk0) * kChunk;
  const int64_t end = min(begin + kChunk, e.n);
  if (e.vec) {
    const int64_t end4 = begin + ((end - begin) & ~int64_t{3});
    float4* p4 = reinterpret_cast<float4*>(e.p);
    const float4* g4 = reinterpret_cast<const float4*>(e.g);
    float4* m4 = reinterpret_cast<float4*>(e.m);
    float4* v4 = reinterpret_cast<float4*>(e.v);
#pragma unroll
    for (int k = 0; k < kVecPerThread; ++k) {
      const int64_t i = begin / 4 + k * kThreads + threadIdx.x;
      if (4 * i >= end4) break;
      float4 p = p4[i], m = m4[i], v = v4[i];
      const float4 g = __ldg(g4 + i);
      adamw_element(p.x, g.x, m.x, v.x, e);
      adamw_element(p.y, g.y, m.y, v.y, e);
      adamw_element(p.z, g.z, m.z, v.z, e);
      adamw_element(p.w, g.w, m.w, v.w, e);
      p4[i] = p, m4[i] = m, v4[i] = v;
    }
    const int64_t i = end4 + threadIdx.x;  // at most 3 elements of the entry's last chunk
    if (i < end) adamw_element(e.p[i], __ldg(e.g + i), e.m[i], e.v[i], e);
    return;
  }
  for (int64_t i = begin + threadIdx.x; i < end; i += kThreads) adamw_element(e.p[i], __ldg(e.g + i), e.m[i], e.v[i], e);
}

}  // namespace

int64_t adamw_chunks(int64_t n) { return (n + kChunk - 1) / kChunk; }

void launch_adamw(const AdamwEntry* entries_dev, int n_entries, int64_t chunks, cudaStream_t st) {
  if (n_entries <= 0 || chunks <= 0) return;
  adamw_kernel<<<static_cast<unsigned>(chunks), kThreads, 0, st>>>(entries_dev, n_entries);
}

}  // namespace bt
