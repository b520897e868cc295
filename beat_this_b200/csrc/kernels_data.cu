// Training batches: the gather, mask and target steps of the reference's BeatTrackingDataset.__getitem__ and
// default_collate (dataset.py:169-241, augment.py:129-201).  The contract is written out in include/beatthis.h
// (bt_train_batch) and DESIGN.md section 9; tests/dataset_reference.py restates it in numpy.
//
// Memory-bound: each output row is 128 fp16 values, 256 bytes, which 16 lanes move as one 16-byte vector each, so a
// warp reads and writes two whole rows per step.  The rows come through the item's row map (the mask augmentation
// resolved on the host), rows past the window or cleared by a zero mask are written as zeros, and the 16-bit values are
// copied as bits.  A second grid-stride pass gives every output frame one thread that writes its beat and downbeat
// targets (a binary search of the frame in the item's sorted frame list) and its padding flag, so every output element
// is written exactly once, without a zero-then-scatter pass.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "bt_kernels.h"

namespace bt {

namespace {

constexpr int kThreads = 256;
constexpr int kLanesPerRow = 16;  // BT_N_MELS fp16 values / 8 per 16-byte vector
constexpr int kRowsPerCta = kThreads / kLanesPerRow;
constexpr int kMaxCtas = 2048;  // grid-stride beyond this: about two waves of 8 resident CTAs on each of 132 SMs

// 1 when t is one of frames[lo, hi) (sorted, duplicates allowed)
__device__ __forceinline__ uint8_t has_frame(const int32_t* frames, int64_t lo, const int64_t end, int32_t t) {
  int64_t hi = end;
  while (lo < hi) {  // first position with frames[pos] >= t
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (frames[mid] < t) lo = mid + 1;
    else hi = mid;
  }
  return lo < end && frames[lo] == t ? 1 : 0;
}

__global__ void __launch_bounds__(kThreads)
train_batch_kernel(const uint4* __restrict__ rows, const int64_t* __restrict__ row_off, int length, int64_t total,
                   const int32_t* __restrict__ row_map, const int32_t* __restrict__ beats,
                   const int64_t* __restrict__ beat_off, const int32_t* __restrict__ downs,
                   const int64_t* __restrict__ down_off, uint4* __restrict__ spect, uint8_t* __restrict__ truth_beat,
                   uint8_t* __restrict__ truth_downbeat, uint8_t* __restrict__ padding_mask) {
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  const int64_t threads = static_cast<int64_t>(gridDim.x) * kThreads;
  const int lane = threadIdx.x % kLanesPerRow;
  // the rows: 16 lanes per output row
  for (int64_t r = tid / kLanesPerRow; r < total; r += threads / kLanesPerRow) {
    const int64_t b = r / length;
    const int32_t t = static_cast<int32_t>(r - b * length);
    const int64_t base = row_off[b];
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (t < row_off[b + 1] - base) {
      const int32_t src = row_map ? row_map[base + t] : t;
      if (src >= 0) v = __ldg(rows + (base + src) * kLanesPerRow + lane);
    }
    spect[r * kLanesPerRow + lane] = v;
  }
  // the targets: one thread per output frame, so the searches of many frames are in flight and the byte stores
  // coalesce
  for (int64_t r = tid; r < total; r += threads) {
    const int64_t b = r / length;
    const int32_t t = static_cast<int32_t>(r - b * length);
    const bool inside = t < row_off[b + 1] - row_off[b];
    truth_beat[r] = inside ? has_frame(beats, beat_off[b], beat_off[b + 1], t) : 0;
    truth_downbeat[r] = inside ? has_frame(downs, down_off[b], down_off[b + 1], t) : 0;
    padding_mask[r] = inside ? 1 : 0;
  }
}

}  // namespace

void launch_train_batch(const uint16_t* rows, const int64_t* row_off, int n_items, int length, const int32_t* row_map,
                        const int32_t* beats, const int64_t* beat_off, const int32_t* downs, const int64_t* down_off,
                        uint16_t* spect, uint8_t* truth_beat, uint8_t* truth_downbeat, uint8_t* padding_mask,
                        cudaStream_t st) {
  const int64_t total = static_cast<int64_t>(n_items) * length;
  if (total <= 0) return;
  const int64_t ctas = std::min<int64_t>((total + kRowsPerCta - 1) / kRowsPerCta, kMaxCtas);
  train_batch_kernel<<<static_cast<unsigned>(ctas), kThreads, 0, st>>>(
      reinterpret_cast<const uint4*>(rows), row_off, length, total, row_map, beats, beat_off, downs, down_off,
      reinterpret_cast<uint4*>(spect), truth_beat, truth_downbeat, padding_mask);
}

}  // namespace bt
