// The MP3 decode kernels of bt_mp3_decode (include/beatthis.h); the arithmetic is mp3.cuh's.
//
// mp3_granules_kernel: one thread per (frame, channel).  The serial part of Layer III is the Huffman walk of one granule
// and channel, and granule 1 may reuse granule 0's scalefactors (scfsi), so one thread walks both granules of its
// channel into their records: scalefactors, then the big-values and count1 lines.  The lookup tables sit in shared
// memory.
// mp3_hybrid_kernel: one CTA per (frame, granule), a thread per line: requantisation of both channels, stereo
// processing, short-block reordering and alias reduction in shared memory, then the IMDCT of the 2 x 32 subbands into
// the granule's stored 36-value blocks.
// mp3_synth_kernel: one CTA per granule: overlap-add with the previous granule's stored blocks, frequency inversion,
// the matrixing of this granule's 18 time slots and the 15 before it (read from the neighbouring granules' blocks, so
// there is no serial state across granules), the 512-tap window, the trim and the output mode.
// Every per-line array lives in shared memory or in the global scratch, so no kernel has local memory.
#include <cuda_runtime.h>

#include <cstdint>

#include "bt_kernels.h"
#include "mp3.cuh"

namespace bt {

namespace {

constexpr int kGranuleThreads = 64;
constexpr int kHybridThreads = mp3::kLines;
constexpr int kSynthThreads = 256;
constexpr int kPastSlots = 15;  // time slots before a granule that its synthesis reads

__device__ __forceinline__ const bt_mp3_frame& frame_of(const Mp3StreamDev& s, int64_t f) {
  return static_cast<const bt_mp3_frame*>(s.frames)[f];
}

__global__ void __launch_bounds__(kGranuleThreads) mp3_granules_kernel(const Mp3StreamDev* __restrict__ streams,
                                                                       const uint32_t* __restrict__ lut_g,
                                                                       int32_t* status) {
  __shared__ uint32_t lut[mp3::kLutEntries + 34];
  for (int i = threadIdx.x; i < mp3::kLutEntries + 34; i += kGranuleThreads) lut[i] = lut_g[i];
  __syncthreads();
  const Mp3StreamDev s = streams[blockIdx.y];
  const int64_t k = static_cast<int64_t>(blockIdx.x) * kGranuleThreads + threadIdx.x;
  if (k >= s.n_frames * s.channels || status[blockIdx.y] != BT_OK) return;
  const int64_t f = k / s.channels;
  const int ch = static_cast<int>(k % s.channels);
  const bt_mp3_frame& fr = frame_of(s, f);
  mp3::GranuleRec* recs = static_cast<mp3::GranuleRec*>(s.recs);
  const bool ok = mp3::decode_frame_channel(s.bytes, s.byte_count, fr.main_start, fr.header, fr.side_info, s.channels,
                                            ch, s.rate_index, lut, recs + f * 2 * s.channels);
  if (!ok) status[blockIdx.y] = BT_ERR_IO;
}

__global__ void __launch_bounds__(kHybridThreads) mp3_hybrid_kernel(const Mp3StreamDev* __restrict__ streams,
                                                                     const float* __restrict__ tables,
                                                                     const int32_t* __restrict__ status) {
  __shared__ float x[2][mp3::kLines], y[2][mp3::kLines];
  __shared__ float tt[mp3::kTransformTable];
  __shared__ int bound[4];
  const Mp3StreamDev s = streams[blockIdx.y];
  const int64_t g = blockIdx.x;  // granule of the stream
  if (g >= 2 * s.n_frames || status[blockIdx.y] != BT_OK) return;
  for (int i = threadIdx.x; i < mp3::kTransformTable; i += kHybridThreads) tt[i] = tables[i];
  if (threadIdx.x < 4) bound[threadIdx.x] = -1;
  __syncthreads();
  const mp3::GranuleRec* recs = static_cast<const mp3::GranuleRec*>(s.recs) + g * s.channels;
  const uint32_t header = frame_of(s, g / 2).header;
  const int i = threadIdx.x;
  mp3::hybrid_requant(recs, s.channels, s.rate_index, i, &x[0][0], bound);
  __syncthreads();
  mp3::hybrid_stereo(recs, s.channels, s.rate_index, header, i, &x[0][0], bound);
  __syncthreads();
  for (int c = 0; c < s.channels; ++c) y[c][i] = x[c][mp3::reorder_src(recs[c], s.rate_index, i)];
  __syncthreads();
  for (int c = 0; c < s.channels; ++c) x[c][i] = mp3::antialias(y[c], recs[c], i);
  __syncthreads();
  for (int c = 0; c < s.channels; ++c)
    for (int o = i; o < 32 * mp3::kBlock; o += kHybridThreads) {
      const int sb = o / mp3::kBlock, n = o % mp3::kBlock;
      s.blocks[((g * s.channels + c) * 32 + sb) * mp3::kBlock + n] = mp3::imdct_value(x[c] + 18 * sb, recs[c], sb, n, tt);
    }
}

__global__ void __launch_bounds__(kSynthThreads) mp3_synth_kernel(const Mp3StreamDev* __restrict__ streams,
                                                                   const float* __restrict__ tables, int mode,
                                                                   void* out, const int32_t* __restrict__ status) {
  __shared__ float win[512], ncos[64 * 32];
  __shared__ float S[mp3::kSlots + kPastSlots][32], V[mp3::kSlots + kPastSlots][64];
  __shared__ float pcm[2][mp3::kLines];
  const Mp3StreamDev s = streams[blockIdx.y];
  const int64_t g = blockIdx.x;  // the grid covers every output sample, decoded or not: a stream that is not decoded
  const int64_t first = g * mp3::kLines - s.skip;  // (bad status, no frames) still gets its zeros
  if (first >= s.n_samples || first + mp3::kLines <= 0) return;
  const bool ok = status[blockIdx.y] == BT_OK && g < 2 * s.n_frames;
  if (ok) {
    for (int i = threadIdx.x; i < 512; i += kSynthThreads) win[i] = tables[mp3::kWindowAt + i];
    for (int i = threadIdx.x; i < 64 * 32; i += kSynthThreads) ncos[i] = tables[mp3::kCosAt + i];
    for (int c = 0; c < s.channels; ++c) {
      __syncthreads();
      for (int e = threadIdx.x; e < (mp3::kSlots + kPastSlots) * 32; e += kSynthThreads)
        S[e / 32][e % 32] = mp3::slot_sample(s.blocks, s.channels, c, g, e / 32 - kPastSlots, e % 32);
      __syncthreads();
      for (int e = threadIdx.x; e < (mp3::kSlots + kPastSlots) * 64; e += kSynthThreads)
        V[e / 64][e % 64] = mp3::matrix_value(S[e / 64], ncos, e % 64);
      __syncthreads();
      for (int e = threadIdx.x; e < mp3::kLines; e += kSynthThreads)
        pcm[c][e] = mp3::window_sum(&V[0][0], win, kPastSlots + e / 32, e % 32);
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < mp3::kLines; e += kSynthThreads) {
    const int64_t t = first + e;
    if (t < 0 || t >= s.n_samples) continue;
    if (mode == BT_MP3_MONO_F32) {
      static_cast<float*>(out)[s.out_off + t] = ok ? mp3::mono_sample(pcm[0][e], pcm[1][e], s.channels) : 0.f;
    } else {
      double* o = static_cast<double*>(out) + s.out_off + t * s.channels;
      for (int c = 0; c < s.channels; ++c) o[c] = ok ? static_cast<double>(pcm[c][e]) : 0.0;
    }
  }
}

}  // namespace

void launch_mp3_granules(const Mp3StreamDev* streams_dev, int n_streams, int64_t max_frames, const uint32_t* lut,
                         int32_t* status, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>((2 * max_frames + kGranuleThreads - 1) / kGranuleThreads), n_streams);
  mp3_granules_kernel<<<grid, kGranuleThreads, 0, st>>>(streams_dev, lut, status);
}

void launch_mp3_hybrid(const Mp3StreamDev* streams_dev, int n_streams, int64_t max_frames, const float* tables,
                       const int32_t* status, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>(2 * max_frames), n_streams);
  mp3_hybrid_kernel<<<grid, kHybridThreads, 0, st>>>(streams_dev, tables, status);
}

void launch_mp3_synth(const Mp3StreamDev* streams_dev, int n_streams, int64_t max_granules, const float* tables,
                      int mode, void* out, const int32_t* status, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>(max_granules), n_streams);
  mp3_synth_kernel<<<grid, kSynthThreads, 0, st>>>(streams_dev, tables, mode, out, status);
}

}  // namespace bt
