// The FLAC decode kernels of bt_flac_decode (include/beatthis.h).
//
// flac_frames_kernel: one thread per frame.  The serial unit of FLAC is a subframe, and a frame's subframes follow one
// another in the bit stream, so one thread walks its frame from the header to the CRC (flac.cuh): CRC-16, each
// subframe into the stream's int64 scratch [channels][n_samples], then the channel decorrelation in place.  The CRC
// table and the LPC coefficients sit in shared memory (coefficients at a stride of the block's width, so a thread's
// 32 slots are one bank each); nothing is indexed on the stack, so the kernel has no local memory.
// flac_output_kernel: one thread per sample, coalesced over time: the mono fp32 mix or the float64 channels.
#include <cuda_runtime.h>

#include <cstdint>

#include "bt_kernels.h"
#include "flac.cuh"

namespace bt {

namespace {

constexpr int kFrameThreads = 32;
constexpr int kOutThreads = 256;

__global__ void __launch_bounds__(kFrameThreads) flac_frames_kernel(const FlacStreamDev* __restrict__ streams,
                                                                    int32_t* status) {
  __shared__ uint16_t crc16[256];
  __shared__ int32_t coef[32 * kFrameThreads];
  for (int b = threadIdx.x; b < 256; b += kFrameThreads) crc16[b] = flac::crc16_byte_slow(0, static_cast<uint8_t>(b));
  __syncthreads();
  const FlacStreamDev s = streams[blockIdx.y];
  const int64_t k = static_cast<int64_t>(blockIdx.x) * kFrameThreads + threadIdx.x;
  if (k >= s.n_frames || status[blockIdx.y] != BT_OK) return;
  const bt_flac_frame fr = static_cast<const bt_flac_frame*>(s.frames)[k];
  // the table is the caller's: a frame outside its stream's bytes or samples is malformed, never read
  bool ok = fr.offset >= 0 && fr.bytes > 0 && fr.offset <= s.byte_count - fr.bytes && fr.block_size >= 1 &&
            fr.first_sample >= 0 && fr.first_sample <= s.n_samples - fr.block_size;
  if (ok)
    ok = flac::decode_frame(s.bytes + fr.offset, fr.bytes, fr.block_size, s.channels, s.bits, crc16,
                            s.scratch + fr.first_sample, s.n_samples, coef + threadIdx.x, kFrameThreads);
  if (!ok) status[blockIdx.y] = BT_ERR_IO;
}

__global__ void __launch_bounds__(kOutThreads) flac_output_kernel(const FlacStreamDev* __restrict__ streams, int mode,
                                                                  void* out, const int32_t* __restrict__ status) {
  const FlacStreamDev s = streams[blockIdx.y];
  const int64_t t = static_cast<int64_t>(blockIdx.x) * kOutThreads + threadIdx.x;
  if (t >= s.n_samples) return;
  const bool ok = status[blockIdx.y] == BT_OK;
  const double scale = flac::scale_of(s.bits);
  if (mode == BT_FLAC_MONO_F32) {
    static_cast<float*>(out)[s.out_off + t] = ok ? flac::mono_sample(s.scratch + t, s.n_samples, s.channels, scale) : 0.f;
  } else {
    double* o = static_cast<double*>(out) + s.out_off + t * s.channels;
    for (int c = 0; c < s.channels; ++c)
      o[c] = ok ? static_cast<double>(s.scratch[c * s.n_samples + t]) * scale : 0.0;
  }
}

}  // namespace

void launch_flac_frames(const FlacStreamDev* streams_dev, int n_streams, int64_t max_frames, int32_t* status,
                        cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>((max_frames + kFrameThreads - 1) / kFrameThreads), n_streams);
  flac_frames_kernel<<<grid, kFrameThreads, 0, st>>>(streams_dev, status);
}

void launch_flac_output(const FlacStreamDev* streams_dev, int n_streams, int64_t max_samples, int mode, void* out,
                        const int32_t* status, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>((max_samples + kOutThreads - 1) / kOutThreads), n_streams);
  flac_output_kernel<<<grid, kOutThreads, 0, st>>>(streams_dev, mode, out, status);
}

}  // namespace bt
