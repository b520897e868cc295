// The Vorbis decode kernels of bt_vorbis_decode (include/beatthis.h); the arithmetic is vorbis.cuh's.
//
// vorbis_packets_kernel: one thread per audio packet.  A packet's bit stream is serial across its channels (residue 2
// interleaves them, and each floor starts where the one before ended), so one thread walks it: floor1 posts of every
// channel, nonzero propagation, then the residue vectors of every submap into the packet's spectrum scratch.  The
// decode tables are read through the read-only cache, within the packet's bytes and the stream's tables.
// vorbis_blocks_kernel: one CTA per packet: floor1 step 2 (a thread per channel), inverse coupling (a thread per line),
// then per channel floor x residue, the IMDCT as an n/4-point Stockham FFT between two shared buffers with pre- and
// post-twiddles, and the window chosen by the block flags, written over the channel's spectrum.
// vorbis_output_kernel: one thread per output sample: overlap-add of the two packets that hold it, trim and output
// mode; zeros for a stream that is not decoded.
// Every per-line array lives in shared memory or in the global scratch, so no kernel has local memory.
#include <cuda_runtime.h>

#include <cstdint>

#include "bt_kernels.h"
#include "vorbis.cuh"

namespace bt {

namespace {

namespace vb = vorbis;

constexpr int kPacketThreads = 64;
constexpr int kBlockThreads = 256;
constexpr int kOutputThreads = 256;
constexpr int kMaxH = 1 << (vb::kMaxLog2 - 2);  // FFT points of the longest block

// A register cap rather than __launch_bounds__(64): with the bounds ptxas settles on 72 registers and spills.
__global__ void __maxnreg__(128) vorbis_packets_kernel(const vb::StreamDev* __restrict__ streams,
                                                                        int32_t* status) {
  const vb::StreamDev& s = streams[blockIdx.y];  // read in place: a by-value copy whose address is taken goes to local memory
  const int64_t p = static_cast<int64_t>(blockIdx.x) * kPacketThreads + threadIdx.x;
  if (p >= s.n_packets || status[blockIdx.y] != BT_OK) return;
  if (vb::decode_packet(s, p) != BT_OK) status[blockIdx.y] = BT_ERR_IO;
}

__global__ void __launch_bounds__(kBlockThreads) vorbis_blocks_kernel(const vb::StreamDev* __restrict__ streams,
                                                                      const float* __restrict__ tables,
                                                                      const int32_t* __restrict__ status) {
  __shared__ vb::BlockShared sh;
  __shared__ float2 buf[2][kMaxH];
  const vb::StreamDev s = streams[blockIdx.y];
  const int64_t p = blockIdx.x;
  if (p >= s.n_packets || status[blockIdx.y] != BT_OK) return;
  const vb::BlockGeom g = vb::block_geom(s, p);
  const int H = g.n / 4, tid = threadIdx.x;
  if (tid < s.channels) vb::block_floor(s, p, g, tid, &sh);
  for (int i = tid; i < g.n / 2; i += kBlockThreads) vb::block_couple(s, p, g, i);
  __syncthreads();
  for (int c = 0; c < s.channels; ++c) {
    for (int k = tid; k < H; k += kBlockThreads) vb::block_pre(s, p, g, c, &sh, tables, k, buf[0]);
    __syncthreads();
    int cur = 0;
    for (int Ns = 1; Ns < H;) {
      const int R = vb::pass_radix(H, Ns);
      for (int j = tid; j < H / R; j += kBlockThreads) vb::block_pass(buf[cur], buf[cur ^ 1], j, Ns, R, g, tables);
      __syncthreads();
      cur ^= 1;
      Ns *= R;
    }
    float* u = reinterpret_cast<float*>(buf[cur ^ 1]);
    for (int k = tid; k < H; k += kBlockThreads) vb::post_twiddle(buf[cur], vb::sig(tables, g.n), g.n, k, u);
    __syncthreads();
    for (int i = tid; i < g.n; i += kBlockThreads) vb::block_out(s, p, g, c, &sh, tables, u, i);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kOutputThreads) vorbis_output_kernel(const vb::StreamDev* __restrict__ streams,
                                                                       int mode, void* out,
                                                                       const int32_t* __restrict__ status) {
  const vb::StreamDev s = streams[blockIdx.y];
  const int64_t t = static_cast<int64_t>(blockIdx.x) * kOutputThreads + threadIdx.x;
  if (t >= s.n_samples) return;
  const bool ok = status[blockIdx.y] == BT_OK && s.n_packets > 0;
  if (mode == BT_VORBIS_MONO_F32) {
    static_cast<float*>(out)[s.out_off + t] = ok ? vb::output_mono(s, t) : 0.f;
  } else {
    double* o = static_cast<double*>(out) + s.out_off + t * s.channels;
    for (int c = 0; c < s.channels; ++c) o[c] = ok ? static_cast<double>(vb::output_sample(s, t, c)) : 0.0;
  }
}

}  // namespace

void launch_vorbis_packets(const vorbis::StreamDev* streams_dev, int n_streams, int64_t max_packets, int32_t* status,
                           cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>((max_packets + kPacketThreads - 1) / kPacketThreads), n_streams);
  vorbis_packets_kernel<<<grid, kPacketThreads, 0, st>>>(streams_dev, status);
}

void launch_vorbis_blocks(const vorbis::StreamDev* streams_dev, int n_streams, int64_t max_packets, const float* tables,
                          const int32_t* status, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>(max_packets), n_streams);
  vorbis_blocks_kernel<<<grid, kBlockThreads, 0, st>>>(streams_dev, tables, status);
}

void launch_vorbis_output(const vorbis::StreamDev* streams_dev, int n_streams, int64_t max_samples, int mode, void* out,
                          const int32_t* status, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>((max_samples + kOutputThreads - 1) / kOutputThreads), n_streams);
  vorbis_output_kernel<<<grid, kOutputThreads, 0, st>>>(streams_dev, mode, out, status);
}

}  // namespace bt
