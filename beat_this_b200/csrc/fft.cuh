// Device pieces of the shared-memory FFT that the log-mel, STFT and inverse STFT kernels (kernels_signal.cu) are built
// from: complex helpers, the register DFTs and the passes of the Stockham FFT.
#pragma once
#include <cuda_runtime.h>

namespace bt {

__host__ __device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__host__ __device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__host__ __device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__host__ __device__ __forceinline__ float2 cmul_mi(float2 a) { return make_float2(a.y, -a.x); }  // a * (-i)

// in-place 8-point DFT (e^{-2 pi i nk/8}), natural order in and out
__host__ __device__ __forceinline__ void dft8(float2 (&v)[8]) {
  constexpr float R = 0.70710678118654752f;
  float2 a[4], b[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { a[j] = cadd(v[j], v[j + 4]); b[j] = csub(v[j], v[j + 4]); }
  b[1] = make_float2(R * (b[1].x + b[1].y), R * (b[1].y - b[1].x));    // * (1 - i) / sqrt 2
  b[2] = cmul_mi(b[2]);                                                 // * (-i)
  b[3] = make_float2(R * (b[3].y - b[3].x), -R * (b[3].x + b[3].y));   // * (-1 - i) / sqrt 2
  auto dft4 = [](const float2 (&c)[4], float2& y0, float2& y1, float2& y2, float2& y3) {
    const float2 s0 = cadd(c[0], c[2]), s1 = csub(c[0], c[2]), s2 = cadd(c[1], c[3]), s3 = cmul_mi(csub(c[1], c[3]));
    y0 = cadd(s0, s2); y2 = csub(s0, s2); y1 = cadd(s1, s3); y3 = csub(s1, s3);
  };
  dft4(a, v[0], v[2], v[4], v[6]);
  dft4(b, v[1], v[3], v[5], v[7]);
}

// ------------------------------------------------------------------------------------------
// The real N-point transform of a frame is one complex H = N/2-point FFT of z[n] = x[2n] + i x[2n+1] and an
// untangling step.  The complex FFT is a Stockham autosort FFT: radix-8 passes while 8 divides what is left, then one
// radix-4 or radix-2 pass.  The pass of radix R after the passes whose radices multiply to Ns has butterflies
// j < H/R: read a[j + r H/R] (r < R), multiply by e^{-2 pi i (j mod Ns) r / (Ns R)}, take a DFT_R and write
// a[(j - j mod Ns) R + j mod Ns + r Ns].  After the last pass Z is in natural order.  Every thread holds eight points
// in registers per pass (one radix-8, two radix-4 or four radix-2 butterflies), so TPF = H/8 threads work on a frame
// and one buffer suffices: a __syncthreads separates each pass's reads from its writes.  Buffer index i is stored at
// i + i/8: the first pass writes with a stride of 8 points, which the padding spreads over all banks.
// A CTA of max(256, TPF) threads transforms FPC = threads / TPF frames at a time.  Twiddles e^{-2 pi i j / N}
// (j < N/2) come from the caller's table through the read-only cache.
// ------------------------------------------------------------------------------------------
template <int LOG2N>
struct MelGeom {
  static constexpr int N = 1 << LOG2N, H = N / 2, TPF = H / 8;
  static constexpr int THREADS = TPF > 256 ? TPF : 256, FPC = THREADS / TPF;
  static constexpr int PITCH = H + H / 8;  // float2 per frame in the FFT buffer
  static constexpr size_t SPEC_OFF = size_t(FPC) * PITCH * sizeof(float2);  // bytes; FPC x (H + 1) floats follow
  static constexpr size_t RED_OFF = (SPEC_OFF + size_t(FPC) * (H + 1) * sizeof(float) + 7) / 8 * 8;  // 32 doubles
  static constexpr size_t SMEM = RED_OFF + 32 * sizeof(double);
};

__device__ __forceinline__ int mel_pad(int i) { return i + (i >> 3); }

template <int N>
__device__ __forceinline__ float2 mel_tw(const float2* __restrict__ tw, int j) {  // e^{-2 pi i j / N}, 0 <= j <= N/2
  const float2 w = __ldg(tw + (j & (N / 2 - 1)));
  return (j & (N / 2)) ? make_float2(-w.x, -w.y) : w;
}

__host__ __device__ __forceinline__ void dft4(float2& a0, float2& a1, float2& a2, float2& a3) {
  const float2 s0 = cadd(a0, a2), s1 = csub(a0, a2), s2 = cadd(a1, a3), s3 = cmul_mi(csub(a1, a3));
  a0 = cadd(s0, s2); a2 = csub(s0, s2); a1 = cadd(s1, s3); a3 = csub(s1, s3);
}

// twiddles, DFT_R and stores of the thread's 8 / R butterflies j = lt + b TPF of the pass after Ns points
template <int R, int LOG2N>
__device__ __forceinline__ void mel_pass_store(float2* __restrict__ a, float2 (&v)[8], int lt, int Ns,
                                               const float2* __restrict__ tw) {
  using G = MelGeom<LOG2N>;
#pragma unroll
  for (int b = 0; b < 8 / R; ++b) {
    const int j = lt + b * G::TPF, k = j & (Ns - 1);
    const int step = G::N / (Ns * R);  // e^{-2 pi i k r / (Ns R)} = e^{-2 pi i k r step / N}
#pragma unroll
    for (int r = 1; r < R; ++r) v[b * R + r] = cmul(v[b * R + r], mel_tw<G::N>(tw, k * r * step));
    if constexpr (R == 8) {
      dft8(v);
    } else if constexpr (R == 4) {
      dft4(v[4 * b], v[4 * b + 1], v[4 * b + 2], v[4 * b + 3]);
    } else {
      const float2 t = v[2 * b];
      v[2 * b] = cadd(t, v[2 * b + 1]);
      v[2 * b + 1] = csub(t, v[2 * b + 1]);
    }
    const int d = (j - k) * R + k;
#pragma unroll
    for (int r = 0; r < R; ++r) a[mel_pad(d + r * Ns)] = v[b * R + r];
  }
}

template <int R, int LOG2N>
__device__ __forceinline__ void mel_pass_load(const float2* __restrict__ a, float2 (&v)[8], int lt) {
  using G = MelGeom<LOG2N>;
#pragma unroll
  for (int b = 0; b < 8 / R; ++b)
#pragma unroll
    for (int r = 0; r < R; ++r) v[b * R + r] = a[mel_pad(lt + b * G::TPF + r * (G::H / R))];
}

// The passes after the first radix-8 pass (whose inputs the caller holds in v): on return the H points are in a, in
// natural order, and a __syncthreads has made them visible to the CTA.
template <int LOG2N>
__device__ __forceinline__ void mel_fft_from_registers(float2* __restrict__ a, float2 (&v)[8], int lt,
                                                       const float2* __restrict__ tw) {
  constexpr int LOG2H = LOG2N - 1, N8 = LOG2H / 3, REM = LOG2H % 3;
  mel_pass_store<8, LOG2N>(a, v, lt, 1, tw);
  __syncthreads();
#pragma unroll
  for (int q = 1; q < N8; ++q) {
    mel_pass_load<8, LOG2N>(a, v, lt);
    __syncthreads();
    mel_pass_store<8, LOG2N>(a, v, lt, 1 << (3 * q), tw);
    __syncthreads();
  }
  if constexpr (REM != 0) {
    constexpr int R = 1 << REM;
    mel_pass_load<R, LOG2N>(a, v, lt);
    __syncthreads();
    mel_pass_store<R, LOG2N>(a, v, lt, 1 << (3 * N8), tw);
    __syncthreads();
  }
}

}  // namespace bt
