// Tempo and pitch augmentation (contracts of bt_stft, bt_phase_vocoder and bt_istft in include/beatthis.h): a complex
// STFT, a phase vocoder that turns one analysis of a clip into any number of time-stretched variants, and the inverse
// STFT with overlap-add.  The FFT is the one of the log-mel kernels (fft.cuh).
#include <algorithm>

#include "bt_kernels.h"
#include "fft.cuh"

namespace bt {

namespace {

// CTAs of `kernel` resident on the whole device at once: the grid of a grid-stride kernel
template <class Kernel>
cudaError_t resident_ctas(Kernel kernel, int threads, size_t smem, int* out) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem);
  if (e == cudaSuccess) *out = std::max(1, sms * per_sm);
  return e;
}

template <int LOG2N>
constexpr size_t fft_smem() { return MelGeom<LOG2N>::SPEC_OFF; }  // the FFT buffer of the CTA's FPC frames

}  // namespace

// ------------------------------------------------------------------------------------------
// STFT: torch.stft(n_fft = N, hop, window, center=True, pad_mode="reflect", onesided, not normalised).  Framing, reflect
// indexing, FFT and untangling as logmel_config_kernel; the N/2 + 1 complex bins of a frame go out as they are.
// Algorithmic HBM bytes: hop * 4 B read + (N/2 + 1) * 8 B written per frame.
// ------------------------------------------------------------------------------------------
template <int LOG2N>
__global__ void __launch_bounds__(MelGeom<LOG2N>::THREADS)
stft_kernel(const float* __restrict__ audio, const int64_t* __restrict__ sample_off, const int64_t* __restrict__ frame_off,
            int n_clips, int64_t total_frames, const float* __restrict__ window, const float2* __restrict__ tw, int hop,
            float2* __restrict__ spec) {
  using G = MelGeom<LOG2N>;
  constexpr int N = G::N, H = G::H, TPF = G::TPF, FPC = G::FPC;
  extern __shared__ float4 aug_smem4[];
  float2* const fft = reinterpret_cast<float2*>(aug_smem4);
  const int tid = threadIdx.x, fl = tid / TPF, lt = tid % TPF;
  float2* const a = fft + fl * G::PITCH;
  for (int64_t g0 = static_cast<int64_t>(blockIdx.x) * FPC; g0 < total_frames; g0 += static_cast<int64_t>(gridDim.x) * FPC) {
    const int64_t g = g0 + fl;
    float2 v[8];
    if (g < total_frames) {
      int lo = 0, hi = n_clips;  // frame_off[lo] <= g < frame_off[hi]
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(frame_off + mid) <= g) lo = mid; else hi = mid;
      }
      const int64_t s0 = __ldg(sample_off + lo), len = __ldg(sample_off + lo + 1) - s0;
      const int64_t base = (g - __ldg(frame_off + lo)) * hop - N / 2;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int n = 2 * (lt + r * (H / 8));
        float xs[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          int64_t i = base + n + e;
          if (i < 0) i = -i;                    // reflect without repeating the edge; len > N/2 makes one
          if (i >= len) i = 2 * (len - 1) - i;  // reflection enough
          xs[e] = __ldg(audio + s0 + i) * __ldg(window + n + e);
        }
        v[r] = make_float2(xs[0], xs[1]);
      }
    } else {
#pragma unroll
      for (int r = 0; r < 8; ++r) v[r] = make_float2(0.f, 0.f);
    }
    mel_fft_from_registers<LOG2N>(a, v, lt, tw);
    // untangle: X[k] = E[k] + e^{-2 pi i k / N} O[k], E = (Z[k] + conj Z[H - k]) / 2, O = -i (Z[k] - conj Z[H - k]) / 2
    if (g < total_frames) {
      float2* const out = spec + g * (H + 1);
      for (int k = lt; k <= H; k += TPF) {
        const float2 zk = a[mel_pad(k & (H - 1))], zc = a[mel_pad((H - k) & (H - 1))];
        const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y - zc.y));
        const float2 o = make_float2(0.5f * (zk.y + zc.y), -0.5f * (zk.x - zc.x));
        out[k] = cadd(e, cmul(mel_tw<N>(tw, k), o));
      }
    }
    __syncthreads();  // the next group's first pass overwrites the buffer
  }
}

template <int LOG2N>
static cudaError_t launch_stft_n(const float* audio, const int64_t* sample_off_dev, const int64_t* frame_off_dev, int n_clips,
                                 int64_t total_frames, const float* window, const float* twiddle, int hop, float* spec,
                                 cudaStream_t st) {
  using G = MelGeom<LOG2N>;
  constexpr size_t smem = fft_smem<LOG2N>();
  cudaError_t e = cudaFuncSetAttribute(stft_kernel<LOG2N>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  static int max_ctas = 0;
  if (max_ctas == 0 && (e = resident_ctas(stft_kernel<LOG2N>, G::THREADS, smem, &max_ctas)) != cudaSuccess) return e;
  const int64_t groups = (total_frames + G::FPC - 1) / G::FPC;
  stft_kernel<LOG2N><<<static_cast<unsigned>(std::min<int64_t>(groups, max_ctas)), G::THREADS, smem, st>>>(
      audio, sample_off_dev, frame_off_dev, n_clips, total_frames, window, reinterpret_cast<const float2*>(twiddle), hop,
      reinterpret_cast<float2*>(spec));
  return cudaSuccess;
}

#define BT_FFT_SIZES(CASE) CASE(6) CASE(7) CASE(8) CASE(9) CASE(10) CASE(11) CASE(12) CASE(13)

cudaError_t launch_stft(int log2n, const float* audio, const int64_t* sample_off_dev, const int64_t* frame_off_dev,
                        int n_clips, int64_t total_frames, const float* window, const float* twiddle, int hop, float* spec,
                        cudaStream_t st) {
  if (n_clips <= 0 || total_frames <= 0) return cudaSuccess;
  switch (log2n) {
#define BT_CASE(L) \
  case L: return launch_stft_n<L>(audio, sample_off_dev, frame_off_dev, n_clips, total_frames, window, twiddle, hop, spec, st);
    BT_FFT_SIZES(BT_CASE)
#undef BT_CASE
    default: return cudaErrorInvalidValue;
  }
}

// ------------------------------------------------------------------------------------------
// Phase vocoder.  One thread per (variant, bin) runs the serial scan over the variant's output frames; threads lie
// along the bins, so the two input frames a step reads and the output frame it writes are coalesced.  blockIdx.y is
// the variant: a caller that lists the variants of a clip together has them scheduled together, and they read the same
// analysis frames while those are in L2.
//
// Only e^{i phi_j} leaves the kernel, and wrap(x - omega_k) + omega_k = x (mod 2 pi): the expected advance omega_k
// cancels, so phi_j = angle X[0] + sum_{m < j} (angle X[i'_m] - angle X[i_m]) (mod 2 pi).  The sum is kept in
// float64 and reduced to [-pi, pi] after every step, so a step adds the errors of its two atan2f values (2 ulp of a
// value <= pi each, 2^-21 rad) and a float64 rounding: |error of phi_j| <= (2 j + 1) * 2^-21 rad, linear in j with no
// term that grows with the size of the phase.  (A float32 running sum of the unreduced increments, up to pi * hop
// each, has lost the phase after a few thousand frames.)
// Magnitude and angle of the two frames of a step stay in registers: a step computes only those it does not hold, and
// the newer frame becomes the older one when the scan reaches it.
// Algorithmic HBM bytes per variant: T * bins * 8 B read (once per clip if L2 serves the other variants) +
// T_out * bins * 8 B written.
// ------------------------------------------------------------------------------------------
constexpr int kVocoderThreads = 128;

__global__ void __launch_bounds__(kVocoderThreads)
phase_vocoder_kernel(const float2* __restrict__ spec, const VocoderVariant* __restrict__ variants, int bins,
                     float2* __restrict__ out) {
  const int k = blockIdx.x * kVocoderThreads + threadIdx.x;
  if (k >= bins) return;
  const VocoderVariant vt = variants[blockIdx.y];
  const float2* __restrict__ x = spec + vt.in_base * bins + k;
  float2* __restrict__ y = out + vt.out_base * bins + k;
  constexpr double kTwoPi = 6.283185307179586476925286766559;
  auto polar = [](float2 c, float& mag, float& ang) {
    mag = sqrtf(c.x * c.x + c.y * c.y);
    ang = atan2f(c.y, c.x);  // atan2f(0, 0) = 0
  };
  auto frame = [&](int64_t i) { return i < vt.T ? __ldg(x + i * bins) : make_float2(0.f, 0.f); };  // frames T, T + 1: zero
  int64_t c0 = 0, c1 = 1;  // the frames whose magnitude and angle (m0, a0) and (m1, a1) hold
  float m0, a0, m1, a1;
  polar(frame(0), m0, a0);
  polar(frame(1), m1, a1);
  double phi = a0;
  for (int64_t j = 0; j < vt.T_out; ++j) {
    const double s = static_cast<double>(j) * vt.rate;
    const int64_t i = static_cast<int64_t>(s);         // floor: s >= 0
    const int64_t i1 = static_cast<int64_t>(s + 1.0);  // i + 1, or i + 2 where the sum rounds up to an integer
    const float alpha = static_cast<float>(s - static_cast<double>(i));
    if (i != c0) {
      if (i == c1) { m0 = m1; a0 = a1; } else polar(frame(i), m0, a0);
      c0 = i;
    }
    if (i1 != c1) {
      polar(frame(i1), m1, a1);
      c1 = i1;
    }
    const float mag = alpha * m1 + (1.f - alpha) * m0;
    float sn, cs;
    sincosf(static_cast<float>(phi), &sn, &cs);
    y[j * bins] = make_float2(mag * cs, mag * sn);
    phi += static_cast<double>(a1) - static_cast<double>(a0);
    phi -= kTwoPi * rint(phi / kTwoPi);
  }
}

void launch_phase_vocoder(const float* spec, const VocoderVariant* variants_dev, int n_variants, int bins, float* out,
                          cudaStream_t st) {
  if (n_variants <= 0) return;
  dim3 grid(static_cast<unsigned>((bins + kVocoderThreads - 1) / kVocoderThreads), static_cast<unsigned>(n_variants));
  phase_vocoder_kernel<<<grid, kVocoderThreads, 0, st>>>(reinterpret_cast<const float2*>(spec), variants_dev, bins,
                                                         reinterpret_cast<float2*>(out));
}

// ------------------------------------------------------------------------------------------
// Inverse STFT in two launches.  istft_frames_kernel: the inverse real transform of every frame times the window, N
// floats per frame into scratch.  The N real samples come from one complex H-point FFT: with E[k] = (X[k] + conj
// X[H - k]) / 2 and O[k] = (X[k] - conj X[H - k]) / 2 * e^{+2 pi i k / N} (the spectra of the even and the odd
// samples), z = IFFT_H(E + i O) has x[2n] = Re z[n], x[2n + 1] = Im z[n], and IFFT_H(Z) = conj(FFT_H(conj Z)) / H runs
// the forward passes.  The imaginary parts of X[0] and X[H] are ignored, as a complex-to-real transform does.
// istft_ola_kernel: output sample n of a sequence gathers the frames f with 0 <= n + N/2 - f hop < N in ascending f,
// and divides by the window envelope sum w^2 summed the same way, so a sample depends on its own sequence's frames only
// and on no order of execution: results are bitwise repeatable and independent of the batch, with no atomics.  Samples
// that no frame covers are zero.
// Two launches rather than one CTA that keeps a run of frames in shared memory: that form transforms a halo of
// N/hop - 1 frames twice per run and needs a run length per (N, hop); this one pays 2 * 4 N B of HBM traffic per frame
// for the scratch on top of the (N/2 + 1) * 8 B read and hop * 4 B written.
// ------------------------------------------------------------------------------------------
template <int LOG2N>
__global__ void __launch_bounds__(MelGeom<LOG2N>::THREADS)
istft_frames_kernel(const float2* __restrict__ spec, int64_t total_frames, const float* __restrict__ window,
                    const float2* __restrict__ tw, float* __restrict__ frames) {
  using G = MelGeom<LOG2N>;
  constexpr int N = G::N, H = G::H, TPF = G::TPF, FPC = G::FPC;
  extern __shared__ float4 aug_smem4[];
  float2* const fft = reinterpret_cast<float2*>(aug_smem4);
  const int tid = threadIdx.x, fl = tid / TPF, lt = tid % TPF;
  float2* const a = fft + fl * G::PITCH;
  for (int64_t g0 = static_cast<int64_t>(blockIdx.x) * FPC; g0 < total_frames; g0 += static_cast<int64_t>(gridDim.x) * FPC) {
    const int64_t g = g0 + fl;
    float2 v[8];
    if (g < total_frames) {
      const float2* __restrict__ X = spec + g * (H + 1);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int k = lt + r * (H / 8);
        float2 xk = __ldg(X + k), xc = __ldg(X + H - k);
        if (k == 0) { xk.y = 0.f; xc.y = 0.f; }
        const float2 e = make_float2(0.5f * (xk.x + xc.x), 0.5f * (xk.y - xc.y));
        const float2 d = make_float2(0.5f * (xk.x - xc.x), 0.5f * (xk.y + xc.y));
        const float2 w = mel_tw<N>(tw, k);                     // e^{-2 pi i k / N}
        const float2 o = cmul(d, make_float2(w.x, -w.y));      // O[k]
        v[r] = make_float2(e.x - o.y, -(e.y + o.x));           // conj(E + i O)
      }
    } else {
#pragma unroll
      for (int r = 0; r < 8; ++r) v[r] = make_float2(0.f, 0.f);
    }
    mel_fft_from_registers<LOG2N>(a, v, lt, tw);
    if (g < total_frames) {
      constexpr float inv = 1.f / H;
      float2* const out = reinterpret_cast<float2*>(frames + g * N);
      for (int n = lt; n < H; n += TPF) {
        const float2 z = a[mel_pad(n)];
        out[n] = make_float2(z.x * inv * __ldg(window + 2 * n), -z.y * inv * __ldg(window + 2 * n + 1));
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
istft_ola_kernel(const float* __restrict__ frames, const int64_t* __restrict__ frame_off,
                 const int64_t* __restrict__ out_off, const float* __restrict__ window, int N, int hop,
                 float* __restrict__ out) {
  const int seq = blockIdx.y;
  const int64_t o0 = out_off[seq], nout = out_off[seq + 1] - o0;
  const int64_t n = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (n >= nout) return;
  const int64_t f0 = frame_off[seq], F = frame_off[seq + 1] - f0;
  const int64_t p = n + N / 2;
  const int64_t f_hi = min(F - 1, p / hop);
  const int64_t f_lo = p < N ? 0 : (p - N) / hop + 1;
  float acc = 0.f, env = 0.f;
  for (int64_t f = f_lo; f <= f_hi; ++f) {
    const int m = static_cast<int>(p - f * hop);
    const float w = __ldg(window + m);
    acc += frames[(f0 + f) * N + m];
    env = fmaf(w, w, env);
  }
  out[o0 + n] = f_lo <= f_hi ? acc / env : 0.f;
}

template <int LOG2N>
static cudaError_t launch_istft_frames_n(const float* spec, int64_t total_frames, const float* window, const float* twiddle,
                                         float* frames, cudaStream_t st) {
  using G = MelGeom<LOG2N>;
  constexpr size_t smem = fft_smem<LOG2N>();
  cudaError_t e = cudaFuncSetAttribute(istft_frames_kernel<LOG2N>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  static int max_ctas = 0;
  if (max_ctas == 0 && (e = resident_ctas(istft_frames_kernel<LOG2N>, G::THREADS, smem, &max_ctas)) != cudaSuccess) return e;
  const int64_t groups = (total_frames + G::FPC - 1) / G::FPC;
  istft_frames_kernel<LOG2N><<<static_cast<unsigned>(std::min<int64_t>(groups, max_ctas)), G::THREADS, smem, st>>>(
      reinterpret_cast<const float2*>(spec), total_frames, window, reinterpret_cast<const float2*>(twiddle), frames);
  return cudaSuccess;
}

cudaError_t launch_istft_frames(int log2n, const float* spec, int64_t total_frames, const float* window,
                                const float* twiddle, float* frames, cudaStream_t st) {
  if (total_frames <= 0) return cudaSuccess;
  switch (log2n) {
#define BT_CASE(L) \
  case L: return launch_istft_frames_n<L>(spec, total_frames, window, twiddle, frames, st);
    BT_FFT_SIZES(BT_CASE)
#undef BT_CASE
    default: return cudaErrorInvalidValue;
  }
}

void launch_istft_ola(const float* frames, const int64_t* frame_off_dev, const int64_t* out_off_dev, int n_seqs,
                      int64_t max_out, const float* window, int n_fft, int hop, float* out, cudaStream_t st) {
  if (n_seqs <= 0 || max_out <= 0) return;
  dim3 grid(static_cast<unsigned>((max_out + 255) / 256), static_cast<unsigned>(n_seqs));
  istft_ola_kernel<<<grid, 256, 0, st>>>(frames, frame_off_dev, out_off_dev, window, n_fft, hop, out);
}

}  // namespace bt
