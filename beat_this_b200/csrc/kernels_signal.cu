// Signal kernels (contracts of bt_logmel, bt_logmel_config, bt_resample, bt_stft, bt_phase_vocoder and bt_istft in
// include/beatthis.h): the log-mel front end, the polyphase resampler, and tempo and pitch augmentation -- a complex
// STFT, a phase vocoder that turns one analysis of a clip into any number of time-stretched variants, and the inverse
// STFT with overlap-add.  The grid-stride kernels logmel_config_kernel, stft_kernel and istft_frames_kernel are built
// on the FFT of fft.cuh and share one launcher; the two forward transforms also share framing and untangling.
#include <algorithm>
#include <type_traits>

#include "bt_kernels.h"
#include "fft.cuh"

namespace bt {

namespace {

constexpr int kMaxGridY = 65535;  // gridDim.y limit: logmel_kernel and resample_kernel loop over the clips beyond it

template <int LOG2N>
constexpr size_t fft_smem() { return MelGeom<LOG2N>::SPEC_OFF; }  // the FFT buffer of the CTA's FPC frames

// The first radix-8 pass's inputs v[r] = z[lt + r H/8] of frame g of the batch's frames flattened over all clips:
// z[n] = x[2n] + i x[2n+1] of the windowed frame, torch.stft(center=True, pad_mode="reflect"); zeros when
// g >= total_frames.  The frame finds its clip by binary search of frame_off.
template <int LOG2N>
__device__ __forceinline__ void stft_frame_load(float2 (&v)[8], int64_t g, int64_t total_frames,
                                                const float* __restrict__ audio, const int64_t* __restrict__ sample_off,
                                                const int64_t* __restrict__ frame_off, int n_clips, int hop,
                                                const float* __restrict__ window, int lt) {
  constexpr int N = MelGeom<LOG2N>::N, H = MelGeom<LOG2N>::H;
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
        if (i < 0) i = -i;                    // reflect without repeating the edge; check_stft_frames guarantees
        if (i >= len) i = 2 * (len - 1) - i;  // len > N/2, which makes one reflection enough
        xs[e] = __ldg(audio + s0 + i) * __ldg(window + n + e);
      }
      v[r] = make_float2(xs[0], xs[1]);
    }
  } else {
#pragma unroll
    for (int r = 0; r < 8; ++r) v[r] = make_float2(0.f, 0.f);
  }
}

// Bin k (0 <= k <= N/2) of the real N-point transform from Z, the H = N/2-point FFT of z in the padded buffer a:
// X[k] = E[k] + e^{-2 pi i k / N} O[k], E = (Z[k] + conj Z[H - k]) / 2, O = -i (Z[k] - conj Z[H - k]) / 2
template <int N>
__device__ __forceinline__ float2 untangle(const float2* a, int k, const float2* __restrict__ tw) {
  constexpr int H = N / 2;
  const float2 zk = a[mel_pad(k & (H - 1))], zc = a[mel_pad((H - k) & (H - 1))];
  const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y - zc.y));
  const float2 o = make_float2(0.5f * (zk.y + zc.y), -0.5f * (zk.x - zc.x));
  return cadd(e, cmul(mel_tw<N>(tw, k), o));
}

// Launches a grid-stride kernel of MelGeom<LOG2N> CTAs over total_frames frames: one CTA per group of FPC frames, but
// no more CTAs than the device holds at once (queried on the first launch of each kernel).
template <int LOG2N, auto kernel, class... Args>
cudaError_t launch_frame_groups(size_t smem, int64_t total_frames, cudaStream_t st, Args... args) {
  using G = MelGeom<LOG2N>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  static int max_ctas = 0;
  if (max_ctas == 0) {
    int dev = 0, sms = 0, per_sm = 0;
    e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, G::THREADS, smem);
    if (e != cudaSuccess) return e;
    max_ctas = std::max(1, sms * per_sm);
  }
  const int64_t groups = (total_frames + G::FPC - 1) / G::FPC;
  kernel<<<static_cast<unsigned>(std::min<int64_t>(groups, max_ctas)), G::THREADS, smem, st>>>(args...);
  return cudaSuccess;
}

// f(std::integral_constant<int, log2n>()) for the transform sizes the kernels are built for, n_fft = 64 ... 8192
template <class F>
cudaError_t with_log2n(int log2n, F f) {
  switch (log2n) {
    case 6: return f(std::integral_constant<int, 6>());
    case 7: return f(std::integral_constant<int, 7>());
    case 8: return f(std::integral_constant<int, 8>());
    case 9: return f(std::integral_constant<int, 9>());
    case 10: return f(std::integral_constant<int, 10>());
    case 11: return f(std::integral_constant<int, 11>());
    case 12: return f(std::integral_constant<int, 12>());
    case 13: return f(std::integral_constant<int, 13>());
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------
// log-mel: reference LogMelSpect.forward (beat_this/preprocessing.py:56-59) =
//   torch.stft(n_fft 1024, hop 441, periodic hann, center reflect, normalized) -> abs ->
//   mel filterbank (slaney, 128 bins, 30..11000 Hz) -> log1p(1000 x).
// Algorithmic HBM bytes: 441 new samples * 4 B read + 128 * 4 B written per frame.
//
// 64 threads per frame, two frames per CTA.  The real 1024-point transform is ONE complex 512-point FFT of
// z[n] = x[2n] + i x[2n+1] followed by the usual untangling step, and 512 = 8 * 8 * 8: three radix-8 passes with the
// eight points of a butterfly in registers,
//   n = 64 n1 + 8 n2 + n3,  k = k1 + 8 k2 + 64 k3:
//   A: thread (n2, n3)  DFT8 over n1, times e^{-2 pi i n2 k1 / 64}          -> T1[k1][n2][n3]
//   B: thread (k1, n3)  DFT8 over n2, times e^{-2 pi i n3 (k1 + 8 k2) / 512} -> T2[n3][k2][k1]
//   C: thread (k2, k1)  DFT8 over n3                                         -> Z[k1 + 8 k2 + 64 k3]
// i.e. two exchanges through shared memory (8-byte accesses, padded pitches: at most the natural two wavefronts per
// warp access) where the radix-2 version of round 1 made ten passes over separate re / im arrays -- that kernel was
// bound by the shared-memory pipe (ncu: l1tex data-pipe wavefronts 97 %), not by HBM.
// ------------------------------------------------------------------------------------------
constexpr int LM_P1 = 72, LM_P2 = 68;  // pitches (float2) of the two exchange buffers

__global__ void __launch_bounds__(128)
logmel_kernel(const float* __restrict__ audio, const int64_t* __restrict__ sample_off,
              const int64_t* __restrict__ frame_off, const float* __restrict__ window,
              const float2* __restrict__ twiddle, const int32_t* __restrict__ fb_start,
              const int32_t* __restrict__ fb_ptr, const float* __restrict__ fb_w,
              float* __restrict__ spect, int n_clips) {
  __shared__ float2 tw[512];                 // e^{-2 pi i j / 1024}, j < 512
  __shared__ float2 t1[2][8 * LM_P1];        // per frame: T1, later Z (512 entries)
  __shared__ float2 t2[2][8 * LM_P2];
  __shared__ float mag[2][516];
  const int tid = threadIdx.x, half = tid >> 6, lt = tid & 63;
  const int t = 2 * blockIdx.x + half;
  // clips blockIdx.y, blockIdx.y + gridDim.y, ...: a grid holds at most kMaxGridY clips, a call any number.  Each shared
  // array is rewritten for the next clip only after a barrier that follows this clip's last read of it.
  for (int clip = blockIdx.y; clip < n_clips; clip += gridDim.y) {
    const int64_t f0 = frame_off[clip];
    const int T = static_cast<int>(frame_off[clip + 1] - f0);
    if (2 * static_cast<int>(blockIdx.x) >= T) continue;  // whole CTA beyond the clip
    const bool active = t < T;
    const int64_t s0 = sample_off[clip];
    const int64_t len = sample_off[clip + 1] - s0;
    for (int i = tid; i < 512; i += 128) tw[i] = twiddle[i];
    auto TW = [&](int j) -> float2 {  // e^{-2 pi i j / 1024}, 0 <= j < 1024
      const float2 w = tw[j & 511];
      return (j & 512) ? make_float2(-w.x, -w.y) : w;
    };
    float2 v[8];
    float2* T1 = t1[half];
    float2* T2 = t2[half];
    {  // ---- pass A: thread (n2, n3) = lt, points z[64 n1 + lt] ----
#pragma unroll
      for (int n1 = 0; n1 < 8; ++n1) {
        const int n = 2 * (64 * n1 + lt);
        float xs[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          int64_t i = 441ll * t + (n + e) - 512;
          if (i < 0) i = -i;                      // reflect (no edge repeat), torch pad_mode="reflect"
          if (i >= len) i = 2 * (len - 1) - i;
          xs[e] = active ? audio[s0 + i] * __ldg(window + n + e) : 0.f;
        }
        v[n1] = make_float2(xs[0], xs[1]);
      }
    }
    __syncthreads();  // twiddle table
    {
      dft8(v);
      const int n2 = lt >> 3;
#pragma unroll
      for (int k1 = 0; k1 < 8; ++k1) T1[k1 * LM_P1 + lt] = k1 == 0 ? v[0] : cmul(v[k1], TW(16 * n2 * k1));
    }
    __syncthreads();
    {  // ---- pass B: thread (k1, n3) = lt ----
      const int k1 = lt >> 3, n3 = lt & 7;
#pragma unroll
      for (int n2 = 0; n2 < 8; ++n2) v[n2] = T1[k1 * LM_P1 + n2 * 8 + n3];
      dft8(v);
#pragma unroll
      for (int k2 = 0; k2 < 8; ++k2) T2[n3 * LM_P2 + k2 * 8 + k1] = cmul(v[k2], TW(2 * n3 * (k1 + 8 * k2)));
    }
    __syncthreads();
    {  // ---- pass C: thread (k2, k1) = lt -> Z[lt + 64 k3] (into T1's storage) ----
#pragma unroll
      for (int n3 = 0; n3 < 8; ++n3) v[n3] = T2[n3 * LM_P2 + lt];
      dft8(v);
#pragma unroll
      for (int k3 = 0; k3 < 8; ++k3) T1[lt + 64 * k3] = v[k3];
    }
    __syncthreads();
    // untangle: X[k] = E[k] + e^{-2 pi i k / 1024} O[k], E = (Z[k] + conj Z[512 - k]) / 2, O = -i (Z[k] - conj Z[512 - k]) / 2;
    // magnitudes of bins 0..512 (normalized=True -> 1 / sqrt(1024))
    for (int k = lt; k <= 512; k += 64) {
      const float2 zk = T1[k & 511], zc = T1[(512 - k) & 511];
      const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y - zc.y));
      const float2 o = make_float2(0.5f * (zk.y + zc.y), -0.5f * (zk.x - zc.x));
      const float2 x = cadd(e, cmul(TW(k), o));
      mag[half][k] = sqrtf(x.x * x.x + x.y * x.y) * 0.03125f;
    }
    __syncthreads();
    if (active) {
#pragma unroll
      for (int mm = 0; mm < 2; ++mm) {
        const int m = lt + 64 * mm;  // mel bin
        const int p0 = fb_ptr[m], p1 = fb_ptr[m + 1];
        const int k0 = fb_start[m];
        float acc = 0.f;
        for (int p = p0; p < p1; ++p) acc = fmaf(mag[half][k0 + (p - p0)], fb_w[p], acc);
        spect[(f0 + t) * 128 + m] = log1pf(1000.0f * acc);
      }
    }
  }
}

void launch_logmel(const float* audio, const int64_t* sample_off_dev, const int64_t* frame_off_dev,
                   int n_clips, int64_t max_frames, const float* window, const float* twiddle,
                   const int32_t* fb_start, const int32_t* fb_ptr, const float* fb_w, float* spect,
                   cudaStream_t st) {
  if (max_frames <= 0 || n_clips <= 0) return;
  dim3 grid(static_cast<unsigned>((max_frames + 1) / 2), static_cast<unsigned>(std::min(n_clips, kMaxGridY)));
  logmel_kernel<<<grid, 128, 0, st>>>(audio, sample_off_dev, frame_off_dev, window,
                                      reinterpret_cast<const float2*>(twiddle), fb_start, fb_ptr, fb_w, spect, n_clips);
}

// ------------------------------------------------------------------------------------------
// General log-mel (bt_logmel_config, contract in include/beatthis.h): STFT with any power-of-two n_fft = N in
// [64, 8192] and any hop -> |.|^power -> CSR mel filterbank -> log1p(log_multiplier x).
// Algorithmic HBM bytes: hop new samples * 4 B read + n_mels * 4 B written per frame.
//
// As in logmel_kernel, the real N-point transform is one complex H = N/2-point FFT of z[n] = x[2n] + i x[2n+1] and the
// untangling step; the FFT (fft.cuh) takes TPF = H/8 threads per frame.  A CTA of max(256, TPF) threads transforms
// FPC = threads / TPF consecutive frames of the batch's frames flattened over all clips (a frame finds its clip by
// binary search of frame_off; a CTA may span clips) and loops over frame groups grid-stride.
// ------------------------------------------------------------------------------------------
template <int LOG2N>
__global__ void __launch_bounds__(MelGeom<LOG2N>::THREADS)
logmel_config_kernel(const float* __restrict__ audio, const int64_t* __restrict__ sample_off,
                     const int64_t* __restrict__ frame_off, int n_clips, int64_t total_frames, MelConfigArgs p) {
  using G = MelGeom<LOG2N>;
  constexpr int N = G::N, H = G::H, TPF = G::TPF, FPC = G::FPC, THREADS = G::THREADS;
  extern __shared__ float4 mel_smem4[];
  unsigned char* const smem = reinterpret_cast<unsigned char*>(mel_smem4);
  float2* const fft = reinterpret_cast<float2*>(smem);
  float* const spec = reinterpret_cast<float*>(smem + G::SPEC_OFF);
  double* const red = reinterpret_cast<double*>(smem + G::RED_OFF);
  const float2* __restrict__ tw = reinterpret_cast<const float2*>(p.twiddle);
  const int tid = threadIdx.x, fl = tid / TPF, lt = tid % TPF;

  float scale = p.norm_mode == 1 ? rsqrtf(static_cast<float>(N)) : 1.f;
  if (p.norm_mode == 2) {  // 1 / sqrt(sum window^2), summed in float64 in a fixed order
    double s = 0.0;
    for (int i = tid; i < N; i += THREADS) s += static_cast<double>(p.window[i]) * p.window[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    s = 0.0;
    for (int w = 0; w < THREADS / 32; ++w) s += red[w];
    scale = static_cast<float>(1.0 / sqrt(s));
  }

  float2* const a = fft + fl * G::PITCH;
  float* const sp = spec + fl * (H + 1);
  for (int64_t g0 = static_cast<int64_t>(blockIdx.x) * FPC; g0 < total_frames; g0 += static_cast<int64_t>(gridDim.x) * FPC) {
    const int64_t g = g0 + fl;
    float2 v[8];
    stft_frame_load<LOG2N>(v, g, total_frames, audio, sample_off, frame_off, n_clips, p.hop, p.window, lt);
    mel_fft_from_registers<LOG2N>(a, v, lt, tw);
    // bins 0..H, then (scale |X|)^power
    for (int k = lt; k <= H; k += TPF) {
      const float2 x = untangle<N>(a, k, tw);
      const float m = sqrtf(x.x * x.x + x.y * x.y) * scale;
      sp[k] = p.power == 1.f ? m : (p.power == 2.f ? m * m : powf(m, p.power));
    }
    __syncthreads();
    // mel bands of the CTA's frames: consecutive threads write consecutive outputs
    const int nm = p.n_mels;
    for (int idx = tid; idx < FPC * nm; idx += THREADS) {
      const int f = idx / nm, m = idx - f * nm;
      if (g0 + f >= total_frames) break;
      const int q0 = __ldg(p.fb_ptr + m), q1 = __ldg(p.fb_ptr + m + 1);
      const float* s = spec + f * (H + 1) + __ldg(p.fb_start + m);
      float acc = 0.f;
      for (int q = q0; q < q1; ++q) acc = fmaf(s[q - q0], __ldg(p.fb_w + q), acc);
      p.spect[(g0 + f) * nm + m] = log1pf(p.log_multiplier * acc);
    }
  }
}

cudaError_t launch_logmel_config(int log2n, const float* audio, const int64_t* sample_off_dev,
                                 const int64_t* frame_off_dev, int n_clips, int64_t total_frames,
                                 const MelConfigArgs& p, cudaStream_t st) {
  if (n_clips <= 0 || total_frames <= 0) return cudaSuccess;
  return with_log2n(log2n, [&](auto l) {
    constexpr int L = decltype(l)::value;
    return launch_frame_groups<L, logmel_config_kernel<L>>(MelGeom<L>::SMEM, total_frames, st, audio, sample_off_dev,
                                                            frame_off_dev, n_clips, total_frames, p);
  });
}

// ------------------------------------------------------------------------------------------
// Polyphase resampler to 22.05 kHz: device stand-in for soxr.resample (reference inference.py:274-275; method and
// filter design in beat_this_b200/preprocessing.py, parity with soxr unpinned).
//   y[n] = sum_k coef[(n M) mod L][k] * x[floor(n M / L) - K/2 + 1 + k],  zeros outside the clip.
// One CTA = 256 consecutive output samples of one clip; the input span they read is staged in shared memory.
// Algorithmic HBM bytes: 4 B per input sample + 4 B per output sample (the L x K bank stays in L1/L2).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
resample_kernel(const float* __restrict__ in, const int64_t* __restrict__ in_off, float* __restrict__ out,
                const int64_t* __restrict__ out_off, int n_clips, const float* __restrict__ coef, int L, int M, int K) {
  extern __shared__ float xs[];
  const int64_t n0 = static_cast<int64_t>(blockIdx.x) * 256;
  // clips blockIdx.y, blockIdx.y + gridDim.y, ...: a grid holds at most kMaxGridY clips, a call any number
  for (int clip = blockIdx.y; clip < n_clips; clip += gridDim.y) {
    const int64_t s0 = in_off[clip], len = in_off[clip + 1] - s0;
    const int64_t o0 = out_off[clip], nout = out_off[clip + 1] - o0;
    if (n0 >= nout) continue;
    const int64_t n_last = min(n0 + 255, nout - 1);
    const int64_t j_lo = (n0 * M) / L - K / 2 + 1;
    const int span = static_cast<int>((n_last * M) / L - K / 2 + K - j_lo + 1);
    for (int i = threadIdx.x; i < span; i += 256) {
      const int64_t j = j_lo + i;
      xs[i] = (j >= 0 && j < len) ? in[s0 + j] : 0.f;
    }
    __syncthreads();
    const int64_t n = n0 + threadIdx.x;
    if (n < nout) {
      const int64_t nm = n * M;
      const int base = static_cast<int>(nm / L - K / 2 + 1 - j_lo);
      const float* c = coef + static_cast<int64_t>(nm % L) * K;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int k = 0;
      for (; k + 4 <= K; k += 4) {
        a0 = fmaf(__ldg(c + k), xs[base + k], a0);
        a1 = fmaf(__ldg(c + k + 1), xs[base + k + 1], a1);
        a2 = fmaf(__ldg(c + k + 2), xs[base + k + 2], a2);
        a3 = fmaf(__ldg(c + k + 3), xs[base + k + 3], a3);
      }
      for (; k < K; ++k) a0 = fmaf(__ldg(c + k), xs[base + k], a0);
      out[o0 + n] = (a0 + a1) + (a2 + a3);
    }
    __syncthreads();  // the next clip's span overwrites xs
  }
}

int64_t resample_smem(int L, int M, int K) { return ((255ll * M) / L + K + 2) * 4; }  // the staged input span

cudaError_t launch_resample(const float* in, const int64_t* in_off_dev, float* out, const int64_t* out_off_dev,
                            int n_clips, int64_t max_out, const float* coef, int L, int M, int K, cudaStream_t st) {
  if (n_clips <= 0 || max_out <= 0) return cudaSuccess;
  const int smem = static_cast<int>(resample_smem(L, M, K));
  const cudaError_t e = smem > 48 * 1024
      ? cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) : cudaSuccess;
  if (e != cudaSuccess) return e;
  dim3 grid(static_cast<unsigned>((max_out + 255) / 256), static_cast<unsigned>(std::min(n_clips, kMaxGridY)));
  resample_kernel<<<grid, 256, smem, st>>>(in, in_off_dev, out, out_off_dev, n_clips, coef, L, M, K);
  return cudaSuccess;
}

// ------------------------------------------------------------------------------------------
// STFT: torch.stft(n_fft = N, hop, window, center=True, pad_mode="reflect", onesided, not normalised).  Framing, FFT
// and untangling as logmel_config_kernel; the N/2 + 1 complex bins of a frame go out as they are.
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
    stft_frame_load<LOG2N>(v, g, total_frames, audio, sample_off, frame_off, n_clips, hop, window, lt);
    mel_fft_from_registers<LOG2N>(a, v, lt, tw);
    if (g < total_frames) {
      float2* const out = spec + g * (H + 1);
      for (int k = lt; k <= H; k += TPF) out[k] = untangle<N>(a, k, tw);
    }
    __syncthreads();  // the next group's first pass overwrites the buffer
  }
}

cudaError_t launch_stft(int log2n, const float* audio, const int64_t* sample_off_dev, const int64_t* frame_off_dev,
                        int n_clips, int64_t total_frames, const float* window, const float* twiddle, int hop, float* spec,
                        cudaStream_t st) {
  if (n_clips <= 0 || total_frames <= 0) return cudaSuccess;
  return with_log2n(log2n, [&](auto l) {
    constexpr int L = decltype(l)::value;
    return launch_frame_groups<L, stft_kernel<L>>(fft_smem<L>(), total_frames, st, audio, sample_off_dev, frame_off_dev,
                                                  n_clips, total_frames, window, reinterpret_cast<const float2*>(twiddle),
                                                  hop, reinterpret_cast<float2*>(spec));
  });
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

cudaError_t launch_istft_frames(int log2n, const float* spec, int64_t total_frames, const float* window,
                                const float* twiddle, float* frames, cudaStream_t st) {
  if (total_frames <= 0) return cudaSuccess;
  return with_log2n(log2n, [&](auto l) {
    constexpr int L = decltype(l)::value;
    return launch_frame_groups<L, istft_frames_kernel<L>>(fft_smem<L>(), total_frames, st,
                                                          reinterpret_cast<const float2*>(spec), total_frames, window,
                                                          reinterpret_cast<const float2*>(twiddle), frames);
  });
}

void launch_istft_ola(const float* frames, const int64_t* frame_off_dev, const int64_t* out_off_dev, int n_seqs,
                      int64_t max_out, const float* window, int n_fft, int hop, float* out, cudaStream_t st) {
  if (n_seqs <= 0 || max_out <= 0) return;
  dim3 grid(static_cast<unsigned>((max_out + 255) / 256), static_cast<unsigned>(n_seqs));
  istft_ola_kernel<<<grid, 256, 0, st>>>(frames, frame_off_dev, out_off_dev, window, n_fft, hop, out);
}

}  // namespace bt
