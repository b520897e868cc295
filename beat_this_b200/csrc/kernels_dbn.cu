// Postprocessor("dbn") on the device: the bar-pointer Viterbi of the host tracker (dbn_host.cpp, Tracker::track and the
// ring-buffer branch of viterbi()) restated as three kernels.  The arithmetic is the host's, operation for operation
// (explicit _rn intrinsics, so nvcc cannot contract an add into an FMA), and every argmax keeps the host's tie-break:
// for equal inputs the scores are bitwise equal and the decoded beats identical.
//
//   dbn_prep       one CTA per clip: activations (sigmoid + eps clamps of postprocessor.py:139-167, or given), the three
//                  log densities per frame, and the threshold window of Tracker::track
//   dbn_viterbi    one CTA per (clip, bar model), one thread per (beat, tempo): ring values and log_tempo in shared
//                  memory, one byte back pointer per (frame, beat, tempo), final (value, lowest state) reduction
//   dbn_backtrace  one thread per clip: best model, backtrace, beat correction, (time, number) pairs
#include <cuda_runtime.h>
#include <math_constants.h>

#include <climits>
#include <cstdint>

#include "bt_kernels.h"

namespace bt {

namespace {

constexpr int kCodeInBeat = 0x80;  // path code of a frame: beat number (1..127) | kCodeInBeat on a (down)beat position

__device__ __forceinline__ double clamp_prob(double x) {
  // torch sigmoid (1 / (1 + exp(-x)), postprocessor.py:139-140) then p * (1 - eps) + eps / 2 (:141-142), rounded
  // after every operation as numpy does
  const double p = __ddiv_rn(1.0, __dadd_rn(1.0, exp(-x)));
  return __dadd_rn(__dmul_rn(p, 1.0 - 1e-5), 1e-5 / 2);
}

__global__ void __launch_bounds__(256)
dbn_prep_kernel(const float* __restrict__ beat, const float* __restrict__ down, const double* __restrict__ act_in,
                const int64_t* __restrict__ fo, double threshold, double observation_lambda, double* __restrict__ act,
                double* __restrict__ dens, int64_t* __restrict__ win) {
  __shared__ long long s_lo, s_hi;
  const int clip = blockIdx.x;
  const int64_t f0 = fo[clip], T = fo[clip + 1] - f0;
  if (threadIdx.x == 0) { s_lo = LLONG_MAX; s_hi = -1; }
  __syncthreads();
  const double half_eps = 1e-5 / 2, lam1 = observation_lambda - 1.0;
  long long lo = LLONG_MAX, hi = -1;
  for (int64_t t = threadIdx.x; t < T; t += blockDim.x) {
    const int64_t g = f0 + t;
    double a0, a1;
    if (act_in) {
      a0 = act_in[2 * g];
      a1 = act_in[2 * g + 1];
    } else {  // (max(bp - dp, eps / 2), dp): the artificial multiclass prediction of postprocessor.py:159-167
      const double bp = clamp_prob(static_cast<double>(beat[g])), dp = clamp_prob(static_cast<double>(down[g]));
      const double dd = __dsub_rn(bp, dp);
      a0 = dd < half_eps ? half_eps : dd;  // np.maximum: a NaN stays NaN
      a1 = dp;
    }
    act[2 * g] = a0;
    act[2 * g + 1] = a1;
    dens[3 * g] = log(__ddiv_rn(__dsub_rn(1.0, __dadd_rn(a0, a1)), lam1));
    dens[3 * g + 1] = log(a0);
    dens[3 * g + 2] = log(a1);
    if (a0 >= threshold || a1 >= threshold) { lo = lo < t ? lo : t; hi = t; }
  }
  if (hi >= 0) { atomicMin(&s_lo, lo); atomicMax(&s_hi, hi); }
  __syncthreads();
  int64_t first = 0, Tw = T;
  if (threshold > 0) {  // first .. last frame with an activation >= threshold; the numpy `.any()` quirk: none when only frame 0
    if (s_hi > 0) { first = s_lo; Tw = s_hi + 1 - s_lo; }
    else Tw = 0;
  }
  int any = 0;  // all-zero activations decode to nothing
  for (int64_t t = threadIdx.x; t < 2 * Tw && !any; t += blockDim.x) any = act[2 * (f0 + first) + t] != 0.0;
  any = __syncthreads_or(any);
  if (threadIdx.x == 0) {
    win[2 * clip] = first;
    win[2 * clip + 1] = any ? Tw : 0;
  }
}

__global__ void __launch_bounds__(1024)
dbn_viterbi_kernel(const DbnModelDev* __restrict__ models, int n_models, const double* __restrict__ dens,
                   const int64_t* __restrict__ fo, const int64_t* __restrict__ win, uint8_t* __restrict__ bp,
                   double* __restrict__ res_logp, int64_t* __restrict__ res_state) {
  extern __shared__ __align__(16) double smem[];
  __shared__ double s_v[32];
  __shared__ long long s_s[32];
  const int clip = blockIdx.x, mi = blockIdx.y, tid = threadIdx.x;
  const int64_t w0 = win[2 * clip], T = win[2 * clip + 1];
  if (T <= 0) return;
  const DbnModelDev m = models[mi];
  const int beats = m.beats, n_int = m.n_int, per_beat = m.per_beat, S = beats * per_beat, bn = beats * n_int;
  double* ring = smem;              // [S] ring value of every state: true log-probability = ring + G
  double* lt = ring + S;            // [n_int][n_int] log_tempo
  double* from = lt + n_int * n_int;  // [beats][n_int] last position of the previous beat, per tempo
  for (int i = tid; i < S; i += blockDim.x) ring[i] = m.init;
  for (int i = tid; i < n_int * n_int; i += blockDim.x) lt[i] = m.log_tempo[i];
  const bool active = tid < bn;
  int b = 0, k = 0, L = 1, base = 0, prev = 0, nrun = 1;
  if (active) {
    b = tid / n_int;
    k = tid - b * n_int;
    L = m.intervals[k];
    base = b * per_beat + m.first[k];
    prev = (b == 0 ? beats - 1 : b - 1) * per_beat + m.first[k];
    nrun = m.nrun[tid];
  }
  const double* d = dens + 3 * (fo[clip] + w0);
  const int dcol = b == 0 ? 2 : 1;
  uint8_t* bk = bp + m.bp_base + fo[clip] * bn + tid;
  const double* fr = from + b * n_int;
  const double* ltk = lt + k;
  int head = 0;  // ring slot of position 0 of this thread's tempo: (-t) mod L
  double G = 0.0;  // sum of the "no beat" densities d0 so far, shared by every state
  double d0 = d[0], d1 = d[dcol];
  __syncthreads();
  for (int64_t t = 0; t < T; ++t) {
    double n0 = 0.0, n1 = 0.0;
    if (t + 1 < T) { n0 = d[3 * (t + 1)]; n1 = d[3 * (t + 1) + dcol]; }
    if (active) {  // last position of beat b-1 at tempo k, before anything is overwritten
      int slot = head + L - 1;
      if (slot >= L) slot -= L;
      from[tid] = ring[prev + slot];
    }
    __syncthreads();
    if (active) {
      // best previous tempo: the first f that attains the maximum (strict >)
      double best = -CUDART_INF;
      int arg = 0;
      for (int f = 0; f < n_int; ++f) {
        const double c = __dadd_rn(fr[f], ltk[f * n_int]);
        if (c > best) { best = c; arg = f; }
      }
      bk[t * bn] = static_cast<uint8_t>(arg);
      head = head == 0 ? L - 1 : head - 1;
      const double rel = __dsub_rn(d1, d0);  // (down)beat density relative to the offset's d0
      double* tr = ring + base;
      int slot = head;
      tr[slot] = __dadd_rn(best, rel);
      for (int p = 1; p < nrun; ++p) {
        if (++slot == L) slot = 0;
        tr[slot] = __dadd_rn(tr[slot], rel);
      }
      G = __dadd_rn(G, d0);
    }
    __syncthreads();
    d0 = n0;
    d1 = n1;
  }
  // best final state, the lowest state index among equal values
  double vb = -CUDART_INF;
  long long sb = LLONG_MAX;
  if (active) {
    const double* tr = ring + base;
    for (int p = 0; p < L; ++p) {
      int slot = head + p;
      if (slot >= L) slot -= L;
      const double v = tr[slot];
      if (p == 0 || v > vb) { vb = v; sb = base + p; }
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_down_sync(0xffffffffu, vb, o);
    const long long os = __shfl_down_sync(0xffffffffu, sb, o);
    if (ov > vb || (ov == vb && os < sb)) { vb = ov; sb = os; }
  }
  if ((tid & 31) == 0) { s_v[tid >> 5] = vb; s_s[tid >> 5] = sb; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w)
      if (s_v[w] > vb || (s_v[w] == vb && s_s[w] < sb)) { vb = s_v[w]; sb = s_s[w]; }
    res_logp[clip * n_models + mi] = __dadd_rn(vb, G);
    res_state[clip * n_models + mi] = sb;
  }
}

__global__ void __launch_bounds__(32)
dbn_backtrace_kernel(const DbnModelDev* __restrict__ models, int n_models, const int64_t* __restrict__ fo,
                     const int64_t* __restrict__ win, const uint8_t* __restrict__ bp, const double* __restrict__ res_logp,
                     const int64_t* __restrict__ res_state, const double* __restrict__ act, uint8_t* __restrict__ codes,
                     int correct, double fps, double* __restrict__ times, int32_t* __restrict__ numbers,
                     int64_t* __restrict__ counts, int64_t* __restrict__ path_out, double* __restrict__ logp_out) {
  if (threadIdx.x != 0) return;
  const int clip = blockIdx.x;
  const int64_t f0 = fo[clip], w0 = win[2 * clip], T = win[2 * clip + 1];
  if (T <= 0) {
    if (counts) counts[clip] = 0;
    return;
  }
  // the more probable bar model; on equal log-probabilities the first (Tracker::track)
  int best = 0;
  double bl = res_logp[clip * n_models];
  for (int i = 1; i < n_models; ++i)
    if (res_logp[clip * n_models + i] > bl) { bl = res_logp[clip * n_models + i]; best = i; }
  const DbnModelDev& m = models[best];
  const int beats = m.beats, n_int = m.n_int, per_beat = m.per_beat, bn = beats * n_int;
  const int64_t s = res_state[clip * n_models + best];
  int b = static_cast<int>(s / per_beat);
  const int r = static_cast<int>(s - static_cast<int64_t>(b) * per_beat);
  int k = 0;
  while (k + 1 < n_int && m.first[k + 1] <= r) ++k;
  int p = r - m.first[k];
  const uint8_t* bk = bp + m.bp_base + f0 * bn;
  uint8_t* cd = codes ? codes + f0 : nullptr;
  for (int64_t t = T - 1; t >= 0; --t) {
    if (path_out) path_out[t] = static_cast<int64_t>(b) * per_beat + m.first[k] + p;
    else cd[t] = static_cast<uint8_t>((b + 1) | (p < m.nrun[b * n_int + k] ? kCodeInBeat : 0));
    if (p == 0) {  // first position of a beat: the stored best previous tempo, last position of the previous beat
      const int f = bk[t * bn + b * n_int + k];
      b = b == 0 ? beats - 1 : b - 1;
      k = f;
      p = m.intervals[f] - 1;
    } else {
      --p;
    }
  }
  if (path_out) {
    *logp_out = bl;
    return;
  }
  const double* a = act + 2 * (f0 + w0);
  double* tm = times + f0;
  int32_t* nm = numbers + f0;
  int64_t n = 0;
  if (correct) {  // every beat region moves to the first argmax of its flattened [frames, 2] activations
    int64_t t = 0;
    while (t < T) {
      if (cd[t] & kCodeInBeat) {
        const int64_t left = t;
        while (t < T && (cd[t] & kCodeInBeat)) ++t;
        int64_t arg = 0;
        for (int64_t i = 1; i < 2 * (t - left); ++i)
          if (a[2 * left + i] > a[2 * left + arg]) arg = i;
        const int64_t peak = arg / 2 + left;
        tm[n] = __ddiv_rn(static_cast<double>(peak + w0), fps);
        nm[n++] = cd[peak] & ~kCodeInBeat;
      } else {
        ++t;
      }
    }
  } else {  // the frames where the beat number changes
    for (int64_t t = 1; t < T; ++t)
      if ((cd[t] & ~kCodeInBeat) != (cd[t - 1] & ~kCodeInBeat)) {
        tm[n] = __ddiv_rn(static_cast<double>(t + w0), fps);
        nm[n++] = cd[t] & ~kCodeInBeat;
      }
  }
  counts[clip] = n;
}

}  // namespace

size_t dbn_viterbi_smem(int beats, int n_int, int per_beat) {
  return sizeof(double) * (static_cast<size_t>(beats) * per_beat + static_cast<size_t>(n_int) * n_int +
                           static_cast<size_t>(beats) * n_int);
}

void launch_dbn_prep(const float* beat, const float* down, const double* act_in, const int64_t* fo_dev, int n_clips,
                     double threshold, double observation_lambda, double* act, double* dens, int64_t* win,
                     cudaStream_t st) {
  if (n_clips <= 0) return;
  dbn_prep_kernel<<<n_clips, 256, 0, st>>>(beat, down, act_in, fo_dev, threshold, observation_lambda, act, dens, win);
}

cudaError_t launch_dbn_viterbi(const DbnModelDev* models_dev, int n_models, int threads, size_t smem, const double* dens,
                               const int64_t* fo_dev, const int64_t* win, int n_clips, uint8_t* bp, double* res_logp,
                               int64_t* res_state, cudaStream_t st) {
  if (n_clips <= 0) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(dbn_viterbi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  dbn_viterbi_kernel<<<dim3(n_clips, n_models), threads, smem, st>>>(models_dev, n_models, dens, fo_dev, win, bp, res_logp,
                                                                      res_state);
  return cudaSuccess;
}

void launch_dbn_backtrace(const DbnModelDev* models_dev, int n_models, const int64_t* fo_dev, const int64_t* win,
                          int n_clips, const uint8_t* bp, const double* res_logp, const int64_t* res_state,
                          const double* act, uint8_t* codes, int correct, double fps, double* times, int32_t* numbers,
                          int64_t* counts, int64_t* path_out, double* logp_out, cudaStream_t st) {
  if (n_clips <= 0) return;
  dbn_backtrace_kernel<<<n_clips, 32, 0, st>>>(models_dev, n_models, fo_dev, win, bp, res_logp, res_state, act, codes,
                                               correct, fps, times, numbers, counts, path_out, logp_out);
}

}  // namespace bt
