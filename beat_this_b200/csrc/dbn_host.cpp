// Host DBN post-processor: bar-pointer HMM + Viterbi, the stand-in for madmom's DBNDownBeatTrackingProcessor
// (Cython in madmom) that the reference configures in model/postprocessor.py:29-37 and calls per piece in
// postprocessor.py:138-173.  Restated from the published algorithm (see beat_this_b200/dbn.py, which holds the
// numpy twin of everything here); parity with madmom is unpinned.  Plain C++ threads, no CUDA.
//
// The state space is never materialised as a transition matrix: inside a beat a state can only be reached from
// the previous position of the same tempo, and the first position of a beat from the LAST position of every
// tempo of the previous beat (n_int x n_int log-probabilities).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <limits>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#if defined(__x86_64__) && defined(__GNUC__)
#include <immintrin.h>
#endif

#include "../../include/beatthis.h"
#include "dbn_model.h"

namespace {

// The inner loop of the Viterbi recursion, compiled for AVX2 / AVX-512 where the host has them (plain adds,
// compares and blends: results are identical to the scalar build).
#if defined(__x86_64__) && defined(__GNUC__)
#define BT_SIMD_CLONES __attribute__((target_clones("avx512f", "avx2", "default")))
#else
#define BT_SIMD_CLONES
#endif

// best[k] = max_f from[f] + log_tempo[f][k], arg[k] = the FIRST f that attains it (f ascending, strict >)
// [klo[f], khi[f]) = the k with a finite log_tempo[f][k] (the exponential tempo model leaves a band around f).
// The argmax is tracked as a double so that every array in the loop has 8-byte lanes (the compiler vectorises it).
BT_SIMD_CLONES void tempo_step_generic(const double* __restrict from, const double* __restrict log_tempo, int n_int,
                                       const int32_t* __restrict klo, const int32_t* __restrict khi, double* __restrict best,
                                       double* __restrict argd) {
  for (int k = 0; k < n_int; ++k) { best[k] = -std::numeric_limits<double>::infinity(); argd[k] = 0.0; }
  for (int f = 0; f < n_int; ++f) {
    const double ff = from[f], fd = static_cast<double>(f);
    const double* __restrict lt = log_tempo + static_cast<size_t>(f) * n_int;
    const int lo = klo[f], hi = khi[f];
    for (int k = lo; k < hi; ++k) {
      const double c = ff + lt[k];
      const double b = best[k];
      argd[k] = c > b ? fd : argd[k];
      best[k] = c > b ? c : b;
    }
  }
}

#if defined(__x86_64__) && defined(__GNUC__)
// The same recursion with best[] / arg[] held in NV zmm registers for the whole sweep over f (the generic form keeps
// them in memory: 42 dependent load-compare-store rounds over short, masked loops -- 0.9 us per call on a 2.1 GHz
// Sapphire Rapids core, 80 % of the decoder's time).  Entries outside the band are -inf in log_tempo: c = -inf never
// passes the strict comparison, so sweeping whole rows gives the identical result (same adds, same compares, same order).
template <int NV>
__attribute__((target("avx512f"))) void tempo_step_avx512(const double* from, const double* log_tempo, int n_int, double* best,
                                                          double* argd) {
  __m512d b[NV], a[NV];
  __mmask8 msk[NV];
#pragma GCC unroll 8
  for (int v = 0; v < NV; ++v) {
    b[v] = _mm512_set1_pd(-std::numeric_limits<double>::infinity());
    a[v] = _mm512_setzero_pd();
    const int left = n_int - 8 * v;
    msk[v] = left >= 8 ? static_cast<__mmask8>(0xff) : static_cast<__mmask8>((1u << (left > 0 ? left : 0)) - 1u);
  }
  for (int f = 0; f < n_int; ++f) {
    const __m512d ff = _mm512_set1_pd(from[f]), fd = _mm512_set1_pd(static_cast<double>(f));
    const double* lt = log_tempo + static_cast<size_t>(f) * n_int;
#pragma GCC unroll 8
    for (int v = 0; v < NV; ++v) {
      const __m512d c = _mm512_add_pd(ff, _mm512_maskz_loadu_pd(msk[v], lt + 8 * v));
      const __mmask8 gt = _mm512_mask_cmp_pd_mask(msk[v], c, b[v], _CMP_GT_OQ);
      b[v] = _mm512_mask_blend_pd(gt, b[v], c);
      a[v] = _mm512_mask_blend_pd(gt, a[v], fd);
    }
  }
#pragma GCC unroll 8
  for (int v = 0; v < NV; ++v) {
    _mm512_mask_storeu_pd(best + 8 * v, msk[v], b[v]);
    _mm512_mask_storeu_pd(argd + 8 * v, msk[v], a[v]);
  }
}
#endif

inline void tempo_step(const double* from, const double* log_tempo, int n_int, const int32_t* klo, const int32_t* khi,
                       double* best, double* argd) {
#if defined(__x86_64__) && defined(__GNUC__)
  static const bool has512 = __builtin_cpu_supports("avx512f");
  if (has512 && n_int <= 64) {
    switch ((n_int + 7) / 8) {
      case 1: return tempo_step_avx512<1>(from, log_tempo, n_int, best, argd);
      case 2: return tempo_step_avx512<2>(from, log_tempo, n_int, best, argd);
      case 3: return tempo_step_avx512<3>(from, log_tempo, n_int, best, argd);
      case 4: return tempo_step_avx512<4>(from, log_tempo, n_int, best, argd);
      case 5: return tempo_step_avx512<5>(from, log_tempo, n_int, best, argd);
      case 6: return tempo_step_avx512<6>(from, log_tempo, n_int, best, argd);
      case 7: return tempo_step_avx512<7>(from, log_tempo, n_int, best, argd);
      default: return tempo_step_avx512<8>(from, log_tempo, n_int, best, argd);
    }
  }
#endif
  tempo_step_generic(from, log_tempo, n_int, klo, khi, best, argd);
}

// Per-worker buffers, kept between pieces and between calls (grow only): with one short-lived allocation per piece,
// 64 threads mmap / munmap megabytes concurrently and the kernel's address-space lock plus the TLB shootdowns
// serialise them (measured: 64 pieces on 128 CPUs took 5x the single-piece time).
struct Scratch {
  std::vector<double> v, nv, from, best, dens;
  std::vector<int16_t> back;
  std::vector<double> argd;
  std::vector<int32_t> nrun, klo, khi, head;
  std::vector<int64_t> first, last, path, best_path;
};

// follow the stored best-previous-tempo decisions back from the final state
void backtrace(int64_t T, int32_t beats, int32_t n_int, int64_t per_beat, const std::vector<int64_t>& first,
               const std::vector<int64_t>& last, const std::vector<int16_t>& back, int64_t state, int64_t* path_out) {
  for (int64_t t = T - 1; t >= 0; --t) {
    path_out[t] = state;
    const int64_t b = state / per_beat, r = state - b * per_beat;
    int k = 0;  // tempo slot of this state (n_int ~ 42: linear scan is fine)
    while (k + 1 < n_int && first[k + 1] <= r) ++k;
    if (r == first[k]) {
      const int f = back[(static_cast<size_t>(t) * beats + b) * n_int + k];
      state = ((b + beats - 1) % beats) * per_beat + last[f];
    } else {
      state -= 1;
    }
  }
}

int viterbi(const double* log_dens, int64_t T, int32_t beats, int32_t n_int, const int32_t* intervals,
            const double* log_tempo, const int32_t* pointers, int64_t* path_out, double* logp_out, Scratch& ws) {
  int64_t per_beat = 0;
  std::vector<int64_t>&first = ws.first, &last = ws.last;
  first.resize(n_int); last.resize(n_int);
  for (int k = 0; k < n_int; ++k) {
    if (intervals[k] <= 0) return BT_ERR_ARG;
    first[k] = per_beat;
    per_beat += intervals[k];
    last[k] = per_beat - 1;
  }
  const int64_t S = per_beat * beats;
  // inside one tempo of one beat the density pointer is a run of (down)beat states followed by non-beat states:
  // nrun[b][k] = length of the leading run that shares the pointer of the first state
  std::vector<int32_t>& nrun = ws.nrun;
  nrun.resize(static_cast<size_t>(beats) * n_int);
  bool runs_ok = true;
  for (int b = 0; b < beats && runs_ok; ++b)
    for (int k = 0; k < n_int && runs_ok; ++k) {
      const int64_t s0 = b * per_beat + first[k];
      int32_t n = 1;
      while (n < intervals[k] && pointers[s0 + n] == pointers[s0]) ++n;
      for (int32_t p = n; p < intervals[k]; ++p) runs_ok = runs_ok && pointers[s0 + p] == 0;
      nrun[static_cast<size_t>(b) * n_int + k] = n;
    }
  std::vector<int32_t>&klo = ws.klo, &khi = ws.khi;
  klo.resize(n_int); khi.resize(n_int);
  for (int f = 0; f < n_int; ++f) {
    int lo = 0, hi = n_int;
    while (lo < n_int && std::isinf(log_tempo[static_cast<size_t>(f) * n_int + lo])) ++lo;
    while (hi > lo && std::isinf(log_tempo[static_cast<size_t>(f) * n_int + hi - 1])) --hi;
    klo[f] = lo; khi[f] = hi;
  }
  std::vector<double>&v = ws.v, &nv = ws.nv, &from = ws.from, &best = ws.best;
  v.assign(S, -std::log(static_cast<double>(S)));
  std::vector<int16_t>& back = ws.back;
  back.resize(static_cast<size_t>(T) * beats * n_int);  // every entry is written before the backtrace reads it
  from.resize(static_cast<size_t>(beats) * n_int); best.resize(static_cast<size_t>(beats) * n_int);
  std::vector<double>& arg = ws.argd;
  arg.resize(n_int);
  if (runs_ok) {
    // Inside a tempo track every state just follows its predecessor, and all but the first few positions of a beat
    // observe the same "no beat" density d0: the track is kept as a RING (head[k] = slot of position 0; advancing one
    // frame = moving the head back by one) and d0 is summed into ONE offset G for the whole state space instead of
    // being added to 10 000 states per frame.  Per frame only the states that change RELATIVE to that offset are
    // touched: the new first position of every (beat, tempo) -- best previous tempo, the 42 x 42 step -- and the up to
    // three following positions that observe the (down)beat density db instead of d0 (they get db - d0).
    // True log-probability of a state = ring value + G.
    std::vector<int32_t>& head = ws.head;
    head.assign(n_int, 0);
    double G = 0.0;
    for (int64_t t = 0; t < T; ++t) {
      const double* d = log_dens + 3 * t;
      for (int b = 0; b < beats; ++b) {  // last positions of the previous beat, before anything is overwritten
        const int64_t prev_base = ((b + beats - 1) % beats) * per_beat;
        double* fr = &from[static_cast<size_t>(b) * n_int];
        for (int k = 0; k < n_int; ++k) {
          const int32_t L = intervals[k];
          int32_t slot = head[k] + L - 1;
          if (slot >= L) slot -= L;
          fr[k] = v[prev_base + first[k] + slot];
        }
      }
      for (int b = 0; b < beats; ++b) {
        tempo_step(&from[static_cast<size_t>(b) * n_int], log_tempo, n_int, klo.data(), khi.data(), &best[static_cast<size_t>(b) * n_int], arg.data());
        int16_t* bk = &back[(static_cast<size_t>(t) * beats + b) * n_int];
        for (int k = 0; k < n_int; ++k) bk[k] = static_cast<int16_t>(arg[k]);
      }
      for (int k = 0; k < n_int; ++k) head[k] = head[k] == 0 ? intervals[k] - 1 : head[k] - 1;
      for (int b = 0; b < beats; ++b) {
        const int64_t base = b * per_beat;
        const double rel = d[b == 0 ? 2 : 1] - d[0];  // (down)beat density relative to the offset's d0
        const double* bs = &best[static_cast<size_t>(b) * n_int];
        for (int k = 0; k < n_int; ++k) {
          const int32_t L = intervals[k];
          double* tr = &v[base + first[k]];
          int32_t slot = head[k];
          tr[slot] = bs[k] + rel;
          const int32_t n = nrun[static_cast<size_t>(b) * n_int + k];
          for (int32_t p = 1; p < n; ++p) {
            if (++slot == L) slot = 0;
            tr[slot] += rel;
          }
        }
      }
      G += d[0];
    }
    // best final state, lowest state index among equals (as the dense form below)
    int64_t state = -1;
    double vbest = -std::numeric_limits<double>::infinity();
    for (int b = 0; b < beats; ++b)
      for (int k = 0; k < n_int; ++k) {
        const int32_t L = intervals[k];
        const double* tr = &v[b * per_beat + first[k]];
        for (int32_t p = 0; p < L; ++p) {
          int32_t slot = head[k] + p;
          if (slot >= L) slot -= L;
          if (tr[slot] > vbest || state < 0) { vbest = tr[slot]; state = b * per_beat + first[k] + p; }
        }
      }
    *logp_out = vbest + G;
    backtrace(T, beats, n_int, per_beat, first, last, back, state, path_out);
    return BT_OK;
  }
  nv.resize(S);
  for (int64_t t = 0; t < T; ++t) {
    const double* d = log_dens + 3 * t;
    for (int b = 0; b < beats; ++b) {
      const int64_t base = b * per_beat, prev_base = ((b + beats - 1) % beats) * per_beat;
      for (int k = 0; k < n_int; ++k) from[k] = v[prev_base + last[k]];
      tempo_step(from.data(), log_tempo, n_int, klo.data(), khi.data(), best.data(), arg.data());  // first position of every tempo: best previous tempo
      int16_t* bk = &back[(static_cast<size_t>(t) * beats + b) * n_int];
      for (int k = 0; k < n_int; ++k) {
        bk[k] = static_cast<int16_t>(arg[k]);
        const int64_t s0 = base + first[k];
        nv[s0] = best[k] + d[pointers[s0]];
        for (int64_t p = 1; p < intervals[k]; ++p) nv[s0 + p] = v[s0 + p - 1] + d[pointers[s0 + p]];
      }
    }
    v.swap(nv);
  }
  int64_t state = 0;
  for (int64_t s = 1; s < S; ++s)
    if (v[s] > v[state]) state = s;
  *logp_out = v[state];
  backtrace(T, beats, n_int, per_beat, first, last, back, state, path_out);
  return BT_OK;
}

using bt::BarModel;

struct Tracker {
  std::vector<BarModel> models;
  double fps = 50.0, threshold = 0.05, observation_lambda = 16.0;
  bool correct = true;

  // beat_this_b200/dbn.py::DBNDownBeatTracker.__call__; returns the number of beats written
  int64_t track(const double* act_in, int64_t T_in, double* times, int32_t* numbers, Scratch& ws) const {
    int64_t first = 0, T = T_in;
    const double* act = act_in;
    if (threshold > 0) {  // decode between the first and the last frame with an activation above the threshold
      int64_t lo = -1, hi = -1;
      for (int64_t t = 0; t < T_in; ++t)
        if (act_in[2 * t] >= threshold || act_in[2 * t + 1] >= threshold) { if (lo < 0) lo = t; hi = t; }
      // np.nonzero(...)[0].any(): false when nothing passes, and (numpy quirk kept) when only frame 0 does
      if (hi > 0) { first = lo; act = act_in + 2 * lo; T = hi + 1 - lo; }
      else T = 0;
    }
    bool any = false;
    for (int64_t t = 0; t < 2 * T && !any; ++t) any = act[t] != 0.0;
    if (!any) return 0;
    std::vector<double>& dens = ws.dens;
    dens.resize(3 * T);
    for (int64_t t = 0; t < T; ++t) {
      dens[3 * t] = std::log((1.0 - (act[2 * t] + act[2 * t + 1])) / (observation_lambda - 1.0));
      dens[3 * t + 1] = std::log(act[2 * t]);
      dens[3 * t + 2] = std::log(act[2 * t + 1]);
    }
    std::vector<int64_t>&best_path = ws.best_path, &path = ws.path;
    path.resize(T);
    double best_logp = -std::numeric_limits<double>::infinity();
    const BarModel* best = nullptr;
    for (const BarModel& m : models) {
      double logp = 0;
      viterbi(dens.data(), T, m.beats, m.n_int, m.intervals.data(), m.log_tempo.data(), m.pointers.data(), path.data(), &logp, ws);
      if (best == nullptr || logp > best_logp) { best_logp = logp; best = &m; best_path.assign(path.begin(), path.end()); }
    }
    int64_t n = 0;
    auto number_of = [&](int64_t t) { return static_cast<int32_t>(best_path[t] / best->per_beat) + 1; };
    if (correct) {  // every beat moves to the strongest activation inside its beat region
      int64_t t = 0;
      while (t < T) {
        if (best->pointers[best_path[t]] >= 1) {
          const int64_t left = t;
          while (t < T && best->pointers[best_path[t]] >= 1) ++t;
          int64_t arg = 0;  // np.argmax over the flattened [frames, 2] block
          for (int64_t i = 1; i < 2 * (t - left); ++i)
            if (act[2 * left + i] > act[2 * left + arg]) arg = i;
          const int64_t peak = arg / 2 + left;
          times[n] = static_cast<double>(peak + first) / fps;
          numbers[n++] = number_of(peak);
        } else {
          ++t;
        }
      }
    } else {
      for (int64_t t = 1; t < T; ++t)
        if (number_of(t) != number_of(t - 1)) { times[n] = static_cast<double>(t + first) / fps; numbers[n++] = number_of(t); }
    }
    return n;
  }
};

}  // namespace

extern "C" int bt_dbn_viterbi(const double* log_dens, int64_t T, int32_t beats, int32_t n_int, const int32_t* intervals,
                              const double* log_tempo, const int32_t* pointers, int64_t* path_out, double* logp_out) {
  if (!log_dens || !intervals || !log_tempo || !pointers || !path_out || !logp_out || T <= 0 || beats <= 0 || n_int <= 0)
    return BT_ERR_ARG;
  Scratch ws;
  return viterbi(log_dens, T, beats, n_int, intervals, log_tempo, pointers, path_out, logp_out, ws);
}

extern "C" int bt_dbn_track(const double* activations, const int64_t* frame_offsets, int32_t n_clips,
                            const int32_t* beats_per_bar, int32_t n_bar_lengths, double min_bpm, double max_bpm,
                            int32_t num_tempi, double transition_lambda, double observation_lambda, double threshold,
                            int32_t correct, double fps, int32_t n_threads, double* times_out, int32_t* numbers_out,
                            int64_t* counts_out) {
  if (!activations || !frame_offsets || !beats_per_bar || !times_out || !numbers_out || !counts_out || n_clips < 0 ||
      n_bar_lengths <= 0 || min_bpm <= 0 || max_bpm <= min_bpm || fps <= 0 || observation_lambda <= 1)
    return BT_ERR_ARG;
  Tracker trk;
  trk.fps = fps; trk.threshold = threshold; trk.observation_lambda = observation_lambda; trk.correct = correct != 0;
  trk.models.resize(n_bar_lengths);
  for (int i = 0; i < n_bar_lengths; ++i) {
    if (beats_per_bar[i] <= 0) return BT_ERR_ARG;
    trk.models[i].build(beats_per_bar[i], 60.0 * fps / max_bpm, 60.0 * fps / min_bpm, num_tempi, transition_lambda, observation_lambda);
  }
  int nt = n_threads > 0 ? n_threads : static_cast<int>(std::thread::hardware_concurrency());
  nt = std::max(1, std::min(nt, static_cast<int>(n_clips)));
  // borrow nt scratch sets from the process-wide pool (returned below; concurrent calls get their own)
  static std::mutex pool_mutex;
  static std::vector<std::unique_ptr<Scratch>> pool_free;
  std::vector<std::unique_ptr<Scratch>> mine;
  {
    std::lock_guard<std::mutex> lk(pool_mutex);
    while (static_cast<int>(mine.size()) < nt && !pool_free.empty()) { mine.push_back(std::move(pool_free.back())); pool_free.pop_back(); }
  }
  while (static_cast<int>(mine.size()) < nt) mine.emplace_back(new Scratch());
  std::atomic<int32_t> next{0};
  auto work = [&](int w) {
    Scratch& ws = *mine[w];
    for (int32_t i = next.fetch_add(1); i < n_clips; i = next.fetch_add(1)) {
      const int64_t f0 = frame_offsets[i], T = frame_offsets[i + 1] - f0;
      counts_out[i] = T > 0 ? trk.track(activations + 2 * f0, T, times_out + f0, numbers_out + f0, ws) : 0;
    }
  };
  std::vector<std::thread> pool;
  for (int i = 1; i < nt; ++i) pool.emplace_back(work, i);
  work(0);
  for (auto& th : pool) th.join();
  {
    std::lock_guard<std::mutex> lk(pool_mutex);
    for (auto& m : mine) pool_free.push_back(std::move(m));
  }
  return BT_OK;
}
