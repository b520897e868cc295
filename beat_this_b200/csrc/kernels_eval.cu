// Beat-tracking evaluation (mir_eval.beat at its defaults: F-measure, Cemgil, continuity), the metric step of the
// reference's evaluation (model/pl_module.py:320-339), for many event sets in one launch.  The contract is written out
// in include/beatthis.h (bt_beat_metrics) and DESIGN.md section 9; tests/beat_metrics_reference.py restates it in numpy.
//
// One warp per set, everything in float64 with explicit _rn intrinsics where an add could be contracted into an FMA.
// No per-set array lives in shared memory: the five metrical variations of the reference are read through an index
// map (Variation), nearest neighbours come from binary searches, and the continuity rule "each reference beat is used
// once" is a segmented scan over tiles of 32 estimates.
#include <cuda_runtime.h>

#include <cstdint>

#include "bt_kernels.h"

namespace bt {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kWarpsPerBlock = 4;

// Variation v of the trimmed reference r[0, n): 0 original, 1 off-beat (midpoints), 2 double tempo
// (np.interp at half-integer indices: r0, m01, r1, ..., r_{n-1}), 3 half tempo r[0::2], 4 half tempo r[1::2].
// Every variation is sorted when r is: r[i] <= mid(i) <= r[i+1] in float64.
struct Variation {
  const double* r;
  int64_t n;
  int kind;

  __device__ __forceinline__ double mid(int64_t i) const {
    return __dadd_rn(r[i], __dmul_rn(0.5, __dsub_rn(r[i + 1], r[i])));
  }
  __device__ __forceinline__ int64_t size() const {
    switch (kind) {
      case 0: return n;
      case 1: return n > 0 ? n - 1 : 0;
      case 2: return n > 0 ? 2 * n - 1 : 0;
      case 3: return (n + 1) / 2;
      default: return n / 2;
    }
  }
  __device__ __forceinline__ double operator[](int64_t k) const {
    switch (kind) {
      case 0: return r[k];
      case 1: return mid(k);
      case 2: return (k & 1) ? mid(k >> 1) : r[k >> 1];
      case 3: return r[2 * k];
      default: return r[2 * k + 1];
    }
  }
};

struct Plain {
  const double* a;
  __device__ __forceinline__ double operator[](int64_t k) const { return a[k]; }
};

// first k in [0, n) with a[k] >= x (n if none)
template <class A>
__device__ __forceinline__ int64_t lower_bound(const A& a, int64_t n, double x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t m = (lo + hi) >> 1;
    if (a[m] < x) lo = m + 1;
    else hi = m;
  }
  return lo;
}

// np.argmin(np.abs(e - v)) over the n > 0 sorted values of v: the lowest index at the minimal rounded distance, and
// that distance.  Left of the insertion point the rounded distance does not increase with the index, so the lowest
// index at the minimum is the first one whose distance is <= it.
template <class A>
__device__ __forceinline__ int64_t nearest(const A& v, int64_t n, double e, double* dist) {
  const int64_t j = lower_bound(v, n, e);
  const double dr = j < n ? fabs(__dsub_rn(e, v[j])) : 0.0;
  if (j > 0) {
    const double dl = fabs(__dsub_rn(e, v[j - 1]));
    if (j == n || dl <= dr) {
      int64_t lo = 0, hi = j - 1;
      while (lo < hi) {
        const int64_t m = (lo + hi) >> 1;
        if (fabs(__dsub_rn(e, v[m])) <= dl) hi = m;
        else lo = m + 1;
      }
      *dist = dl;
      return lo;
    }
  }
  *dist = dr;
  return j;
}

__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = __dadd_rn(x, __shfl_xor_sync(kFull, x, o));
  return x;
}

// Greedy maximum matching of hits (est - w <= ref <= est + w), refs in order, each taking the earliest unmatched
// estimate whose window holds it.  Both window ends are non-decreasing in the estimate, so the estimates skipped for
// one ref cannot hold a later one and greedy is maximum.
__device__ __forceinline__ int64_t count_matches(const double* r, int64_t nr, const double* e, int64_t ne, double w) {
  int64_t j = 0, hits = 0;
  for (int64_t i = 0; i < nr && j < ne; ++i) {
    const double x = r[i];
    while (j < ne && __dadd_rn(e[j], w) < x) ++j;
    if (j < ne && __dsub_rn(e[j], w) <= x) {
      ++hits;
      ++j;
    }
  }
  return hits;
}

// Cemgil accuracy of one variation: sum over its beats of exp(-d^2 / (2 sigma^2)), d = distance to the nearest
// estimate, over 0.5 * (n_est + n_variation).  0 for an empty variation.
__device__ __forceinline__ double cemgil(const Variation& v, const double* e, int64_t ne, double two_sigma_sq, int lane) {
  const int64_t nv = v.size();
  double acc = 0.0;
  for (int64_t k = lane; k < nv; k += 32) {
    const double x = v[k];
    const int64_t j = lower_bound(Plain{e}, ne, x);
    double d = j < ne ? fabs(__dsub_rn(x, e[j])) : INFINITY;
    if (j > 0) d = fmin(d, fabs(__dsub_rn(x, e[j - 1])));
    acc = __dadd_rn(acc, exp(__ddiv_rn(-__dmul_rn(d, d), two_sigma_sq)));
  }
  acc = warp_sum(acc);
  return nv > 0 ? __ddiv_rn(acc, __dmul_rn(0.5, static_cast<double>(ne + nv))) : 0.0;
}

// Continuity of one variation: (longest run of successful estimates, successes) over max(n_variation, n_est).
// Estimate m is a candidate when its phase |d / ref_int| and period |1 - est_int / ref_int| errors are both below the
// thresholds (intervals forward when m == 0 or its nearest ref is the first, backward otherwise; Python's x[-1] makes
// both 0 for a one-element array, and a zero ref interval fails).  A candidate succeeds when no earlier estimate with
// the same nearest ref was one; nearest is non-decreasing in m, so that is the most recent candidate overall.
__device__ __forceinline__ void continuity(const Variation& v, const double* e, int64_t ne, double phase_thr, double period_thr,
                           int lane, double* c_out, double* t_out) {
  const int64_t nv = v.size();
  if (nv == 0) {
    *c_out = *t_out = 0.0;
    return;
  }
  int64_t carry = -1;  // nearest ref of the most recent candidate
  int64_t total = 0, best = 0, cur = 0;
  for (int64_t base = 0; base < ne; base += 32) {
    const int64_t m = base + lane;
    const bool valid = m < ne;
    const double em = valid ? e[m] : e[ne - 1];
    double d;
    const int64_t k = nearest(v, nv, em, &d);
    bool cand = false;
    if (valid) {
      double ref_int, est_int;
      if (m == 0 || k == 0) {
        ref_int = __dsub_rn(k + 1 < nv ? v[k + 1] : v[k], k + 1 < nv ? v[k] : v[k > 0 ? k - 1 : nv - 1]);
        est_int = __dsub_rn(m + 1 < ne ? e[m + 1] : em, m + 1 < ne ? em : e[m > 0 ? m - 1 : ne - 1]);
      } else {
        ref_int = __dsub_rn(v[k], v[k - 1]);
        est_int = __dsub_rn(em, e[m - 1]);
      }
      if (ref_int != 0.0) {
        const double phase = fabs(__ddiv_rn(d, ref_int));
        const double period = fabs(__dsub_rn(1.0, __ddiv_rn(est_int, ref_int)));
        cand = phase < phase_thr && period < period_thr;
      }
    }
    const unsigned cm = __ballot_sync(kFull, cand);
    const unsigned below = cm & ((1u << lane) - 1u);
    const int64_t kprev = __shfl_sync(kFull, static_cast<long long>(k), below ? 31 - __clz(below) : lane);
    const bool succ = cand && (below ? kprev : carry) != k;
    const unsigned sm = __ballot_sync(kFull, succ);
    if (cm) carry = __shfl_sync(kFull, static_cast<long long>(k), 31 - __clz(cm));
    total += __popc(sm);
    if (sm == kFull) {
      cur += 32;
    } else {
      best = max(best, cur + (__ffs(~sm) - 1));  // the run continuing from the previous tile
      int inner = 0;
      for (unsigned x = sm; x; x &= x >> 1) ++inner;  // longest run of ones inside the tile
      best = max(best, static_cast<int64_t>(inner));
      cur = __clz(~sm);  // the run reaching the end of the tile
    }
  }
  best = max(best, cur);
  const double L = static_cast<double>(max(nv, ne));
  *c_out = __ddiv_rn(static_cast<double>(best), L);
  *t_out = __ddiv_rn(static_cast<double>(total), L);
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
beat_metrics_kernel(const double* __restrict__ est, const int64_t* __restrict__ est_off, const double* __restrict__ ref,
                    const int64_t* __restrict__ ref_off, int n_sets, BeatMetricParams p, double* __restrict__ out) {
  const int set = blockIdx.x * kWarpsPerBlock + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (set >= n_sets) return;  // warp-uniform
  const double* e = est + est_off[set];
  int64_t ne = est_off[set + 1] - est_off[set];
  const double* r = ref + ref_off[set];
  int64_t nr = ref_off[set + 1] - ref_off[set];
  // mir_eval.beat.trim_beats: keep times >= min_beat_time
  const int64_t te = lower_bound(Plain{e}, ne, p.min_beat_time), tr = lower_bound(Plain{r}, nr, p.min_beat_time);
  e += te;
  ne -= te;
  r += tr;
  nr -= tr;
  // Results go to memory as soon as they are known: a value held in a register across the double division's slow-path
  // call would be spilled.  The per-variation results of the warp's set wait in shared memory.
  __shared__ double s_res[kWarpsPerBlock][5][3];
  double(*res)[3] = s_res[threadIdx.x / 32];
  double* o = out + static_cast<int64_t>(set) * kBeatMetricCols;
  const bool scored = ne > 0 && nr > 0;
  long long hits = 0;
  if (scored && lane == 0) hits = count_matches(r, nr, e, ne, p.f_window);
  if (lane == 0) {
    const double matches = static_cast<double>(hits);
    const double P = scored ? __ddiv_rn(matches, static_cast<double>(ne)) : 0.0;
    const double R = scored ? __ddiv_rn(matches, static_cast<double>(nr)) : 0.0;
    o[0] = static_cast<double>(nr);
    o[1] = static_cast<double>(ne);
    o[2] = matches;
    o[3] = P;
    o[4] = R;
    o[5] = (P == 0.0 && R == 0.0) ? 0.0 : __ddiv_rn(__dmul_rn(__dmul_rn(2.0, P), R), __dadd_rn(P, R));
  }
  if (!scored) {
    if (lane < kBeatMetricCols - 6) o[6 + lane] = 0.0;
    return;
  }
  const double two_sigma_sq = __dmul_rn(2.0, __dmul_rn(p.cemgil_sigma, p.cemgil_sigma));
#pragma unroll 1
  for (int kind = 0; kind < 5; ++kind) {
    const Variation v{r, nr, kind};
    const double cem = cemgil(v, e, ne, two_sigma_sq, lane);
    double c, t;
    continuity(v, e, ne, p.phase_threshold, p.period_threshold, lane, &c, &t);
    if (lane == 0) {
      res[kind][0] = cem;
      res[kind][1] = c;
      res[kind][2] = t;
    }
  }
  __syncwarp();
  if (lane < 3) {  // lane 0: cemgil, 1: CMLc / AMLc, 2: CMLt / AMLt (the same warp wrote res)
    double mx = res[0][lane];
    for (int kind = 1; kind < 5; ++kind) mx = fmax(mx, res[kind][lane]);
    const int first = lane == 0 ? 6 : 7 + lane;  // cemgil -> 6, CMLc -> 8, CMLt -> 9
    o[first] = res[0][lane];
    o[lane == 0 ? 7 : 9 + lane] = mx;  // cemgil_max -> 7, AMLc -> 10, AMLt -> 11
  }
}

}  // namespace

void launch_beat_metrics(const double* est, const int64_t* est_off_dev, const double* ref, const int64_t* ref_off_dev,
                         int n_sets, const BeatMetricParams& p, double* out, cudaStream_t st) {
  const int blocks = static_cast<int>((static_cast<int64_t>(n_sets) + kWarpsPerBlock - 1) / kWarpsPerBlock);
  beat_metrics_kernel<<<blocks, kWarpsPerBlock * 32, 0, st>>>(est, est_off_dev, ref, ref_off_dev, n_sets, p, out);
}

}  // namespace bt
