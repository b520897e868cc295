"""Float64 numpy restatement of the beat-metric contract of bt_beat_metrics (include/beatthis.h, DESIGN.md section 9):
mir_eval.beat's F-measure, Cemgil and continuity at their defaults, after trim_beats.  The device kernel is compared
with it bitwise (Cemgil within 1e-12: CUDA's double exp and the summation order differ); tests/test_cpu_eval.py ties it
to literal per-beat loops, to scipy's maximum bipartite matching and, where it is installed, to mir_eval itself."""
from __future__ import annotations

import numpy as np

FIELDS = ("n_ref", "n_est", "matches", "P", "R", "F", "cemgil", "cemgil_max", "CMLc", "CMLt", "AMLc", "AMLt")
DEFAULTS = dict(min_beat_time=5.0, f_window=0.07, cemgil_sigma=0.04, phase_threshold=0.175, period_threshold=0.175)


def variations(r: np.ndarray) -> list[np.ndarray]:
    """Original, off-beat, double tempo (np.interp at half-integer indices), half tempo odd and even."""
    mid = r[:-1] + 0.5 * (r[1:] - r[:-1])
    double = np.empty(max(2 * len(r) - 1, 0))
    double[0::2] = r
    double[1::2] = mid
    return [r, mid, double, r[0::2], r[1::2]]


def match_count(ref: np.ndarray, est: np.ndarray, window: float) -> int:
    """Size of a maximum matching of hits est - w <= ref <= est + w (greedy: each ref in order takes the earliest
    unmatched estimate whose window holds it)."""
    lo, hi = est - window, est + window
    j = hits = 0
    for x in ref.tolist():
        while j < len(est) and hi[j] < x:
            j += 1
        if j == len(est):
            break
        if lo[j] <= x:
            hits += 1
            j += 1
    return hits


def nearest(v: np.ndarray, e: np.ndarray):
    """np.argmin(np.abs(e_m - v)) for every e_m (v sorted, non-empty), and the minimal distances."""
    n = len(v)
    j = np.searchsorted(v, e, side="left")
    dr = np.where(j < n, np.abs(e - v[np.minimum(j, n - 1)]), np.inf)
    dl = np.where(j > 0, np.abs(e - v[np.maximum(j - 1, 0)]), np.inf)
    left = dl <= dr
    k = np.where(left, np.searchsorted(v, v[np.maximum(j - 1, 0)], side="left"), j)
    # distinct values at the same rounded distance: move to the lowest of them
    for i in np.flatnonzero(left & (k > 0)):
        while k[i] > 0 and abs(e[i] - v[k[i] - 1]) <= dl[i]:
            k[i] -= 1
    return k, np.where(left, dl, dr)


def cemgil(v: np.ndarray, e: np.ndarray, sigma: float) -> float:
    if len(v) == 0:
        return 0.0
    j = np.searchsorted(e, v, side="left")
    d = np.minimum(np.where(j < len(e), np.abs(v - e[np.minimum(j, len(e) - 1)]), np.inf),
                   np.where(j > 0, np.abs(v - e[np.maximum(j - 1, 0)]), np.inf))
    return float(np.sum(np.exp(-(d * d) / (2.0 * sigma**2)))) / (0.5 * (len(e) + len(v)))


def continuity(v: np.ndarray, e: np.ndarray, phase_thr: float, period_thr: float) -> tuple[float, float]:
    """(longest run of successes, successes) over max(len(v), len(e)) for one variation; 0 for an empty one."""
    nv, ne = len(v), len(e)
    if nv == 0:
        return 0.0, 0.0
    k, d = nearest(v, e)
    m = np.arange(ne)
    fwd = (m == 0) | (k == 0)
    # forward intervals, backward at the last element; index -1 wraps as in Python (one element: interval 0)
    kn, kp = np.where(k + 1 < nv, k + 1, k), np.where(k + 1 < nv, k, k - 1)
    mn, mp = np.where(m + 1 < ne, m + 1, m), np.where(m + 1 < ne, m, m - 1)
    ref_int = np.where(fwd, v[kn] - v[kp], v[k] - v[k - 1])
    est_int = np.where(fwd, e[mn] - e[mp], e[m] - e[m - 1])
    with np.errstate(divide="ignore", invalid="ignore"):
        phase = np.abs(d / ref_int)
        period = np.abs(1 - est_int / ref_int)
    cand = (ref_int != 0) & (phase < phase_thr) & (period < period_thr)
    ci = np.flatnonzero(cand)
    first = np.ones(len(ci), dtype=bool)
    first[1:] = k[ci[1:]] != k[ci[:-1]]  # each ref is used once: only the first candidate of a nearest ref succeeds
    succ = np.zeros(ne, dtype=np.int64)
    succ[ci[first]] = 1
    fails = np.flatnonzero(np.concatenate(([0], succ, [0])) == 0)
    L = float(max(nv, ne))
    return float(np.max(np.diff(fails)) - 1) / L, float(succ.sum()) / L


def set_metrics(est, ref, min_beat_time=5.0, f_window=0.07, cemgil_sigma=0.04, phase_threshold=0.175,
                period_threshold=0.175) -> np.ndarray:
    """One row of FIELDS for one (estimates, references) pair."""
    e = np.asarray(est, dtype=np.float64)
    r = np.asarray(ref, dtype=np.float64)
    e, r = e[e >= min_beat_time], r[r >= min_beat_time]
    row = np.zeros(len(FIELDS))
    row[0], row[1] = len(r), len(e)
    if len(e) == 0 or len(r) == 0:
        return row
    hits = match_count(r, e, f_window)
    P, R = hits / len(e), hits / len(r)
    row[2:6] = hits, P, R, 0.0 if P == 0 and R == 0 else 2.0 * P * R / (P + R)
    cem = [cemgil(v, e, cemgil_sigma) for v in variations(r)]
    cont = [continuity(v, e, phase_threshold, period_threshold) for v in variations(r)]
    row[6], row[7] = cem[0], max(cem)
    row[8], row[9] = cont[0]
    row[10], row[11] = max(c for c, _ in cont), max(t for _, t in cont)
    return row


def beat_metrics(estimates, references, **params) -> np.ndarray:
    """[n_sets, 12] float64, the layout of bt_beat_metrics."""
    out = np.zeros((len(estimates), len(FIELDS)))
    for i, (e, r) in enumerate(zip(estimates, references)):
        out[i] = set_metrics(e, r, **{**DEFAULTS, **params})
    return out


# ---- seeded test sets (tests/test_gpu_eval.py, tools/eval_rates.py) ---------------------------------------------------
def tracked_piece(rng, seconds: float):
    """(estimates, references) of one piece: a jittered reference at 60-200 BPM and an estimate with dropped and
    inserted beats that is now and then at double or half tempo or off-beat."""
    period = 60.0 / rng.uniform(60, 200)
    ref = np.arange(rng.uniform(0, period), seconds, period)
    ref = np.sort(np.clip(ref + rng.normal(0, 0.008, len(ref)), 0, None))
    kind = rng.choice(["same", "double", "half", "offbeat"], p=[0.7, 0.1, 0.1, 0.1])
    est = {"same": ref, "double": variations(ref)[2], "half": ref[::2], "offbeat": variations(ref)[1]}[kind]
    est = est[rng.random(len(est)) > rng.uniform(0, 0.1)]  # dropped beats
    est = est + rng.normal(0, rng.uniform(0.005, 0.04), len(est))
    est = np.concatenate([est, rng.uniform(0, seconds, rng.poisson(seconds / 30))])  # inserted beats
    return np.sort(np.clip(est, 0, None)), ref


def pieces(seed: int, n: int, min_s: float = 30.0, max_s: float = 600.0):
    """Beats and downbeats of n pieces of min_s..max_s seconds: 2n (estimates, references) sets, beats first."""
    rng = np.random.default_rng(seed)
    beats = [tracked_piece(rng, rng.uniform(min_s, max_s)) for _ in range(n)]
    downs = []
    for est, ref in beats:
        meter = rng.integers(3, 5)
        downs.append((est[rng.integers(0, meter) :: meter], ref[rng.integers(0, meter) :: meter]))
    return [e for e, _ in beats] + [e for e, _ in downs], [r for _, r in beats] + [r for _, r in downs]
