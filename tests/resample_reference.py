"""Float64 restatement of the polyphase resampler (resample_kernel through bt_resample / Engine.resample_cat) at chosen
output indices, the elementwise bound its unit tests hold it to, and the rates it serves.  Shared by
tests/test_gpu_resample.py (runs the kernel) and tests/test_cpu_resample_reference.py (holds a float32 emulation of
the kernel's operation order to the bound, and shows that indexing mistakes break it).

Restatement: the definition in beat_this_b200/preprocessing.py, evaluated by oracle.resample_direct_terms (the
arithmetic of oracle.resample_direct, at any output indices, so long clips can be checked by sampling):
  y[n] = sum_j x[j] s h(s (n M / L - j)),  h(t) = rho sinc(rho t) kaiser(t / Z) for |t| <= Z, 0 beyond
over the samples j = q - K/2 - 1 .. q + K/2 + 1 of the clip (zeros outside it), q = floor(n M / L), K = 2 ceil(Z / s).

The kernel: c = coef[(n M) mod L] (fp32), the K staged samples x[q - K/2 + 1 + k] (fp32, zeros outside the clip),
  a_i = fmaf chain over k = i, i + 4, ... (i = 0..3, floor(K/4) terms each); a_0 then takes the K mod 4 tail terms;
  y = (a_0 + a_1) + (a_2 + a_3).

Bound per output, with S = sum_j |w_j x_j| over the kernel's K taps (w_j: the float64 weights of the direct form) and
X = sum_j |x_j| over the direct form's K + 3 samples:
  coefficients  the bank holds fp32(w~_j), w~_j the float64 bank value: 2^-24 S.
  sum           a chain of m products from 0 rounds m times, so a_0 (floor(K/4) + K mod 4 <= ceil(K/4) + 1 terms) and
                the three others are each within gamma_m of the sum of their terms' magnitudes; the two final adds
                round twice more: gamma_{ceil(K/4) + 3} (1 + 2^-24) S with gamma_m = m 2^-24 / (1 - m 2^-24).
  truncation    the direct form's samples the kernel does not read (j = q - K/2 - 1, q - K/2, q + K/2 + 1) sit at
                |s t| >= Z; their weight is 0 except at |s t| = Z exactly (t = K/2 + (nM mod L)/L = Z/s), where h(Z),
                about 2e-8, remains: the exact sum of |w_j x_j| over those three samples.
  float64       the phase n M / L - j is an integer plus (n M mod L) / L, rounded once: 2^-52 (Z / s + 2) in input
                samples; s h' has slope at most 4 s per sample (H_SLOPE, checked by the CPU test), so each weight is
                off by at most 4 s^2 2^-52 (Z / s + 2) <= 2^-44, for the direct form and for the bank alike; h's own
                float64 evaluation (sinc, i0, sqrt) and the float64 sum of at most 52 000 terms stay below 2^-37 of
                S.  E64 = 2^-36 (S + X) covers both with room.
  |kernel - y| <= B + truncation,  B = (2^-24 + gamma_{ceil(K/4) + 3} (1 + 2^-24)) S + E64.
The tests report (|kernel - y| - truncation) / B.
"""
import functools
import inspect
import math

import numpy as np

from beat_this_b200 import augment as A
from beat_this_b200 import preprocessing as P
from numerics import U
from oracle import beat_this_oracle as O

E64 = 2.0**-36
H_SLOPE = 4.0  # max |d/dt h(t)|, t in output-band zero crossings (test_cpu_resample_reference checks it)
SR = P.SAMPLE_RATE
MAX_SMEM = 200 * 1024  # kResampleMaxSmem (bt_kernels.h): bt_resample refuses a staged input span above it
SMEM_OPT_IN = 48 * 1024  # above this the launch raises the kernel's dynamic shared memory limit first


def gamma(m: int) -> float:
    return m * U / (1 - m * U)


# ------------------------------------------------------------------------------------------------------------ rates
# inputs the inference front door resamples to 22.05 kHz (22050 itself runs the filter too: L = M = 1 is a low-pass)
INFERENCE_RATES = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000]


def pitch_rate_pairs(sr: int):
    """(sr_in, sr) of every pitch-shift step of augment.Augmenter's default range: resampled from int(sr / r) Hz to
    sr Hz with r = augment.shift_rate(n)."""
    lo, hi = inspect.signature(A.Augmenter).parameters["pitch"].default
    return [(int(sr / A.shift_rate(n)), sr) for n in range(lo, hi + 1) if n != 0]


def staged_bytes(L: int, M: int, K: int) -> int:
    """resample_smem (kernels_signal.cu): the input span one CTA of 256 outputs stages in shared memory."""
    return ((255 * M) // L + K + 2) * 4


def taps(sr_in: int, sr_out: int = SR) -> int:
    L, M = P.resample_ratio(sr_in, sr_out)
    return 2 * math.ceil(P.RESAMPLE_ZERO_CROSSINGS / min(1.0, L / M))


def largest_integer_ratio() -> int:
    """The largest k such that k * 22050 Hz -> 22050 Hz stages no more than MAX_SMEM."""
    k = 1
    while staged_bytes(1, k + 1, taps((k + 1) * SR)) <= MAX_SMEM:
        k += 1
    return k


OPT_IN_RATE = 32 * SR  # 705.6 kHz: K = 6016, about 57 KB staged
MAX_RATE = largest_integer_ratio() * SR
REFUSED_RATE = MAX_RATE + SR
HUGE_BANK_RATE = 400_003  # coprime with 22050: L = 22050, M = 400003, L * K > 2^26


@functools.lru_cache(maxsize=None)
def bank(sr_in: int, sr_out: int = SR):
    """preprocessing.resample_filter_bank, built once per ratio."""
    return P.resample_filter_bank(sr_in, sr_out)


# ------------------------------------------------------------------------------------------------------------ reference
def direct(x, sr_in: int, sr_out: int, n):
    """(y, B, T): the float64 direct form at the output indices n of the clip x (the float64 values of its fp32
    samples), and the bound of the module docstring split into its rounding part B and its truncation part T."""
    xv, w = O.resample_direct_terms(x, sr_in, sr_out, np.asarray(n, dtype=np.int64))
    K = xv.shape[1] - 3  # the direct form reads K + 3 samples, the kernel the K from the third on
    a = np.abs(xv * w)
    S = a[:, 2 : K + 2].sum(1)
    trunc = a[:, 0] + a[:, 1] + a[:, K + 2]
    B = (U + gamma(math.ceil(K / 4) + 3) * (1 + U)) * S + E64 * (S + np.abs(xv).sum(1))
    return (xv * w).sum(1), B, trunc


def ratio(got, y, B, T) -> float:
    """The largest (|got - y| - T) / B: at most 1 where got is within the bound B + T.  Reported against the rounding
    part alone, since T is exact (an isolated sample at |s t| = Z makes |got - y| = T, and T / (B + T) ~ 1 would say
    nothing about the arithmetic).  An unwritten (NaN) output counts as infinitely far; an output whose error is within
    T counts as 0, also where B is 0 (no input sample in reach)."""
    err = np.nan_to_num(np.abs(np.asarray(got, np.float64) - y), nan=np.inf) - T
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.max(np.where(err <= 0, 0.0, err / B), initial=0.0))


def emulate(x, coef, L: int, M: int, K: int, n, tap_shift=0, row_shift=0, drop_tail=False, outside=None):
    """resample_kernel's arithmetic in float32 at output indices n of the clip x (fp32): the same products in the same
    order (fmaf as the float64 sum of an exact product, rounded to float32: a second rounding of at most 2^-53
    relative, far inside the bound).  The keywords plant the indexing mistakes the CPU test must catch: read tap
    k + tap_shift, take phase row (n M + row_shift) mod L, drop the K mod 4 tail, or read `outside` (the samples of
    the neighbouring clips: outside[0] ends just before the clip, outside[1] starts just after it) instead of zeros."""
    x = np.asarray(x, dtype=np.float32)
    n = np.asarray(n, dtype=np.int64)
    j = ((n * M) // L - K // 2 + 1)[:, None] + np.arange(K)[None, :] + tap_shift
    if outside is None:
        xs = np.where((j >= 0) & (j < len(x)), x[np.clip(j, 0, max(len(x) - 1, 0))] if len(x) else 0, 0)
    else:
        before, after = (np.asarray(o, dtype=np.float32) for o in outside)
        ext = np.concatenate([before, x, after])
        xs = ext[np.clip(j + len(before), 0, len(ext) - 1)]
    xs = xs.astype(np.float32)
    c = coef[(n * M + row_shift) % L]
    acc = np.zeros((4, len(n)), np.float32)

    def fma(a, b, s):
        return (a.astype(np.float64) * b + s).astype(np.float32)

    k = 0
    while k + 4 <= K:
        for i in range(4):
            acc[i] = fma(c[:, k + i], xs[:, k + i], acc[i])
        k += 4
    while k < K and not drop_tail:
        acc[0] = fma(c[:, k], xs[:, k], acc[0])
        k += 1
    return ((acc[0] + acc[1]) + (acc[2] + acc[3])).astype(np.float64)


def sample_indices(n_out: int, K: int, rng, n_random: int = 20000, n_boundaries: int = 300):
    """Output indices of a long clip worth checking: the first and last 2K, +-2 around n_boundaries 256-output CTA
    boundaries spread over the clip, and n_random random ones."""
    edge = np.r_[np.arange(min(2 * K, n_out)), np.arange(max(n_out - 2 * K, 0), n_out)]
    cta = np.linspace(1, max((n_out - 1) // 256, 1), n_boundaries).astype(np.int64) * 256
    around = (cta[:, None] + np.arange(-2, 3)[None, :]).ravel()
    idx = np.unique(np.r_[edge, around, rng.integers(0, n_out, n_random)])
    return idx[(idx >= 0) & (idx < n_out)]
