"""float64 numpy restatement of the contracts of bt_stft, bt_phase_vocoder and bt_istft (include/beatthis.h), the
composed time stretch and pitch-shift stretch, and elementwise error bounds of the fp32 device kernels against them.
"""
from __future__ import annotations

import math

import numpy as np

from numerics import U

ATAN2F_ERR = 2.0 ** -21  # 2 ulp of a value <= pi (CUDA math API: atan2f max error 2 ulp)


def hash_signal(seed: int, n: int) -> np.ndarray:
    """Deterministic test signal of n samples, fp32 in [-1, 1): 16-bit PCM from integer arithmetic only (splitmix64
    of the sample index, four 12-bit fields summed for a bell-shaped noise, plus a square wave from the seed).
    Vectorised, so long clips are cheap; fixtures store (seed, n)."""
    with np.errstate(over="ignore"):
        z = (np.arange(n, dtype=np.uint64) + np.uint64(seed)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    acc = sum(((z >> np.uint64(12 * k)) & np.uint64(0xFFF)).astype(np.int64) for k in range(4))
    period, level = 8 + seed % 61, 1000 + 37 * (seed % 97)
    sq = np.where((np.arange(n) // period) % 2 == 1, level, -level)
    return (((acc - 8190) // 4 + sq).astype(np.float32) / 32768).astype(np.float32)


def hann(n_fft: int) -> np.ndarray:
    """The periodic Hann window as its fp32 values (torch.hann_window(periodic=True)), in float64."""
    import torch

    return torch.hann_window(n_fft, periodic=True).double().numpy()


def stft(x, n_fft: int, hop: int) -> np.ndarray:
    """[1 + len // hop, n_fft // 2 + 1] complex128: center=True, reflect padding, onesided, not normalised."""
    x = np.asarray(x, np.float64)
    xp = np.pad(x, n_fft // 2, mode="reflect")
    T = 1 + len(x) // hop
    frames = xp[np.arange(T)[:, None] * hop + np.arange(n_fft)[None, :]]
    return np.fft.rfft(frames * hann(n_fft), axis=1)


def vocoder_frames(T: int, rate: float) -> int:
    return int(math.ceil(T / rate))


def next_index(s) -> np.ndarray:
    """The frame paired with floor(s): floor(s + 1) with the sum rounded to float64, as torchaudio indexes it.  That is
    floor(s) + 1, except where s lies within an ulp below an integer: there the sum rounds up and it is floor(s) + 2."""
    return np.floor(s + 1.0).astype(np.int64)


def phase_vocoder(X, rate: float, hop: int) -> np.ndarray:
    """The contract as written: [ceil(T / rate), bins] complex128 from X [T, bins]."""
    X = np.asarray(X, np.complex128)
    T, bins = X.shape
    s = np.arange(vocoder_frames(T, rate), dtype=np.float64) * rate
    i = np.floor(s).astype(np.int64)
    alpha = (s - i)[:, None]
    Xp = np.concatenate([X, np.zeros((2, bins), np.complex128)])
    x0, x1 = Xp[i], Xp[next_index(s)]
    omega = np.pi * hop * np.arange(bins) / (bins - 1)
    d = np.angle(x1) - np.angle(x0) - omega
    d = d - 2 * np.pi * np.round(d / (2 * np.pi)) + omega
    phi = np.cumsum(np.concatenate([np.angle(X[:1]), d[:-1]]), axis=0)
    mag = alpha * np.abs(x1) + (1 - alpha) * np.abs(x0)
    return mag * np.exp(1j * phi)


def istft_parts(Y, n_fft: int, hop: int, length: int):
    """(overlap-added windowed frames, window envelope) of the `length` samples after the n_fft // 2 centre padding,
    zero where no frame covers a sample."""
    Y = np.asarray(Y, np.complex128).copy()
    Y[:, 0] = Y[:, 0].real
    Y[:, -1] = Y[:, -1].real
    w = hann(n_fft)
    frames = np.fft.irfft(Y, n=n_fft, axis=1) * w
    F = len(Y)
    total = max(n_fft + hop * (F - 1), n_fft // 2 + length)
    acc, env = np.zeros(total), np.zeros(total)
    for f in range(F):
        acc[f * hop : f * hop + n_fft] += frames[f]
        env[f * hop : f * hop + n_fft] += w * w
    return acc[n_fft // 2 : n_fft // 2 + length], env[n_fft // 2 : n_fft // 2 + length]


def istft(Y, n_fft: int, hop: int, length: int) -> np.ndarray:
    acc, env = istft_parts(Y, n_fft, hop, length)
    covered = np.arange(length) + n_fft // 2 < n_fft + hop * (len(Y) - 1)
    if covered.any() and env[covered].min() < 1e-11:
        raise ValueError("window envelope below 1e-11")
    return np.where(covered, acc / np.where(covered, env, 1.0), 0.0)


def stretched_length(n: int, rate: float) -> int:
    return int(round(n / rate))


def stretch(x, rate: float, n_fft: int, hop: int) -> np.ndarray:
    """Analysis -> vocoder -> synthesis to round(len / rate) samples."""
    return istft(phase_vocoder(stft(x, n_fft, hop), rate, hop), n_fft, hop, stretched_length(len(x), rate))


# ---- bounds of the fp32 kernels ----------------------------------------------------------------------------------


def fft_delta(n_fft: int, l2_norm):
    """Per-output error of an n_fft-point fp32 transform of data with that l2 norm per unit of output scale: the
    derivation of logmel_reference.device_bound (Higham thm. 24.2 per radix-2 stage, two stages for the untangling and
    window, the rms share of the norm-wise bound times a safety factor 8)."""
    return 8 * (math.log2(n_fft) + 2) * 8 * U * math.sqrt(2.0) * np.asarray(l2_norm)


def stft_bound(x, n_fft: int, hop: int) -> np.ndarray:
    """[T, 1]: |X_device - X| <= this for every bin of a frame (complex modulus)."""
    x = np.asarray(x, np.float64)
    xp = np.pad(x, n_fft // 2, mode="reflect")
    T = 1 + len(x) // hop
    frames = xp[np.arange(T)[:, None] * hop + np.arange(n_fft)[None, :]] * hann(n_fft)
    return fft_delta(n_fft, np.sqrt((frames * frames).sum(1)))[:, None]


def vocoder_bound(X, rate: float) -> np.ndarray:
    """[T_out, bins]: |Y_device - Y| <= this, for the device's fp32 input X.  Magnitude: two sqrtf and the fp32
    interpolation, 8u (|X[i]| + |X[i+1]|).  Phase: two atan2f per step accumulated in float64 and reduced modulo 2 pi,
    (2 j + 1) 2^-21 rad at frame j, plus sincosf and the rounding of phi to fp32, 2^-21."""
    X = np.asarray(X, np.complex128)
    T, bins = X.shape
    n = vocoder_frames(T, rate)
    s = np.arange(n, dtype=np.float64) * rate
    i = np.floor(s).astype(np.int64)
    alpha = (s - i)[:, None]
    Xp = np.abs(np.concatenate([X, np.zeros((2, bins), np.complex128)]))
    i1 = next_index(s)
    mag = alpha * Xp[i1] + (1 - alpha) * Xp[i]
    phase_err = (2 * np.arange(n)[:, None] + 2) * ATAN2F_ERR
    return mag * phase_err + 8 * U * (Xp[i] + Xp[i1]) + 1e-30


def istft_bound(Y, n_fft: int, hop: int, length: int) -> np.ndarray:
    """[length]: |y_device - y| <= this.  Each sample of frame f's inverse transform x_f is off by the rms share
    fft_delta(||x_f||_2) / sqrt(n_fft) of the transform's norm-wise error; the window scales it; the fp32 sums of c
    frames and of the envelope add (c + 2) u relative to the sum of moduli; the division adds u."""
    Y = np.asarray(Y, np.complex128).copy()
    Y[:, 0] = Y[:, 0].real
    Y[:, -1] = Y[:, -1].real
    w = hann(n_fft)
    x = np.fft.irfft(Y, n=n_fft, axis=1)
    e = fft_delta(n_fft, np.sqrt((x * x).sum(1))) / math.sqrt(n_fft)  # per sample of frame f: the rms share
    F = len(Y)
    total = max(n_fft + hop * (F - 1), n_fft // 2 + length)
    err, mod, env = np.zeros(total), np.zeros(total), np.zeros(total)
    for f in range(F):
        sl = slice(f * hop, f * hop + n_fft)
        err[sl] += w * e[f]
        mod[sl] += np.abs(w * x[f])
        env[sl] += w * w
    sl = slice(n_fft // 2, n_fft // 2 + length)
    c = math.ceil(n_fft / hop)
    envs = np.where(env[sl] > 0, env[sl], 1.0)
    return (err[sl] + (2 * c + 6) * U * mod[sl]) / envs + 1e-30
