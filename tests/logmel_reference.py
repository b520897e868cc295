"""float64 numpy restatement of bt_logmel_config's contract (include/beatthis.h) and the elementwise error bound of the
fp32 device kernel against it.

Contract: frames of n_fft samples every hop_length samples of the signal reflect-padded by n_fft // 2 at each end
(no edge repeat), times the window (the periodic Hann window, taken as its fp32 values), onesided DFT, scaled by
n_fft^-1/2 ("frame_length"), 1 / sqrt(sum window^2) (True, "window") or 1 (False), magnitude to the power `power`,
times the filterbank (torchaudio's fp32 coefficients, exact in float64), log1p(log_multiplier * mel).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from numerics import U


def pcm_signal(seed: int, n: int) -> np.ndarray:
    """Deterministic test signal of n samples, fp32 in [-1, 1): 16-bit PCM built from integers only (a 64-bit linear
    congruential generator, four of its 12-bit outputs summed for a bell-shaped noise, plus a square wave whose period
    and level come from the seed), so every platform makes the same samples and fixtures store (seed, n) instead."""
    state, mask = seed * 2654435761 + 1, (1 << 64) - 1
    period, level = 8 + seed % 61, 1000 + 37 * (seed % 97)
    out = np.empty(n, np.int64)
    for i in range(n):
        acc = 0
        for _ in range(4):
            state = (state * 6364136223846793005 + 1442695040888963407) & mask
            acc += state >> 52
        out[i] = (acc - 8190) // 4 + (level if (i // period) % 2 else -level)
    return (out.astype(np.float32) / 32768).astype(np.float32)


def spectrum(x, n_fft: int, hop_length: int, normalized) -> tuple[np.ndarray, np.ndarray]:
    """|X[t, k]| times the normalisation (float64, [T, n_fft // 2 + 1]) and the frames' window-weighted l2 norms [T]."""
    x = np.asarray(x, np.float64)
    xp = np.pad(x, n_fft // 2, mode="reflect")
    T = 1 + len(x) // hop_length
    frames = xp[np.arange(T)[:, None] * hop_length + np.arange(n_fft)[None, :]]
    w = torch.hann_window(n_fft, periodic=True).double().numpy()
    if normalized == "frame_length":
        scale = n_fft ** -0.5
    elif normalized is True or normalized == "window":
        scale = 1.0 / math.sqrt(float((w * w).sum()))
    elif normalized is False:
        scale = 1.0
    else:
        raise ValueError(f"Invalid normalized parameter: {normalized}")
    xw = frames * w
    return np.abs(np.fft.rfft(xw, axis=1)) * scale, np.sqrt((xw * xw).sum(1)) * scale


def logmel(x, fb, n_fft: int, hop_length: int, normalized, power: float, log_multiplier: float) -> np.ndarray:
    """The contract in float64: [T, n_mels]."""
    mag, _ = spectrum(x, n_fft, hop_length, normalized)
    return np.log1p(log_multiplier * (mag ** power) @ np.asarray(fb, np.float64))


def device_bound(x, fb, n_fft: int, hop_length: int, normalized, power: float, log_multiplier: float):
    """(lo, hi) [T, n_mels] that the fp32 kernel's output must lie in, derived from the float64 values:

    - FFT: Higham, Accuracy and Stability of Numerical Algorithms, thm. 24.2: a radix-2 FFT with twiddles accurate to
      mu has ||dX||_2 <= log2(n) eta ||X||_2, eta = mu + gamma_4 (sqrt 2 + mu) ~ 7u for mu = u (fp32 tables rounded
      from float64).  Each radix-8 pass is three such stages, radix 4 two and radix 2 one; the untangling step, the
      window product and the reflected read charge two stages more.  So ||dX||_2 <= (log2(n_fft) + 2) 8u ||X||_2 with
      ||X||_2 = sqrt(n_fft) ||x w||_2 for the full transform.  That is a norm over all bins; the round-off of a pass is
      spread over its outputs, so each bin is charged the rms share sqrt(2 / n_fft) of it, times a safety factor 8
      (the norm-wise bound itself is sqrt(n_fft / 2) times larger): delta = 8 (log2 n_fft + 2) 8u sqrt 2 ||x w||_2.
    - power: |X| in [|X| - delta, |X| + delta] maps to S in [(|X| - delta)_+^p, (|X| + delta)^p], widened by 4u
      relative for powf and the magnitude's sqrt.
    - mel: the fp32 sum over a band's b terms adds (b + 2) u relative to the sum of |terms|.
    - log1p(m x) maps the mel interval exactly; this is where m turns absolute error in x into m times as much near 0.
      log1pf and the product m x add 4u relative plus an absolute 1e-7.
    """
    mag, xw_norm = spectrum(x, n_fft, hop_length, normalized)
    fb = np.asarray(fb, np.float64)
    delta = 8 * (math.log2(n_fft) + 2) * 8 * U * math.sqrt(2.0) * xw_norm[:, None]
    s_lo = np.clip(mag - delta, 0.0, None) ** power * (1 - 4 * U)
    s_hi = (mag + delta) ** power * (1 + 4 * U)
    terms = (fb != 0).sum(0)[None, :]
    mel_lo, mel_hi = s_lo @ fb, s_hi @ fb
    mel_lo = np.clip(mel_lo * (1 - (terms + 2) * U), 0.0, None)
    mel_hi = mel_hi * (1 + (terms + 2) * U)
    lo = np.log1p(log_multiplier * mel_lo)
    hi = np.log1p(log_multiplier * mel_hi)
    return lo - 4 * U * np.abs(lo) - 1e-7, hi + 4 * U * np.abs(hi) + 1e-7
