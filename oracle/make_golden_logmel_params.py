"""Generate tests/golden/logmel_params.npz by running the UNMODIFIED reference's LogMelSpect (beat_this/preprocessing.py,
a torchaudio MelSpectrogram plus log1p) on the CPU for analysis parameters other than its defaults.

    BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_logmel_params.py

Per configuration k the fixture holds cfg{k} (the constructor's keyword arguments as JSON), the filterbank the
reference's MelSpectrogram holds (spect_class.mel_scale.fb) as fb_shape{k}, fb_nnz{k} (non-zero weights per band) and
fb_sha256{k}, the SHA-256 of its C-contiguous fp32 bytes: that pins the coefficients bitwise at 32 bytes where the
weights themselves would be most of the file.  Per signal j, sig{k}_{j} = (seed, length) of the
input, which tests/logmel_reference.py's pcm_signal rebuilds bit for bit (integer-only 16-bit PCM), and y{k}_{j}
(output [T, n_mels]).  The configurations cover n_fft 64 .. 8192, hops from 1 to beyond n_fft, six sample rates, both
mel scales, the four `normalized` values, power 0.5 / 1 / 2, log_multiplier 1 / 1000 / 1e4, 1 .. 256 bands (one
configuration with all-zero bands), explicit and None f_max, and the defaults.  Signal 0 of every configuration is
exactly n_fft // 2 + 1 samples long (the shortest torch's reflect padding accepts); signal 1 is two hops and a few
samples longer (one hop at hops of 1024 and more).  Signals, frame counts and the bands at n_fft 8192 are kept short
or narrow so that the file stays small.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if not os.environ.get("BEAT_THIS_REFERENCE"):
    sys.exit("usage: BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_logmel_params.py")
sys.path.insert(0, os.environ["BEAT_THIS_REFERENCE"])

import numpy as np
import torch

from beat_this.preprocessing import LogMelSpect  # the reference

sys.path.insert(0, os.path.join(ROOT, "tests"))
from logmel_reference import pcm_signal  # noqa: E402  (the inputs, rebuilt by the tests from their seeds)

GOLD = os.path.join(ROOT, "tests", "golden")


def _cfg(sample_rate, n_fft, hop_length, f_min, f_max, n_mels, mel_scale, normalized, power, log_multiplier):
    return dict(sample_rate=sample_rate, n_fft=n_fft, hop_length=hop_length, f_min=f_min, f_max=f_max, n_mels=n_mels,
                mel_scale=mel_scale, normalized=normalized, power=power, log_multiplier=log_multiplier)


CONFIGS = [
    _cfg(22050, 1024, 441, 30, 11000, 128, "slaney", "frame_length", 1, 1000),  # the defaults
    _cfg(8000, 64, 1, 0, None, 40, "htk", False, 2.0, 1e4),  # 33 bins for 40 bands: all-zero bands
    _cfg(11025, 256, 300, 20, None, 80, "slaney", "window", 0.5, 1.0),  # odd rate, hop > n_fft
    _cfg(16000, 512, 160, 0, 8000, 80, "htk", True, 2.0, 1000),
    _cfg(22050, 1024, 512, 30, None, 229, "slaney", "frame_length", 1, 1e4),
    _cfg(44100, 2048, 512, 30, 11000, 80, "htk", False, 2.0, 1000),
    _cfg(44100, 2048, 512, 30, None, 128, "slaney", "frame_length", 1, 1000),
    _cfg(22050, 4096, 441, 30, 11000, 128, "slaney", "frame_length", 1, 1000),
    _cfg(48000, 8192, 2048, 0, 8000, 256, "slaney", "window", 0.5, 1.0),
    _cfg(44100, 8192, 8200, 50, 2000, 1, "htk", False, 1, 1000),  # hop > n_fft, one band
    _cfg(11025, 128, 7, 0, None, 1, "slaney", "frame_length", 2.0, 1e4),
    _cfg(16000, 512, 160, 0, None, 80, "slaney", "frame_length", 1, 1000),
    _cfg(48000, 256, 64, 0, 24000, 128, "htk", "window", 1, 1000),
    _cfg(8000, 4096, 1024, 100, 3500, 256, "htk", True, 2.0, 1e4),
    _cfg(22050, 1024, 32, 30, 11000, 128, "slaney", "frame_length", 1, 1000),  # the defaults at a small hop
    _cfg(16000, 2048, 2049, 0, None, 40, "slaney", False, 0.5, 1.0),  # hop > n_fft
]


def main():
    rng = np.random.default_rng(2026)
    out = {}
    for k, cfg in enumerate(CONFIGS):
        mel = LogMelSpect(**cfg)
        n, hop = cfg["n_fft"], cfg["hop_length"]
        lens = (n // 2 + 1, n // 2 + 1 + (hop if hop >= 1024 else 2 * hop) + int(rng.integers(0, 64)))
        out[f"cfg{k}"] = np.array(json.dumps(cfg))
        fb = np.ascontiguousarray(mel.spect_class.mel_scale.fb.numpy(), dtype=np.float32)
        out[f"fb_shape{k}"] = np.asarray(fb.shape, np.int64)
        out[f"fb_nnz{k}"] = (fb != 0).sum(0).astype(np.int32)
        out[f"fb_sha256{k}"] = np.array(hashlib.sha256(fb.tobytes()).hexdigest())
        for j, length in enumerate(lens):
            seed = 100 * k + j
            with torch.no_grad():
                y = mel(torch.tensor(pcm_signal(seed, length))).numpy()
            out[f"sig{k}_{j}"] = np.asarray([seed, length], np.int64)
            out[f"y{k}_{j}"] = y
    out["n"] = np.int64(len(CONFIGS))
    path = os.path.join(GOLD, "logmel_params.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {len(CONFIGS)} configurations to {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
