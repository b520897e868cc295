"""Writes tests/golden/augment.npz (CPU only).

* The phase-vocoder contract from code this project does not own: ``torch.stft`` ->
  ``torchaudio.functional.phase_vocoder`` (its time steps taken as the products j * rate, see ``product_arange``) ->
  ``torch.istft(length=round(len / rate))`` in float64 on seeded signals
  (``tests/augment_reference.hash_signal``; the fixture stores the seeds), down-sampled to probes: every PROBE_SAMPLE-th
  output sample and, of every PROBE_FRAME-th vocoder frame, every PROBE_BIN-th bin.
* What the unmodified reference's ``precomputed_augmentation_filenames``, ``stretch_annotations``,
  ``stretch_filename`` and ``shift_filename`` (beat_this/dataset/augment.py) return for a handful of inputs.

    python oracle/make_golden_augment.py /path/to/beat_this
"""
import json
import os
import sys
from unittest import mock
from pathlib import Path

import numpy as np
import torch
import torchaudio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from augment_reference import hash_signal  # noqa: E402

PROBE_SAMPLE, PROBE_FRAME, PROBE_BIN = 97, 13, 7

# (n_fft, hop, rate, samples): edge lengths n_fft/2 + 1, = 0 and = hop - 1 (mod hop); the last is ten minutes of frames
CONFIGS = [
    (64, 16, 0.8, 33),
    (64, 16, 4.0, 16 * 40),
    (64, 1, 1.2, 700),
    (512, 128, 0.84, 128 * 31 + 127),
    (512, 256, 2 ** (5 / 12), 9001),
    (512, 441, 0.25, 12000),
    (2048, 512, 1.0, 30000),
    (2048, 512, 1.2, 44100),
    (2048, 512, 0.8, 44100),
    (2048, 512, 2 ** (-5 / 12), 40000),
    (2048, 512, 2 ** (-6 / 12), 40000),
    (2048, 1024, 0.84, 30000),
    (8192, 2048, 1.2, 70000),
    (64, 16, 1.04, 16 * 50000),
]


_arange = torch.arange


def product_arange(start, end, step, **kw):
    """torch.arange(0, T, rate) with the values the contract names, s_j = j * rate rounded once.  torch's own kernel
    accumulates them differently by an ulp, which moves floor(s_j) at some of the frames where j * rate is an integer
    (rate 1.2: 92 of the 2154 frames of a 30 s clip at hop 512) -- an accident of its vectorisation, not part of the
    vocoder.  Everything else in phase_vocoder runs as torchaudio wrote it."""
    assert start == 0
    n = len(_arange(start, end, step, **kw))
    return _arange(n, **kw) * step


def vocoder_case(n_fft, hop, rate, n, seed):
    x = torch.from_numpy(hash_signal(seed, n)).double()
    w = torch.hann_window(n_fft, periodic=True).double()
    X = torch.stft(x, n_fft, hop, n_fft, w, center=True, pad_mode="reflect", normalized=False, onesided=True,
                   return_complex=True)
    adv = torch.linspace(0, np.pi * hop, n_fft // 2 + 1, dtype=torch.float64)[..., None]
    with mock.patch("torch.arange", product_arange):
        Y = torchaudio.functional.phase_vocoder(X, rate, adv)
    y = torch.istft(Y, n_fft, hop, n_fft, w, length=int(round(n / rate)))
    return Y.numpy().T[::PROBE_FRAME, ::PROBE_BIN], y.numpy()[::PROBE_SAMPLE], Y.shape[1], len(y)


def helper_cases(ref_root):
    # the file itself, not the package: beat_this.dataset imports the training stack on import
    import importlib.util

    spec = importlib.util.spec_from_file_location("ref_augment", os.path.join(ref_root, "beat_this", "dataset", "augment.py"))
    A = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(A)

    dicts = [{}, {"pitch": {"min": -5, "max": 6}}, {"tempo": {"min": -20, "max": 20, "stride": 4}},
             {"pitch": {"min": -5, "max": 6}, "tempo": {"min": -20, "max": 20, "stride": 4}},
             {"tempo": {"min": -8, "max": 8, "stride": 8}, "pitch": {"min": -1, "max": 1}}]
    names = [[A.precomputed_augmentation_filenames(d), A.precomputed_augmentation_filenames(d, "wav")] for d in dicts]
    beats = np.array([0.5, 1.0, 1.52, 2.75, 10.0])
    items = []
    for amount in (-20, -4, 0, 4, 20, 6):
        item = {"spect_path": Path("data/audio/spectrograms/ballroom/Albums-Cafe_Paradiso-05/track.npy"),
                "beat_time": beats}
        items.append({"amount": amount,
                      "stretch_path": str(A.stretch_filename(item, amount)["spect_path"]),
                      "shift_path": str(A.shift_filename(item, amount)["spect_path"]),
                      "beat_time": A.stretch_annotations(item, amount)["beat_time"].tolist()})
    return {"dicts": dicts, "names": names, "beats": beats.tolist(), "items": items}


def main(ref_root):
    out = {"configs": np.array([(a, b, d) for a, b, _, d in CONFIGS], np.int64),
           "rates": np.array([c for _, _, c, _ in CONFIGS], np.float64),
           "seeds": np.arange(len(CONFIGS), dtype=np.int64) + 11,
           "probe": np.array([PROBE_SAMPLE, PROBE_FRAME, PROBE_BIN], np.int64)}
    shapes = []
    for k, (n_fft, hop, rate, n) in enumerate(CONFIGS):
        Y, y, frames, length = vocoder_case(n_fft, hop, rate, n, 11 + k)
        out[f"Y{k}"], out[f"y{k}"] = Y, y
        shapes.append((frames, length))
    out["shapes"] = np.array(shapes, np.int64)
    out["helpers"] = np.frombuffer(json.dumps(helper_cases(ref_root)).encode(), np.uint8)
    path = os.path.join(ROOT, "tests", "golden", "augment.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
