"""Tempo and pitch augmentation of audio on the device, and the pure helpers of the reference's
``beat_this/dataset/augment.py`` that name the precomputed variants and move the annotations with them.

The reference's ``launch_scripts/preprocess_audio.py`` time-stretches and pitch-shifts with pedalboard (Rubber Band),
whose arithmetic is not part of the reference; parity with it is unpinned (DESIGN.md section 2).  Here both effects are
the classic phase vocoder as ``torch.stft`` -> ``torchaudio.functional.phase_vocoder`` -> ``torch.istft`` define it
(contracts of ``bt_stft``, ``bt_phase_vocoder`` and ``bt_istft`` in include/beatthis.h):

* time stretch by ``p`` percent (the reference's meaning: the tempo changes by p %, ``stretch_factor = 1 + p / 100``,
  positive is faster and shorter, beat times divide by the factor): vocoder rate ``r = 1 + p / 100``, output length
  ``round(len / r)`` (Python's round);
* pitch shift by ``n`` semitones, after ``torchaudio.functional.pitch_shift``: stretch at ``r = 2 ** (-n / 12)``, resample
  from ``int(sr / r)`` Hz to ``sr`` Hz with this project's resampler (``preprocessing.resample_filter_bank``, not
  torchaudio's), then cut or zero-pad to the input length.

One analysis of a clip serves all of its variants.  ``number_of_precomputed_augmentations`` of the reference is left
out on purpose: it unpacks ``augmentations.values()`` as pairs and raises for every augmentation dict the reference
uses.  ``augment_mask_`` (a training-time spectrogram augmentation) is not part of this module.
"""
from __future__ import annotations

import math
import numbers

import torch

from . import _lib
from .preprocessing import MEL_N_FFT_RANGE, fft_twiddles

# ---- the reference's pure helpers, restated ---------------------------------------------------------------------


def precomputed_augmentation_filenames(augmentations, ext="npy"):
    """File names of the precomputed variants of a piece, the unaugmented ``track`` first, then per key of
    ``augmentations`` in its order: "pitch" {"min", "max"} (inclusive, semitones) and "tempo" {"min", "max", "stride"}
    (inclusive, percent), zero skipped."""
    filenames = [f"track.{ext}"]
    for method, params in augmentations.items():
        if method == "pitch":
            filenames += [f"track_ps{n}.{ext}" for n in range(params["min"], params["max"] + 1) if n != 0]
        elif method == "tempo":
            filenames += [f"track_ts{p}.{ext}" for p in range(params["min"], params["max"] + 1, params["stride"]) if p != 0]
    return filenames


def stretch_annotations(item, percentage):
    """The item with its "beat_time" divided by 1 + percentage / 100 (the tempo changes by that percentage)."""
    if not percentage:
        return item
    item = dict(item)
    item["beat_time"] = item["beat_time"] / (1.0 + percentage / 100)
    return item


def stretch_filename(item, percentage):
    """The item with "spect_path" (a pathlib path) renamed to its time-stretched variant <stem>_ts<percentage>."""
    path = item["spect_path"]
    if percentage:
        path = path.with_stem(path.stem + f"_ts{percentage}")
    return {**item, "spect_path": path}


def shift_filename(item, semitones):
    """The item with "spect_path" renamed to its pitch-shifted variant <stem>_ps<semitones>."""
    path = item["spect_path"]
    if semitones:
        path = path.with_stem(path.stem + f"_ps{semitones}")
    return {**item, "spect_path": path}


def augmentation_dict(pitch, tempo) -> dict:
    """The reference's augmentation dict from preprocess_audio.py's (LOW, HIGH) semitones and (MAX, STRIDE) percent;
    None leaves a kind out."""
    aug = {}
    if pitch is not None:
        aug["pitch"] = {"min": int(pitch[0]), "max": int(pitch[1])}
    if tempo is not None:
        aug["tempo"] = {"min": -int(tempo[0]), "max": int(tempo[0]), "stride": int(tempo[1]) if len(tempo) > 1 else 1}
    return aug


# ---- the contract's host arithmetic ---------------------------------------------------------------------------------


def stretch_rate(percent) -> float:
    return 1.0 + percent / 100


def shift_rate(semitones) -> float:
    return 2.0 ** (-float(semitones) / 12)


def check_rate(rate: float) -> float:
    lo, hi = _lib.VOCODER_RATE_RANGE
    if not (math.isfinite(rate) and lo <= rate <= hi):
        raise ValueError(f"phase vocoder rate {rate} outside [{lo}, {hi}]")
    return float(rate)


def stretched_length(n_samples: int, rate: float) -> int:
    """round(len / rate) with Python's round (half to even), as torchaudio.functional.pitch_shift."""
    return int(round(n_samples / rate))


class StftTables:
    """Constants of one bt_stft / bt_istft analysis on a device: the config struct, the periodic Hann window and the
    FFT twiddles.  ``NotImplementedError`` for an n_fft that is not a power of two in [64, 8192] or hop_length < 1."""

    def __init__(self, n_fft, hop_length, device):
        lo, hi = MEL_N_FFT_RANGE
        if not (isinstance(n_fft, numbers.Integral) and lo <= n_fft <= hi and n_fft & (n_fft - 1) == 0
                and isinstance(hop_length, numbers.Integral) and hop_length >= 1):
            raise NotImplementedError(f"the STFT kernels take a power-of-two n_fft in [{lo}, {hi}] and hop_length >= 1 "
                                      f"(got n_fft={n_fft}, hop_length={hop_length})")
        self.n_fft, self.hop_length, self.bins = int(n_fft), int(hop_length), int(n_fft) // 2 + 1
        self.config = _lib.bt_stft_config(self.n_fft, self.hop_length)
        self.window = torch.hann_window(self.n_fft, periodic=True).to(device)
        self.twiddle = torch.from_numpy(fft_twiddles(self.n_fft)).to(device)


class Augmenter:
    """Time-stretched and pitch-shifted variants of clips at ``sr`` Hz on the device.

    ``pitch``: (LOW, HIGH) semitones inclusive, ``tempo``: (MAX, STRIDE) percent (-MAX .. MAX), either may be None;
    the variants and their names are ``precomputed_augmentation_filenames`` of that dict.  A batch is processed in
    groups whose spectrograms fit ``group_bytes``: per group one analysis launch, one vocoder launch for all variants of
    all its clips, one synthesis call, and one resampling call per pitch step.  The polyphase bank of a pitch step
    (``resample_filter_bank(int(sr / r), sr)``) is built the first time the step is used and kept by the engine."""

    def __init__(self, sr, pitch=(-5, 6), tempo=(20, 4), n_fft=2048, hop_length=512, device="cuda", group_bytes=4 << 30,
                 _engine=None):
        from .engine import Engine

        if not (isinstance(sr, numbers.Integral) and sr > 0):
            raise ValueError("sr must be a positive integer")
        self.sr = int(sr)
        self.augmentations = augmentation_dict(pitch, tempo)
        self.names = [f[:-4] for f in precomputed_augmentation_filenames(self.augmentations)]
        self.variants = []  # (name, rate, rate to resample from or None) of every name but "track"
        for name in self.names[1:]:
            kind, amount = name[6:8], int(name[8:])
            rate = check_rate(shift_rate(amount) if kind == "ps" else stretch_rate(amount))
            self.variants.append((name, rate, int(self.sr / rate) if kind == "ps" else None))
        self.engine = _engine if _engine is not None else Engine(None, None, device)
        self.tables = StftTables(n_fft, hop_length, self.engine.device)
        self.group_bytes = int(group_bytes)

    # bytes of device memory the variants of one clip take: the analysis, the variant spectrograms, and bt_istft's
    # scratch of n_fft floats per variant frame
    def clip_bytes(self, n_samples: int, rates) -> int:
        t = self.tables
        T = 1 + n_samples // t.hop_length
        frames_out = sum(math.ceil(T / r) for r in rates)
        return 8 * t.bins * (T + frames_out) + 4 * t.n_fft * frames_out

    def _signals(self, signals):
        sigs = [torch.as_tensor(s, dtype=torch.float32, device=self.engine.device).contiguous() for s in signals]
        for s in sigs:
            if s.ndim != 1:
                raise ValueError("signals must be one-dimensional")
            if s.numel() <= self.tables.n_fft // 2:
                raise ValueError(f"a clip of {s.numel()} samples is too short for n_fft={self.tables.n_fft} "
                                 "(reflect padding needs more than n_fft / 2 samples)")
        return sigs

    def apply(self, signals, variants):
        """variants: (name, rate, resample_from) triples applied to every clip.  Returns per clip {name: tensor}."""
        sigs = self._signals(signals)
        rates = [check_rate(r) for _, r, _ in variants]
        out = [dict() for _ in sigs]
        lo = 0
        while lo < len(sigs) and variants:
            hi, used = lo, 0
            while hi < len(sigs) and (hi == lo or used + self.clip_bytes(sigs[hi].numel(), rates) <= self.group_bytes):
                used += self.clip_bytes(sigs[hi].numel(), rates)
                hi += 1
            self._group(sigs[lo:hi], variants, out[lo:hi])
            lo = hi
        return out

    def _group(self, sigs, variants, out):
        eng, nv = self.engine, len(variants)
        so = _lib.offsets(s.numel() for s in sigs)
        spec, fo = eng.stft_cat(torch.cat(sigs) if len(sigs) > 1 else sigs[0], so, self.tables)
        # clip-major: the variants of a clip run together and share its analysis
        v_clip = [c for c in range(len(sigs)) for _ in variants]
        v_rate = [r for _ in sigs for _, r, _ in variants]
        vspec, vfo = eng.phase_vocoder_cat(spec, fo, v_clip, v_rate)
        lengths = [stretched_length(sigs[c].numel(), r) for c, r in zip(v_clip, v_rate)]
        audio, vso = eng.istft_cat(vspec, vfo, lengths, self.tables)
        del spec, vspec
        for k, (name, _, sr_from) in enumerate(variants):
            seqs = [c * nv + k for c in range(len(sigs))]
            parts = [audio[vso[q] : vso[q + 1]] for q in seqs]
            if sr_from is None:
                for c, p in enumerate(parts):
                    out[c][name] = p
                continue
            po = _lib.offsets(p.numel() for p in parts)
            res, ro = eng.resample_cat(torch.cat(parts) if len(parts) > 1 else parts[0].contiguous(), po, sr_from, self.sr)
            for c in range(len(sigs)):
                n, y = sigs[c].numel(), res[ro[c] : ro[c + 1]]
                out[c][name] = y[:n] if y.numel() >= n else torch.nn.functional.pad(y, (0, n - y.numel()))

    def batch(self, signals):
        """For every clip a dict {name: fp32 device tensor} in ``names`` order: "track" (the clip itself), then
        "track_ps<n>" and "track_ts<p>"."""
        sigs = self._signals(signals)
        res = self.apply(sigs, self.variants) if self.variants else [dict() for _ in sigs]
        return [{"track": s, **r} for s, r in zip(sigs, res)]


def time_stretch(signals, sr, percent, n_fft=2048, hop_length=512, device="cuda"):
    """Every clip (1-D arrays or tensors at ``sr`` Hz) with its tempo changed by ``percent`` percent: fp32 device
    tensors of round(len / (1 + percent / 100)) samples."""
    aug = Augmenter(sr, None, None, n_fft, hop_length, device)
    res = aug.apply(signals, [("ts", check_rate(stretch_rate(percent)), None)])
    return [r["ts"] for r in res]


def pitch_shift(signals, sr, semitones, n_fft=2048, hop_length=512, device="cuda"):
    """Every clip shifted by ``semitones`` semitones at its own length."""
    aug = Augmenter(sr, None, None, n_fft, hop_length, device)
    rate = check_rate(shift_rate(semitones))
    res = aug.apply(signals, [("ps", rate, int(aug.sr / rate))])
    return [r["ps"] for r in res]
