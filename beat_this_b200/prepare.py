"""Prepare training spectrograms on the device: the work of the reference's ``launch_scripts/preprocess_audio.py``.

For every annotated piece: mono mix, the unaugmented ``track`` resampled straight from the file's rate to 22.05 kHz,
and -- from the piece at ``aug_sr`` (44.1 kHz) -- its pitch-shifted and time-stretched variants (``augment.Augmenter``),
each resampled to 22.05 kHz; the log-mel spectrogram of each (``LogMelSpect`` at the reference defaults) as float16
members ``<stem>/track.npy``, ``<stem>/track_ps-5.npy``, ... of ``OUT/audio/spectrograms/<dataset>.npz``, an uncompressed
zip in the order ``create_npz`` writes (pieces sorted by name, members in ``precomputed_augmentation_filenames``
order), with the ``.beats`` files under ``OUT/annotations/<dataset>/annotations/beats/``: the layout
``evaluate.discover_data`` and the reference's dataset read.

Two departures from the reference: it stores every variant as a 16-bit WAV file before taking its spectrogram and this
does not quantise; and a piece that fails is reported and skipped, at its own cost only.

    python -m beat_this_b200.prepare --audio DIR --annotations DIR --out DATA_DIR --dataset NAME
"""
from __future__ import annotations

import argparse
import os
import shutil
import sys
import zipfile
from pathlib import Path

import numpy as np
import torch

from . import _lib
from .augment import Augmenter, augmentation_dict, precomputed_augmentation_filenames
from .preprocessing import SAMPLE_RATE, load_audio

GROUP_SECONDS = 600.0  # audio a group of pieces may hold; the Augmenter splits further by its own byte budget


class BundleWriter:
    """Writes ``<stem>/<name>.npy`` members into an uncompressed .npz, piece by piece; the file appears under its name
    when the writer is closed without an error."""

    def __init__(self, path):
        self.path = Path(path)
        self.path.parent.mkdir(parents=True, exist_ok=True)
        self.tmp = self.path.with_name(self.path.name + f".tmp{os.getpid()}")
        self.zip = zipfile.ZipFile(self.tmp, "w", zipfile.ZIP_STORED, allowZip64=True)

    def add(self, stem: str, members: dict):
        for name, spect in members.items():
            with self.zip.open(f"{stem}/{name}.npy", "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.ascontiguousarray(spect, dtype=np.float16), allow_pickle=False)

    def close(self, ok: bool = True):
        self.zip.close()
        if ok:
            os.replace(self.tmp, self.path)
        else:
            self.tmp.unlink(missing_ok=True)

    def __enter__(self):
        return self

    def __exit__(self, exc_type, *_):
        self.close(exc_type is None)


def audio_files(paths) -> list:
    """Files named by ``paths`` (directories searched recursively, ``.beats`` files left out), sorted by stem."""
    files = []
    for p in map(Path, [paths] if isinstance(paths, (str, os.PathLike)) else paths):
        files += [f for f in p.rglob("*") if f.is_file() and f.suffix != ".beats"] if p.is_dir() else [p]
    return sorted(files, key=lambda f: f.stem)


def _load_group(paths, infos, device, host_threads: int = 8):
    """Files of one sample rate -> (flat mono fp32 device audio, sample offsets): WAV files through the native reader
    (_lib.stage_wav_files, the path of File2Beats.batch), anything else (infos[i] None) through load_audio."""
    decoded = {i: load_audio(p, dtype="float32")[0] for i, p in enumerate(paths) if infos[i] is None}
    so = _lib.offsets(infos[i].frames if infos[i] is not None else len(decoded[i]) for i in range(len(paths)))
    host = torch.empty(so[-1], dtype=torch.float32, pin_memory=True)
    wav = [i for i in range(len(paths)) if infos[i] is not None]
    if wav:  # file k of the call lands at its own slot so[wav[k]] of host
        _lib.stage_wav_files([paths[i] for i in wav], [infos[i] for i in wav], host, [so[i] for i in wav] + [so[-1]],
                             host_threads)
    for i, w in decoded.items():
        w = np.asarray(w, dtype=np.float32)
        host[so[i] : so[i + 1]] = torch.from_numpy(w if w.ndim == 1 else w.mean(axis=1))
    return host.to(device, non_blocking=True), so


def prepare(audio, annotations, out, dataset, pitch_shift=(-5, 6), time_stretch=(20, 4), aug_sr=44100, augment=True,
            batch=8, device="cuda", verbose=False) -> dict:
    """Write the bundle of ``dataset`` under ``out`` from the audio files ``audio`` (files or directories) and the
    ``<stem>.beats`` files of ``annotations``.  Returns {"written": [stems], "skipped": {stem: reason},
    "bundle": path, "members": [names]}."""
    from .engine import Engine
    from .preprocessing import LogMelSpect

    out = Path(out)
    ann_in = Path(annotations)
    ann_out = out / "annotations" / dataset / "annotations" / "beats"
    augmentations = augmentation_dict(pitch_shift, time_stretch) if augment else {}
    names = [f[:-4] for f in precomputed_augmentation_filenames(augmentations)]
    engine = Engine.mel_only(device)
    logmel = LogMelSpect(_engine=engine)
    augmenter = Augmenter(aug_sr, pitch_shift, time_stretch, _engine=engine) if len(names) > 1 else None
    written, skipped = [], {}

    def skip(stem, reason):
        skipped[stem] = reason
        print(f"skipping {stem}: {reason}", file=sys.stderr)

    def spectrograms(audio_dev, so, sr):
        """float16 host spectrograms of the clips of flat device audio at sr Hz."""
        if sr != SAMPLE_RATE:
            audio_dev, so = engine.resample_cat(audio_dev, so, sr, SAMPLE_RATE)
        spects = logmel.batch([audio_dev[so[i] : so[i + 1]] for i in range(len(so) - 1)])
        return [s.to(torch.float16).cpu().numpy() for s in spects]

    def run_group(group, sr):
        """[(path, info)] of one sample rate -> per piece {name: float16 spectrogram}."""
        audio_dev, so = _load_group([p for p, _ in group], [i for _, i in group], engine.device)
        n = len(group)
        members = [{"track": s} for s in spectrograms(audio_dev, so, sr)]
        if augmenter is not None:
            if sr != aug_sr:
                audio_dev, so = engine.resample_cat(audio_dev, so, sr, aug_sr)
            variants = augmenter.batch([audio_dev[so[i] : so[i + 1]] for i in range(n)])
            for name in names[1:]:
                parts = [variants[i][name] for i in range(n)]
                po = _lib.offsets(p.numel() for p in parts)
                for i, s in enumerate(spectrograms(torch.cat(parts) if n > 1 else parts[0].contiguous(), po, aug_sr)):
                    members[i][name] = s
        return members

    todo = []
    files = audio_files(audio)
    infos, is_wav = _lib.wav_probe(files)
    for f, info, ok in zip(files, infos, is_wav):
        if not (ann_in / f"{f.stem}.beats").exists():
            skip(f.stem, f"beat annotation {f.stem}.beats not found")
            continue
        info = info if ok else None
        try:
            sr = int(info.sample_rate) if info is not None else int(load_audio(f)[1])
        except Exception as e:
            skip(f.stem, str(e))
            continue
        todo.append((f, info, sr))

    bundle = out / "audio" / "spectrograms" / f"{dataset}.npz"
    with BundleWriter(bundle) as writer:
        lo = 0
        while lo < len(todo):  # runs of consecutive pieces of one sample rate, in the bundle's order
            sr, hi, seconds = todo[lo][2], lo, 0.0
            while hi < len(todo) and todo[hi][2] == sr and hi - lo < batch and (hi == lo or seconds < GROUP_SECONDS):
                frames = todo[hi][1].frames if todo[hi][1] is not None else 0
                seconds += frames / sr
                hi += 1
            group = [(f, info) for f, info, _ in todo[lo:hi]]
            try:
                results = run_group(group, sr)
            except Exception:
                results = []
                for item in group:  # isolate the failure: one piece at a time
                    try:
                        results += run_group([item], sr)
                    except Exception as e:
                        results.append(None)
                        skip(item[0].stem, f"{type(e).__name__}: {e}")
            for (f, _), members in zip(group, results):
                if members is None:
                    continue
                writer.add(f.stem, {name: members[name] for name in names})
                ann_out.mkdir(parents=True, exist_ok=True)
                if not (ann_out / f"{f.stem}.beats").exists():
                    shutil.copyfile(ann_in / f"{f.stem}.beats", ann_out / f"{f.stem}.beats")
                written.append(f.stem)
                if verbose:
                    print(f"{f.stem}: {len(names)} spectrograms")
            lo = hi
    return {"written": written, "skipped": skipped, "bundle": str(bundle), "members": names}


def _ints(value):
    return tuple(map(int, value.split(":"))) if value else None


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m beat_this_b200.prepare", description=__doc__.split("\n\n")[0])
    add = ap.add_argument
    add("--audio", nargs="+", required=True, help="audio files or directories")
    add("--annotations", required=True, help="directory of <stem>.beats files")
    add("--out", required=True, help="dataset directory to write (audio/spectrograms/ and annotations/)")
    add("--dataset", required=True, help="name of the dataset (of the .npz bundle)")
    add("--pitch_shift", metavar="LOW:HIGH", default="-5:6", help="pitch shift in semitones (default: %(default)s)")
    add("--time_stretch", metavar="MAX:STRIDE", default="20:4",
        help="time stretch in percentage and stride (default: %(default)s)")
    add("--aug-sr", type=int, default=44100, help="sample rate the augmentations run at (default: %(default)s)")
    add("--no-augment", action="store_true", help="write the unaugmented track only")
    add("--batch", type=int, default=8, help="pieces per group (default: %(default)s)")
    add("--device", default="cuda")
    add("--verbose", action="store_true")
    a = ap.parse_args(argv)
    res = prepare(a.audio, a.annotations, a.out, a.dataset, _ints(a.pitch_shift), _ints(a.time_stretch), a.aug_sr,
                  not a.no_augment, a.batch, a.device, a.verbose)
    print(f"wrote {len(res['written'])} pieces x {len(res['members'])} spectrograms to {res['bundle']}"
          + (f"; skipped {len(res['skipped'])}" if res["skipped"] else ""))
    return 0 if res["written"] else 1


if __name__ == "__main__":
    sys.exit(main())
