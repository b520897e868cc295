#!/usr/bin/env python3
"""``beat_this`` command line tool on the H100 engine (reference beat_this/cli.py:22-191: same options, same
output naming, same ``.beats`` / ``.npy`` files), re-organised around the batched device path: the work list is
built first, then ``--batch`` files at a time are claimed and handed to ``File2Beats.batch`` (native WAV, FLAC, MP3 and Ogg
Vorbis decode: host threads -> pinned ring -> device, groups of one sample rate share launches, decode of the next group overlaps
the kernels of the current one); under ``torchrun`` every rank takes every WORLD_SIZE-th task (tasks are
independent: no collective).  A file that fails costs only itself, and its --touch-first placeholder is removed.

    python -m beat_this_b200.cli song.wav                     # -> song.beats
    python -m beat_this_b200.cli music_dir -o out --float16    # directory tree -> out/.../*.beats
    torchrun --nproc-per-node 8 -m beat_this_b200.cli music_dir -o out --skip-existing --touch-first
"""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import numpy as np

from .utils import save_beat_tsv


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="beat_this_b200", description="Beat and downbeat times for audio files (Beat This! model on the H100 engine).")
    add = ap.add_argument
    add("inputs", nargs="+", help="audio files and/or directories that are searched recursively")
    add("--model", default="final0", help="checkpoint name or path [%(default)s]")
    add("--output", "-o", default=None, help="result file (one input file) or result directory; default: next to each input")
    add("--suffix", "-s", default=".beats", help="extension of the result files [%(default)s]")
    add("--append", action="store_true", help="keep the audio extension and add the suffix after it")
    add("--skip-existing", action="store_true", help="leave results that already exist untouched")
    add("--touch-first", action="store_true", help="create the (empty) result file before working on it: with --skip-existing, "
                                                   "several processes can split one directory between them")
    add("--dbn", default=False, action=argparse.BooleanOptionalAction, help="DBN post-processing instead of peak picking")
    add("--dbn-impl", default="auto", choices=["auto", "madmom", "native", "device"],
        help="DBN decoder: madmom if installed else the host C++ tracker (auto), madmom, the host C++ tracker (native) "
             "or the same tracker on the GPU (device) [%(default)s]")
    add("--gpu", type=int, default=None, help="CUDA device index [LOCAL_RANK or 0]; a GPU is required")
    add("--float16", action="store_true", help="fp16 tensor-core kernels (fast path) instead of fp32")
    add("--activations", action="store_true", help="also write the frame activations as <result>.npy (2 x frames)")
    add("--batch", type=int, default=256, help="files claimed and queued at a time [%(default)s]; the device works on groups of up to 64 clips")
    return ap


def output_path_for(src: Path, suffix: str, append: bool, out_dir: Path | None = None, root: Path | None = None) -> Path:
    """Where the result of `src` goes: next to it, or under `out_dir` keeping the path relative to the directory
    `root` that was named on the command line; the suffix replaces the old one unless `append`."""
    if out_dir is None:
        dst = src
    else:
        dst = out_dir / (src.relative_to(root) if root is not None else src.name)
    return dst.parent / (dst.name + suffix) if append else dst.with_suffix(suffix)


def collect_tasks(inputs, output, suffix, append, skip_existing):
    """[(audio file, output file)] for the command line; a single plain file may name its output file directly."""
    inputs = [Path(p) for p in inputs]
    output = Path(output) if output is not None else None
    if len(inputs) == 1 and not inputs[0].is_dir():
        dst = output
        if dst is None or dst.is_dir():
            dst = output_path_for(inputs[0], suffix, append, dst)
        return [(inputs[0], dst)], True
    tasks = []
    for item in inputs:
        if item.is_dir():
            for fn in sorted(item.rglob("*")):
                if fn.is_dir() or fn.name.endswith(suffix):
                    continue
                dst = output_path_for(fn, suffix, append, output, root=item)
                if not skip_existing or not dst.exists():
                    tasks.append((fn, dst))
        else:
            tasks.append((item, output_path_for(item, suffix, append, output)))
    return tasks, False


def _claim(dst: Path, skip_existing: bool, touch_first: bool) -> bool:
    """Reference cli.py:171-177: with --touch-first the empty output file is the lock."""
    if touch_first:
        try:
            dst.parent.mkdir(parents=True, exist_ok=True)
            dst.touch(exist_ok=not skip_existing)
        except FileExistsError:
            return False
        return True
    return not (skip_existing and dst.exists())


def _release(dst: Path, touch_first: bool) -> None:
    """A file we claimed with --touch-first but could not process: remove the empty placeholder again, otherwise a
    rerun with --skip-existing would silently skip it."""
    if touch_first:
        try:
            if dst.exists() and dst.stat().st_size == 0:
                dst.unlink()
        except OSError:
            pass


def run(inputs, model="final0", output=None, suffix=".beats", append=False, skip_existing=False, touch_first=False,
        dbn=False, gpu=None, float16=False, activations=False, batch=256, dbn_impl="auto") -> int:
    from .inference import File2Beats
    from .preprocessing import load_audio

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    if gpu is None:
        gpu = int(os.environ.get("LOCAL_RANK", "0"))
    if gpu < 0:
        raise SystemExit("beat_this_b200 has no CPU path: --gpu must name a CUDA device")
    tasks, single = collect_tasks(inputs, output, suffix, append, skip_existing)
    tasks = tasks[rank::world]
    f2b = File2Beats(model, f"cuda:{gpu}", float16, dbn, dbn_impl=dbn_impl)
    failed = 0

    def fail(src, dst, why=""):
        nonlocal failed
        failed += 1
        _release(dst, touch_first)
        print(f'Could not process "{src}"{why}. Rerun with this file alone for details.', file=sys.stderr)

    step = max(1, batch)
    for b0 in range(0, len(tasks), step):
        # claim right before working on a slice, so that several processes can share one directory (cli.py:178-184)
        group = [(src, dst) for src, dst in tasks[b0 : b0 + step] if single or _claim(dst, skip_existing, touch_first)]
        if not group:
            continue
        if single:  # one file: let errors surface, as the reference does for its single-file case
            src, dst = group[0]
            if activations:
                wav, sr = load_audio(src)
                beat, down = f2b.spect2frames(f2b.signal2spect(wav, sr))
                dst.parent.mkdir(parents=True, exist_ok=True)
                np.save(dst.with_suffix(".npy"), np.vstack([beat.cpu().numpy(), down.cpu().numpy()]))
                beats, downbeats = f2b.frames2beats(beat, down)
            else:
                beats, downbeats = f2b(src)
            save_beat_tsv(beats, downbeats, dst)
            continue
        if activations:  # logits wanted on the host as well: one file at a time through the three public stages
            for src, dst in group:
                try:
                    wav, sr = load_audio(src)
                    beat, down = f2b.spect2frames(f2b.signal2spect(wav, sr))
                    dst.parent.mkdir(parents=True, exist_ok=True)
                    np.save(dst.with_suffix(".npy"), np.vstack([beat.cpu().numpy(), down.cpu().numpy()]))
                    save_beat_tsv(*f2b.frames2beats(beat, down), dst)
                except Exception:
                    fail(src, dst)
            continue
        # a failure inside a device batch costs only the file that caused it: File2Beats.batch(on_error="skip")
        # retries the files of a failed batch one by one and reports None for the ones that really fail
        results = f2b.batch([src for src, _ in group], on_error="skip")
        for (src, dst), res in zip(group, results):
            if res is None:
                fail(src, dst)
                continue
            try:
                save_beat_tsv(res[0], res[1], dst)
            except Exception:
                fail(src, dst, " (writing the result failed)")
    return 1 if failed else 0


def main(argv=None) -> int:
    return run(**vars(build_parser().parse_args(argv)))


if __name__ == "__main__":
    sys.exit(main())
