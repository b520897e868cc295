"""Rates of training-batch assembly (beat_this_b200.dataset.TrainingBatches, bt_train_batch) on a seeded synthetic
dataset.

    python tools/batch_rates.py [--pieces 200] [--out batch_rates.json]

The dataset: `--pieces` pieces of 30 s to 5 min at 50 fps in one float16 bundle in a temporary directory (track, one
pitch and two tempo variants per piece; just written, so in the page cache as a dataset trained on for a while would
be), with pitch, tempo and permute-mask augmentation.  For B = 8 and 64 at L = 1500 it reports:
* batches/s of iterating TrainingBatches (host clock around `--batches` batches after `--warmup`, ending in a
  device synchronise; the consumer does nothing);
* host staging per batch: the draws, and the window copies into pinned memory (host clock, medians);
* H2D per batch: CUDA events around the copy of one batch's windows from pinned memory;
* the bt_train_batch call: library profile over `--launches` launches after warm-up (the gap between launches, which
  also holds the upload of the tables and any wait for the host), and the kernel's median duration from a
  torch.profiler trace of 50 launches, with the bytes it must move (windows read, spectrogram and three byte targets
  written) over that duration, against 3.35 TB/s.
The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from beat_this_b200 import dataset as D  # noqa: E402

AUG = {"pitch": {"min": 0, "max": 1}, "tempo": {"min": -4, "max": 4, "stride": 8},
       "mask": {"kind": "permute", "min_count": 1, "max_count": 6, "min_len": 0.1, "max_len": 2.0, "min_parts": 5,
                "max_parts": 9}}
HBM_BYTES_PER_S = 3.35e12


def write_dataset(root: Path, pieces: int, seed: int = 0):
    """One float16 bundle (the layout prepare writes and the paper's data uses), every member a distinct slice of a
    random pool."""
    from beat_this_b200.prepare import BundleWriter

    rng = np.random.default_rng(seed)
    pool = rng.standard_normal((300 * 50 + 5000, 128), dtype=np.float32).astype(np.float16)
    ann = root / "annotations" / "synth"
    (ann / "annotations" / "beats").mkdir(parents=True)
    (ann / "info.json").write_text(json.dumps({"has_downbeats": True}))
    names = []
    with BundleWriter(root / "audio" / "spectrograms" / "synth.npz") as w:
        for i in range(pieces):
            stem = f"p{i:04d}"
            T = int(rng.integers(30 * 50, 300 * 50 + 1))
            w.add(stem, {v[:-4]: pool[(o := int(rng.integers(0, 5000))) : o + T]
                         for v in D.precomputed_augmentation_filenames(AUG)})
            t = np.arange(0.2, T / 50, 0.5)
            (ann / "annotations" / "beats" / f"{stem}.beats").write_text(
                "".join(f"{a:.3f}\t{1 + k % 4}\n" for k, a in enumerate(t)))
            names.append(f"synth/{stem}")
    return names


def profiled_ms(lib, ctx, name):
    for i in range(lib.bt_profile_count(ctx)):
        buf = ctypes.create_string_buffer(64)
        ms, n = ctypes.c_double(), ctypes.c_int64()
        lib.bt_profile_get(ctx, i, buf, 64, ctypes.byref(ms), ctypes.byref(n))
        if buf.value.decode() == name:
            return ms.value, n.value
    return 0.0, 0


def measure(ds, B, args):
    tb = D.TrainingBatches(ds, batch_size=B, seed=0, device="cuda:0")
    res = {}

    def epochs():
        while True:
            yield from tb

    it = epochs()
    for _ in range(args.warmup):
        next(it)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.batches):
        next(it)
    torch.cuda.synchronize()
    res["batches_per_s"] = args.batches / (time.perf_counter() - t0)
    # host staging: draws and window copies of one batch (a fresh instance: the iterator above holds a staged batch)
    tb = D.TrainingBatches(ds, batch_size=B, seed=0, device="cuda:0")
    order = list(range(len(ds)))
    draws, host = [], []
    for k in range(args.batches):
        idx = order[(k * B) % (len(ds) - B) :][:B]
        t0 = time.perf_counter()
        [ds.draw(i) for i in idx]
        draws.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        s = tb._stage(idx)
        for f in s.copies:
            f.result()
        host.append(time.perf_counter() - t0)
        tb._launch(s)
    torch.cuda.synchronize()
    res["host_draws_ms_median"] = 1e3 * float(np.median(draws))
    res["host_stage_ms_median"] = 1e3 * float(np.median(host))
    rows = int(s.rows[-1])
    res["window_rows_last"] = rows
    # H2D of one batch's windows
    src = tb._host[s.slot][: rows * 128]
    dst = torch.empty(rows * 128, dtype=torch.int16, device="cuda:0")
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(5):
        dst.copy_(src, non_blocking=True)
    a.record()
    for _ in range(args.batches):
        dst.copy_(src, non_blocking=True)
    b.record()
    torch.cuda.synchronize()
    res["h2d_ms"] = a.elapsed_time(b) / args.batches
    res["h2d_GB_per_s"] = rows * 256 / (res["h2d_ms"] * 1e-3) / 1e9
    # the kernel alone, on the last batch's tables
    ex = s.excerpts
    L = s.length
    maps = np.concatenate([e.row_map for e in ex])
    boff = np.concatenate(([0], np.cumsum([len(e.beat_frames) for e in ex]))).astype(np.int64)
    doff = np.concatenate(([0], np.cumsum([len(e.downbeat_frames) for e in ex]))).astype(np.int64)
    beats = np.concatenate([e.beat_frames for e in ex])
    downs = np.concatenate([e.downbeat_frames for e in ex])
    spect = torch.empty((B, L, 128), dtype=torch.float16, device="cuda:0")
    outs = [torch.empty((B, L), dtype=torch.bool, device="cuda:0") for _ in range(3)]
    eng = tb.engine
    call = lambda: eng.train_batch(dst, s.rows, L, maps, beats, boff, downs, doff, spect, *outs)  # noqa: E731
    for _ in range(20):
        call()
    torch.cuda.synchronize()
    eng.lib.bt_profile_enable(eng.ctx, 1)
    eng.lib.bt_profile_reset(eng.ctx)
    for _ in range(args.launches):
        call()
    eng.lib.bt_profile_collect(eng.ctx)
    ms, n = profiled_ms(eng.lib, eng.ctx, "train_batch")
    eng.lib.bt_profile_enable(eng.ctx, 0)
    # the kernel's own duration from a trace (the profile's gap between launches also holds the tables' upload and
    # any wait for the host)
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            call()
        torch.cuda.synchronize()
    durs = [e.device_time for e in prof.events() if "train_batch_kernel" in e.name]
    traced_ms = 1e-3 * float(np.median(durs)) if durs else float("nan")
    moved = rows * 256 + B * L * 256 + 3 * B * L
    res.update(profile_us=1e3 * ms / max(n, 1), profile_launches=n, kernel_traced_us=1e3 * traced_ms,
               kernel_traced_launches=len(durs), kernel_bytes=moved, kernel_GB_per_s=moved / (traced_ms * 1e-3) / 1e9,
               kernel_share_of_hbm=moved / (traced_ms * 1e-3) / HBM_BYTES_PER_S)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--pieces", type=int, default=200)
    ap.add_argument("--batches", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("batch_rates needs a CUDA device")
    res = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip()}
    with tempfile.TemporaryDirectory() as tmp:
        root = Path(tmp)
        names = write_dataset(root, args.pieces)
        ds = D.BeatTrackingDataset(names, root, train_length=1500, augmentations=AUG)
        res["pieces"] = len(ds)
        res["frames"] = int(sum(ds.get_frame_count(i) for i in range(len(ds))))
        for B in (8, 64):
            res[f"B{B}"] = measure(ds, B, args)
            print(json.dumps({f"B{B}": res[f"B{B}"]}), flush=True)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
