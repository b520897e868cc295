"""Rates of native FLAC input (bt_flac_decode) against WAV on a seeded corpus.

    python tools/flac_rates.py [--clips 64] [--distinct 8] [--seconds 30] [--rounds 5] [--out flac_rates.json]

The corpus: `--clips` stereo 16-bit 44.1 kHz files of `--seconds` s, encoded by the test encoder (tests/flac_reference.py)
at typical settings -- block size 4096, mid/side, LPC order 12 with 15-bit coefficients, partition order 6 -- with WAV
twins of the same samples.  The encoder is numpy and slow, so `--distinct` clips are generated from the seed and the
corpus repeats them under other names: the device does the same work for every copy.  Reported in one run:
* the decode kernels' time for the whole corpus as one group (CUDA events around `--launches` bt_flac_decode calls
  into mono fp32, after a warm-up), with decoded samples/s (per channel) and compressed bytes/s;
* File2Beats.batch clips/s on the FLAC files and on the WAV twins (host clock around a call that ends in results on
  the host), alternated over `--rounds` rounds after one warm-up call of each;
* the card's name and power limit.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import flac_reference as F  # noqa: E402
from beat_this_b200 import _lib, synthetic  # noqa: E402


def corpus(d: Path, clips: int, distinct: int, seconds: float):
    style = F.FrameStyle(assignment="mid_side", subframes=F.Subframe(kind="lpc", order=12, precision=15, porder=6))
    made = []
    for k in range(distinct):
        x = synthetic.synth_clip(500 + k, seconds, sr=44100)
        y = synthetic.synth_clip(900 + k, seconds, sr=44100)
        v = np.clip(np.round(np.stack([0.7 * x + 0.3 * y, 0.3 * x + 0.7 * y], axis=1) * 32767), -32768, 32767)
        made.append((F.encode(v.astype(np.int64), 44100, 16, 4096, style).data, F.wav_twin(v, 44100, 16)))
    flacs, wavs = [], []
    for i in range(clips):
        fl, wv = made[i % distinct]
        flacs.append(d / f"c{i:03d}.flac")
        flacs[-1].write_bytes(fl)
        wavs.append(d / f"c{i:03d}.wav")
        wavs[-1].write_bytes(wv)
    return flacs, wavs


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # the numbers still stand with the device name torch reports
        return torch.cuda.get_device_name(0), f"unknown ({type(e).__name__})"


def decode_time(paths, launches: int):
    from beat_this_b200.engine import Engine

    probed = _lib.probe_audio(paths)
    infos = [info for _, info in probed]
    fo, status_at, bo, total = _lib.flac_layout(infos)
    host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    nf, ns, status = _lib.stage_flac_files(paths, infos, host.data_ptr(), 0)
    assert not any(status)
    dev = torch.device("cuda:0")
    buf = host.to(dev)
    so = _lib.offsets(ns)
    out = torch.empty(so[-1], dtype=torch.float32, device=dev)
    eng = Engine.mel_only(dev)
    streams = _lib.flac_streams(infos, nf, ns, so[:-1])
    for _ in range(3):
        eng.flac_decode(buf, streams, _lib.BT_FLAC_MONO_F32, out, status_at)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        eng.flac_decode(buf, streams, _lib.BT_FLAC_MONO_F32, out, status_at)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / launches
    lib = _lib.load()  # the split between the two kernels, from the library's per-kernel profile
    lib.bt_profile_enable(eng.ctx, 1)
    lib.bt_profile_reset(eng.ctx)
    for _ in range(launches):
        eng.flac_decode(buf, streams, _lib.BT_FLAC_MONO_F32, out, status_at)
    torch.cuda.synchronize()
    lib.bt_profile_collect(eng.ctx)
    kernels = {}
    name, kms, cnt = ctypes.create_string_buffer(64), ctypes.c_double(), ctypes.c_int64()
    for i in range(lib.bt_profile_count(eng.ctx)):
        lib.bt_profile_get(eng.ctx, i, name, 64, ctypes.byref(kms), ctypes.byref(cnt))
        kernels[name.value.decode()] = kms.value / max(cnt.value, 1)
    lib.bt_profile_enable(eng.ctx, 0)
    samples = sum(ns)
    comp = sum(info.frames_bytes for info in infos)
    return {"group_ms": ms, "kernel_ms": kernels, "samples": samples, "channel_samples": samples * 2, "compressed_bytes": comp,
            "samples_per_s": samples / (ms / 1e3), "compressed_bytes_per_s": comp / (ms / 1e3)}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--model", default="final0")
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("flac_rates measures on a CUDA device; none is present")
    from beat_this_b200.inference import File2Beats

    with tempfile.TemporaryDirectory() as td:
        t0 = time.perf_counter()
        flacs, wavs = corpus(Path(td), a.clips, a.distinct, a.seconds)
        res = {"corpus_s": time.perf_counter() - t0, "clips": a.clips, "distinct": a.distinct, "seconds": a.seconds}
        res["decode"] = decode_time([str(p) for p in flacs], a.launches)
        ckpt = synthetic.write_checkpoint(os.path.join(td, f"{a.model}.ckpt"), a.model, 0)
        f2b = File2Beats(ckpt, "cuda:0", float16=True)
        f2b.batch(flacs)
        f2b.batch(wavs)
        rates = {"flac": [], "wav": []}
        for _ in range(a.rounds):
            for kind, files in (("flac", flacs), ("wav", wavs)):
                t = time.perf_counter()
                f2b.batch(files)
                rates[kind].append(len(files) / (time.perf_counter() - t))
        res["clips_per_s"] = rates
        res["flac_over_wav"] = float(np.median(rates["flac"]) / np.median(rates["wav"]))
        res["card"], res["power_limit"] = card()
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
