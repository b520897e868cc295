"""Rates of native MP3 input (bt_mp3_decode) against WAV.

    python tools/mp3_rates.py [--clips 64] [--rounds 5] [--out mp3_rates.json]

The corpus: `--clips` files of about 30 s, each the 383 frames of tests/golden/kings_of_swing_383.mp3 (320 kbit/s CBR,
44.1 kHz joint stereo) written three times over -- valid streams, since main_data_begin is 0 in every frame -- and WAV
twins holding the decoded samples (16-bit PCM WAV of the channels decode).  Reported in one run:
* the decode kernels' time for the whole corpus as one group (CUDA events around `--launches` bt_mp3_decode calls
  into mono fp32, after a warm-up), per kernel from the library's profile, with decoded samples/s (per channel) and
  compressed bytes/s;
* File2Beats.batch clips/s on the MP3 files and on the WAV twins (host clock around a call that ends in results on
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

from beat_this_b200 import _lib, synthetic  # noqa: E402


def corpus(d: Path, clips: int):
    import wave

    fixture = open(os.path.join(ROOT, "tests", "golden", "kings_of_swing_383.mp3"), "rb").read()
    one = d / "one.mp3"
    one.write_bytes(fixture * 3)
    from beat_this_b200.preprocessing import load_audio

    x, sr = load_audio(one)  # float64 [time, 2] of the device decode
    pcm = np.clip(np.round(x * 32767), -32768, 32767).astype("<i2").tobytes()
    mp3s, wavs = [], []
    for i in range(clips):
        mp3s.append(d / f"c{i:03d}.mp3")
        mp3s[-1].write_bytes(fixture * 3)
        wavs.append(d / f"c{i:03d}.wav")
        with wave.open(str(wavs[-1]), "wb") as w:
            w.setnchannels(2)
            w.setsampwidth(2)
            w.setframerate(sr)
            w.writeframes(pcm)
    return mp3s, wavs


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
    fo, status_at, bo, total = _lib.mp3_layout(infos)
    host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    nf, mb, status = _lib.stage_mp3_files(paths, infos, host.data_ptr(), 0)
    assert not any(status)
    dev = torch.device("cuda:0")
    buf = host.to(dev)
    ns = [info.n_samples for info in infos]
    so = _lib.offsets(ns)
    out = torch.empty(so[-1], dtype=torch.float32, device=dev)
    eng = Engine.mel_only(dev)
    streams = _lib.mp3_streams(infos, nf, mb, so[:-1])
    for _ in range(3):
        eng.mp3_decode(buf, streams, _lib.BT_MP3_MONO_F32, out, status_at)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        eng.mp3_decode(buf, streams, _lib.BT_MP3_MONO_F32, out, status_at)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / launches
    lib = _lib.load()  # the split between the three kernels, from the library's per-kernel profile
    lib.bt_profile_enable(eng.ctx, 1)
    lib.bt_profile_reset(eng.ctx)
    for _ in range(launches):
        eng.mp3_decode(buf, streams, _lib.BT_MP3_MONO_F32, out, status_at)
    torch.cuda.synchronize()
    lib.bt_profile_collect(eng.ctx)
    kernels = {}
    name, kms, cnt = ctypes.create_string_buffer(64), ctypes.c_double(), ctypes.c_int64()
    for i in range(lib.bt_profile_count(eng.ctx)):
        lib.bt_profile_get(eng.ctx, i, name, 64, ctypes.byref(kms), ctypes.byref(cnt))
        kernels[name.value.decode()] = kms.value / max(cnt.value, 1)
    lib.bt_profile_enable(eng.ctx, 0)
    samples = sum(ns)
    comp = total  # bytes that cross to the device: frame tables, statuses and main data
    return {"group_ms": ms, "kernel_ms": kernels, "samples": samples, "channel_samples": samples * 2, "compressed_bytes": comp,
            "samples_per_s": samples / (ms / 1e3), "compressed_bytes_per_s": comp / (ms / 1e3)}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--model", default="final0")
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("mp3_rates measures on a CUDA device; none is present")
    from beat_this_b200.inference import File2Beats

    with tempfile.TemporaryDirectory() as td:
        t0 = time.perf_counter()
        mp3s, wavs = corpus(Path(td), a.clips)
        res = {"corpus_s": time.perf_counter() - t0, "clips": a.clips, "seconds": 3 * 383 * 1152 / 44100}
        res["decode"] = decode_time([str(p) for p in mp3s], a.launches)
        ckpt = synthetic.write_checkpoint(os.path.join(td, f"{a.model}.ckpt"), a.model, 0)
        f2b = File2Beats(ckpt, "cuda:0", float16=True)
        f2b.batch(mp3s)
        f2b.batch(wavs)
        rates = {"mp3": [], "wav": []}
        for _ in range(a.rounds):
            for kind, files in (("mp3", mp3s), ("wav", wavs)):
                t = time.perf_counter()
                f2b.batch(files)
                rates[kind].append(len(files) / (time.perf_counter() - t))
        res["clips_per_s"] = rates
        res["mp3_over_wav"] = float(np.median(rates["mp3"]) / np.median(rates["wav"]))
        res["spread"] = {k: [float(min(v)), float(max(v))] for k, v in rates.items()}
        res["card"], res["power_limit"] = card()
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
