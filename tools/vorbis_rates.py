"""Rates of native Ogg Vorbis input (bt_vorbis_decode) against WAV.

    python tools/vorbis_rates.py [--clips 64] [--rounds 5] [--out vorbis_rates.json]

The corpus: `--clips` copies of one 30 s stereo 44.1 kHz stream from the test encoder (tests/vorbis_reference.py) with
a setup in the manner of libvorbis's: blocks 256 / 2048, floor1, square-polar coupling and residue 2, a block sequence
with every window transition; and WAV twins holding the decoded samples (16-bit PCM WAV of the channels decode).
Reported in one run:
* the decode kernels' time for the whole corpus as one group (CUDA events around `--launches` bt_vorbis_decode calls
  into mono fp32, after a warm-up), per kernel from the library's profile, with decoded samples/s (per channel) and
  compressed bytes/s;
* File2Beats.batch clips/s on the Ogg Vorbis files and on the WAV twins (host clock around a call that ends in results
  on the host), alternated over `--rounds` rounds after one warm-up call of each;
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

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import vorbis_reference as V

    rng = np.random.default_rng(0)
    n = 30 * 44100
    t = np.arange(n) / 44100
    base = np.sin(2 * np.pi * 220 * t) * (1 + np.sin(2 * np.pi * 2 * t)) + 0.2 * rng.standard_normal(n)
    sig = 0.15 * np.stack([base, 0.7 * base + 0.2 * rng.standard_normal(n)], axis=1)
    flags = [1 if (k // 7) % 5 else 0 for k in range(n // 1024 * 2)]
    flags = flags[: next(k for k in range(len(flags)) if V.ends_of(flags[:k + 1], (256, 2048))[1][-1] >= n) + 2]
    fixture = V.encode(sig, V.Plan(V.standard_setup(), flags, page_bytes=4096))
    one = d / "one.ogg"
    one.write_bytes(fixture)
    from beat_this_b200.preprocessing import load_audio

    x, sr = load_audio(one)  # float64 [time, 2] of the device decode
    pcm = np.clip(np.round(x * 32767), -32768, 32767).astype("<i2").tobytes()
    oggs, wavs = [], []
    for i in range(clips):
        oggs.append(d / f"c{i:03d}.ogg")
        oggs[-1].write_bytes(fixture)
        wavs.append(d / f"c{i:03d}.wav")
        with wave.open(str(wavs[-1]), "wb") as w:
            w.setnchannels(2)
            w.setsampwidth(2)
            w.setframerate(sr)
            w.writeframes(pcm)
    return oggs, wavs


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
    fo, status_at, bo, total = _lib.vorbis_layout(infos)
    host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    npk, pb, bs, status = _lib.stage_vorbis_files(paths, infos, host.data_ptr(), 0)
    assert not any(status)
    dev = torch.device("cuda:0")
    buf = host.to(dev)
    ns = [info.n_samples for info in infos]
    so = _lib.offsets(ns)
    out = torch.empty(so[-1], dtype=torch.float32, device=dev)
    eng = Engine.mel_only(dev)
    streams = _lib.vorbis_streams(infos, npk, pb, bs, so[:-1])
    for _ in range(3):
        eng.vorbis_decode(buf, streams, _lib.BT_VORBIS_MONO_F32, out, status_at)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        eng.vorbis_decode(buf, streams, _lib.BT_VORBIS_MONO_F32, out, status_at)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / launches
    lib = _lib.load()  # the split between the three kernels, from the library's per-kernel profile
    lib.bt_profile_enable(eng.ctx, 1)
    lib.bt_profile_reset(eng.ctx)
    for _ in range(launches):
        eng.vorbis_decode(buf, streams, _lib.BT_VORBIS_MONO_F32, out, status_at)
    torch.cuda.synchronize()
    lib.bt_profile_collect(eng.ctx)
    kernels = {}
    name, kms, cnt = ctypes.create_string_buffer(64), ctypes.c_double(), ctypes.c_int64()
    for i in range(lib.bt_profile_count(eng.ctx)):
        lib.bt_profile_get(eng.ctx, i, name, 64, ctypes.byref(kms), ctypes.byref(cnt))
        kernels[name.value.decode()] = kms.value / max(cnt.value, 1)
    lib.bt_profile_enable(eng.ctx, 0)
    samples = sum(ns)
    comp = total  # bytes that cross to the device: packet tables, statuses, packets and decode tables
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
        raise SystemExit("vorbis_rates measures on a CUDA device; none is present")
    from beat_this_b200.inference import File2Beats

    with tempfile.TemporaryDirectory() as td:
        t0 = time.perf_counter()
        oggs, wavs = corpus(Path(td), a.clips)
        res = {"corpus_s": time.perf_counter() - t0, "clips": a.clips, "seconds": 30.0}
        res["decode"] = decode_time([str(p) for p in oggs], a.launches)
        ckpt = synthetic.write_checkpoint(os.path.join(td, f"{a.model}.ckpt"), a.model, 0)
        f2b = File2Beats(ckpt, "cuda:0", float16=True)
        f2b.batch(oggs)
        f2b.batch(wavs)
        rates = {"vorbis": [], "wav": []}
        for _ in range(a.rounds):
            for kind, files in (("vorbis", oggs), ("wav", wavs)):
                t = time.perf_counter()
                f2b.batch(files)
                rates[kind].append(len(files) / (time.perf_counter() - t))
        res["clips_per_s"] = rates
        res["vorbis_over_wav"] = float(np.median(rates["vorbis"]) / np.median(rates["wav"]))
        res["spread"] = {k: [float(min(v)), float(max(v))] for k, v in rates.items()}
        res["card"], res["power_limit"] = card()
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
