"""Time the log-mel kernels against torchaudio's MelSpectrogram (what the reference's LogMelSpect wraps) on the same
GPU at the same batch.

    python tools/logmel_rates.py [--clips 64] [--secs 30] [--out logmel_rates.json]

Workloads: the reference defaults on both kernels (bt_logmel, and bt_logmel_config through LogMelSpect's test switch),
n_fft 2048 / hop 512 / 44.1 kHz / 128 mels, n_fft 4096 / hop 441 / 22.05 kHz, n_fft 512 / hop 160 / 16 kHz / 80 mels.
Each runs `--clips` clips of `--secs` seconds of noise: ours as one call on the concatenated clips, torchaudio as one
call on the [clips, samples] batch followed by log1p(m x).  CUDA events around `--iters` calls after `--warmup`.
Effective GB/s counts the algorithmic HBM bytes: every input sample read once and every output written once.  The
card's name, power limit and SM clocks are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from beat_this_b200.preprocessing import LogMelSpect  # noqa: E402

WORKLOADS = [
    ("default_fused", {}, False),
    ("default_general", {}, True),
    ("nfft2048_hop512_44k1_128", dict(sample_rate=44100, n_fft=2048, hop_length=512, f_max=None), False),
    ("nfft4096_hop441", dict(n_fft=4096, hop_length=441), False),
    ("nfft512_hop160_16k_80", dict(sample_rate=16000, n_fft=512, hop_length=160, n_mels=80, f_min=0, f_max=None), False),
]


def time_ms(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main(argv=None):
    import torchaudio

    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--secs", type=float, default=30.0)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("logmel_rates needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "clips": args.clips, "secs": args.secs}
    gen = torch.Generator(device=dev).manual_seed(0)
    for name, kw, general in WORKLOADS:
        mel = LogMelSpect(**kw, device=dev, _general=general)
        p = dict(zip(("sample_rate", "n_fft", "hop_length", "f_min", "f_max", "n_mels", "mel_scale", "normalized", "power",
                      "log_multiplier"), LogMelSpect.DEFAULTS))
        p.update(kw)
        n = int(args.secs * p["sample_rate"])
        audio = torch.randn(args.clips, n, device=dev, generator=gen) * 0.1
        flat = audio.reshape(-1).contiguous()
        so = [i * n for i in range(args.clips + 1)]
        eng = mel.engine
        if mel.tables is None:
            ours = lambda: eng.logmel_cat(flat, so)  # noqa: E731
        else:
            ours = lambda: eng.logmel_config_cat(flat, so, mel.tables, mel.device_tables)  # noqa: E731
        ta = torchaudio.transforms.MelSpectrogram(
            sample_rate=p["sample_rate"], n_fft=p["n_fft"], hop_length=p["hop_length"], f_min=p["f_min"], f_max=p["f_max"],
            n_mels=p["n_mels"], mel_scale=p["mel_scale"], normalized=p["normalized"], power=p["power"]).to(dev)
        ref = lambda: torch.log1p(p["log_multiplier"] * ta(audio).transpose(-1, -2))  # noqa: E731
        frames = args.clips * (1 + n // p["hop_length"])
        nbytes = 4 * args.clips * n + 4 * frames * p["n_mels"]
        with torch.no_grad():
            t_ours = time_ms(ours, args.warmup, args.iters)
            t_ref = time_ms(ref, args.warmup, args.iters)
            diff = float((ours()[0].reshape(args.clips, -1, p["n_mels"]) - ref()).abs().max())
        res[name] = {
            "ms": round(t_ours, 4), "torchaudio_ms": round(t_ref, 4), "speedup": round(t_ref / t_ours, 2),
            "frames_per_s": round(frames / t_ours * 1e3), "torchaudio_frames_per_s": round(frames / t_ref * 1e3),
            "effective_GBps": round(nbytes / t_ours / 1e6, 1), "max_abs_diff_vs_torchaudio": diff,
        }
        print(name, json.dumps(res[name]), flush=True)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
