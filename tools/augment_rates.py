"""Time the augmentation path: `--clips` clips of `--seconds` s of noise at 44.1 kHz, n_fft 2048, hop 512, the 21
variants of the reference defaults (pitch -5..6, tempo +-20 % in steps of 4).

    python tools/augment_rates.py [--clips 64] [--out augment_rates.json]

Reports, with the card's name, power limit and SM clocks read in the same run:
* ms per kernel class of one `Augmenter.batch` (the ctx's launch profile: CUDA events around every launch), and
  clips/s through it and through the resample to 22.05 kHz + log-mel that `prepare` adds (host wall clock around a
  device synchronise, three rounds);
* the vocoder alone on one group, variants listed clip-major (a clip's variants adjacent, sharing its analysis in L2)
  against variant-major, alternating, CUDA events over `--iters` calls; effective GB/s counting each analysis value
  once per variant (pessimistic) and once per clip (optimistic), plus the output once;
* the same variants through torchaudio.functional.phase_vocoder + torch.istft on this GPU and on the host's cores.
A run without a CUDA device fails.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from beat_this_b200.augment import Augmenter, stretched_length  # noqa: E402
from beat_this_b200.preprocessing import LogMelSpect  # noqa: E402

SR, N_FFT, HOP = 44100, 2048, 512


def events_ms(fn, warmup, iters):
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


def torchaudio_variants(x, rates, device):
    import torchaudio

    x = x.to(device)
    w = torch.hann_window(N_FFT, device=device)
    X = torch.stft(x, N_FFT, HOP, N_FFT, w, return_complex=True)
    adv = torch.linspace(0, math.pi * HOP, N_FFT // 2 + 1, device=device)[..., None]
    out = []
    for r in rates:
        Y = torchaudio.functional.phase_vocoder(X, r, adv)
        out.append(torch.istft(Y, N_FFT, HOP, N_FFT, w, length=stretched_length(x.shape[-1], r)))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("augment_rates needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                                  "--format=csv,noheader"], capture_output=True, text=True).stdout.strip(),
           "clips": args.clips, "seconds": args.seconds}
    n = int(args.seconds * SR)
    gen = torch.Generator(device="cpu").manual_seed(0)
    clips = [(torch.randn(n, generator=gen) * 0.1).to(dev) for _ in range(args.clips)]
    aug = Augmenter(SR, device=dev)
    eng = aug.engine
    logmel = LogMelSpect(_engine=None, device=dev)
    rates = [r for _, r, _ in aug.variants]
    res["variants"] = len(rates)
    res["clip_bytes"] = aug.clip_bytes(n, rates)

    def batch():
        return aug.batch(clips)

    def batch_to_spectrograms():
        for per_clip in aug.batch(clips):
            parts = list(per_clip.values())
            po = np.concatenate([[0], np.cumsum([p.numel() for p in parts])]).tolist()
            audio, so = eng.resample_cat(torch.cat(parts), po, SR, 22050)
            logmel.batch([audio[so[i] : so[i + 1]] for i in range(len(parts))])

    batch()  # builds the eleven resampling banks, grows the scratch
    torch.cuda.synchronize()
    eng.profile_enable(True)
    eng.profile_reset()
    batch()
    torch.cuda.synchronize()
    res["kernel_ms_per_batch"] = {k: round(ms, 3) for k, (ms, _) in eng.profile_results().items()}
    res["kernel_launches_per_batch"] = {k: c for k, (_, c) in eng.profile_results().items()}
    eng.profile_enable(False)
    rounds = {"augmenter": [], "augmenter_resample_logmel": []}
    batch_to_spectrograms()
    for _ in range(3):  # alternating rounds
        for name, fn in (("augmenter", batch), ("augmenter_resample_logmel", batch_to_spectrograms)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            rounds[name].append(args.clips / (time.perf_counter() - t0))
    res["clips_per_s"] = {k: [round(v, 2) for v in vs] for k, vs in rounds.items()}

    # the vocoder alone, one group of 4 clips: clip-major against variant-major order of the variant table
    g = min(4, args.clips)
    so = [i * n for i in range(g + 1)]
    spec, fo = eng.stft_cat(torch.cat(clips[:g]), so, aug.tables)
    orders = {"clip_major": ([c for c in range(g) for _ in rates], [r for _ in range(g) for r in rates]),
              "variant_major": ([c for _ in rates for c in range(g)], [r for r in rates for _ in range(g)])}
    voc = {k: [] for k in orders}
    for _ in range(3):
        for k, (vc, vr) in orders.items():
            voc[k].append(events_ms(lambda: eng.phase_vocoder_cat(spec, fo, vc, vr), 2, args.iters))
    T = fo[1]
    out_frames = sum(math.ceil(T / r) for r in rates) * g
    bins = N_FFT // 2 + 1
    res["vocoder_ms"] = {k: [round(v, 3) for v in vs] for k, vs in voc.items()}
    best = min(voc["clip_major"])
    res["vocoder_GBps_clip_major"] = {
        "analysis_once_per_variant": round(8 * bins * (T * g * len(rates) + out_frames) / best / 1e6, 1),
        "analysis_once_per_clip": round(8 * bins * (T * g + out_frames) / best / 1e6, 1)}
    del spec

    # torchaudio: the same variants of one clip on this GPU (events) and on the host (wall clock, one run)
    x = clips[0]
    res["torchaudio_gpu_ms_per_clip"] = round(events_ms(lambda: torchaudio_variants(x, rates, dev), 1, 3), 2)
    ours_one = Augmenter(SR, None, (20, 4), device=dev, _engine=eng)
    stretch_rates = [(f"v{i}", r, None) for i, r in enumerate(rates)]
    res["ours_stretch_only_ms_per_clip"] = round(events_ms(lambda: ours_one.apply([x], stretch_rates), 1, 3), 2)
    xc = x.cpu()
    t0 = time.perf_counter()
    torchaudio_variants(xc, rates, torch.device("cpu"))
    res["torchaudio_host_ms_per_clip"] = round((time.perf_counter() - t0) * 1e3, 1)
    res["host_threads"] = torch.get_num_threads()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
