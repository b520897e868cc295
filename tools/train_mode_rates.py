"""Time a final0 training step in training mode (dropout 0.1 / 0.2, batch-statistics BatchNorm) against the same step
in eval mode, alternating the two in one process.

    python tools/train_mode_rates.py [--batch 8] [--length 1500] [--rounds 3] [--out train_mode_rates.json]

A step is BeatThisModule's forward, an upstream gradient at both logits and the backward pass to every trainable
parameter and the spectrogram.  Each round times `--iters` steps of each mode with CUDA events after `--warmup` steps;
the spread over rounds is printed.  The per-kernel-class times (the three attention passes among them) come from the
library's profile in a separate pass per mode.  The card's name and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from beat_this_b200 import synthetic  # noqa: E402
from beat_this_b200.train import BeatThisModule  # noqa: E402

ATTENTION = ("train_attention", "train_attention_dq", "train_attention_dkv")


def time_ms(step, warmup, iters):
    for _ in range(warmup):
        step()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--length", type=int, default=1500)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    module = BeatThisModule.from_checkpoint(synthetic.make_checkpoint("final0", 0), dev, train_mode=True)
    B, L = args.batch, args.length
    x = torch.rand(B, L, 128, device=dev, generator=torch.Generator(dev).manual_seed(B)) * 4
    x.requires_grad_(True)
    g = torch.randn(2, B, L, device=dev, generator=torch.Generator(dev).manual_seed(B + 1))

    def step():
        module.zero_grad(set_to_none=True)
        x.grad = None
        out = module(x)
        torch.autograd.backward((out["beat"], out["downbeat"]), (g[0], g[1]))

    times = {"train": [], "eval": []}
    for _ in range(args.rounds):
        for mode in ("train", "eval"):
            module.train(mode == "train")
            times[mode].append(time_ms(step, args.warmup, args.iters))
    eng = module.engine
    profile = {}
    for mode in ("train", "eval"):
        module.train(mode == "train")
        step()
        torch.cuda.synchronize()
        eng.profile_reset()
        eng.profile_enable(True)
        step()
        prof = eng.profile_results()
        eng.profile_enable(False)
        total = sum(v[0] for v in prof.values())
        attn = sum(prof[k][0] for k in ATTENTION if k in prof)
        profile[mode] = {"kernel_ms_total": round(total, 3), "attention_ms": round(attn, 3),
                         "attention_share": round(attn / total, 4),
                         "kernel_ms": {k: round(v[0], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])}}
    row = {"B": B, "L": L, "card": card,
           "train_ms_per_step": [round(t, 2) for t in times["train"]],
           "eval_ms_per_step": [round(t, 2) for t in times["eval"]],
           "overhead": round(min(times["train"]) / min(times["eval"]) - 1, 4),
           "profile": profile}
    print(json.dumps(row))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(row, f, indent=1)


if __name__ == "__main__":
    main()
