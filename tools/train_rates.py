"""Time one training step (bt_train_forward + bt_train_backward through BeatThisModule) of a final0-shaped model against
torch fp32 autograd of the oracle restatement of the same eval-mode model on the same GPU.

    python tools/train_rates.py [--batches 8 32] [--length 1500] [--out train_rates.json]

A step is forward, a loss-shaped upstream gradient and backward to every trainable parameter.  FLOPs are counted from
the shapes: 2 M N K per GEMM and 4 n^2 32 per attention head and sequence for the forward pass, three times that for
a step (the backward pass needs two GEMMs per forward GEMM).  Torch runs with TF32 off, its default for matmuls.  CUDA
events around `--iters` steps after `--warmup` steps; the per-kernel-class times come from the library's profile in a
separate pass.  The card's name and power limit are printed with the numbers.
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
from oracle import beat_this_oracle as O  # noqa: E402


def _rope_on_device(t, freqs):
    """O.rope with its position table on t's device (the oracle builds it on the CPU)."""
    n = t.shape[-2]
    pos = torch.arange(n, dtype=torch.float32, device=t.device)
    ang = (pos[:, None] * freqs[None, :].float()).repeat_interleave(2, dim=-1)
    t2 = t.reshape(*t.shape[:-1], -1, 2)
    rot = torch.stack((-t2[..., 1], t2[..., 0]), dim=-1).reshape(t.shape)
    return t * ang.cos() + rot * ang.sin()


def forward_flops(hp: dict, B: int, L: int) -> float:
    D, BL = hp["transformer_dim"], B * L
    C, F, total = 32, 32, 2.0 * BL * 32 * 32 * 12  # stem
    for _ in range(3):
        if hp["partial_transformers"]:
            tok = BL * F
            # two (attention, FFN) pairs: qkv, gates, out and the FFN's two GEMMs each
            total += 2 * 2.0 * tok * (3 * C * C + (C // 32) * C + C * C + 2 * 4 * C * C)
            total += 4.0 * F * F * 32 * (C // 32) * BL + 4.0 * L * L * 32 * (C // 32) * B * F  # attnF, attnT
        total += 2.0 * BL * (F // 2) * (2 * C) * (C * 6)
        C, F = 2 * C, F // 2
    total += 2.0 * BL * D * C * F  # frontend.linear
    per_layer = 2.0 * BL * (3 * D * D + (D // 32) * D + D * D + 2 * hp["ff_mult"] * D * D) + 4.0 * L * L * D * B
    return total + hp["n_layers"] * per_layer + 2.0 * BL * 2 * D


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
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--length", type=int, default=1500)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    hp = synthetic.model_hparams("final0")
    module = BeatThisModule.from_checkpoint(synthetic.make_checkpoint("final0", 0), dev)
    sd = {k: v.detach().clone().requires_grad_(v.requires_grad) if v.is_floating_point() else v
          for k, v in module.state_dict(keep_vars=True).items()}
    O.rope = _rope_on_device
    results = []
    for B in args.batches:
        L = args.length
        x = torch.rand(B, L, 128, device=dev, generator=torch.Generator(dev).manual_seed(B)) * 4
        g = torch.randn(2, B, L, device=dev, generator=torch.Generator(dev).manual_seed(B + 1))

        def ours():
            module.zero_grad(set_to_none=True)
            out = module(x)
            torch.autograd.backward((out["beat"], out["downbeat"]), (g[0], g[1]))

        def theirs():
            for v in sd.values():
                v.grad = None
            beat, down = O.forward(sd, x, sum_head=hp["sum_head"])
            torch.autograd.backward((beat, down), (g[0], g[1]))

        flops = 3 * forward_flops(hp, B, L)
        ms = time_ms(ours, args.warmup, args.iters)
        eng = module.engine
        eng.profile_reset()
        eng.profile_enable(True)
        ours()
        prof = eng.profile_results()
        eng.profile_enable(False)
        try:
            torch_ms = time_ms(theirs, args.warmup, args.iters)
        except torch.OutOfMemoryError:
            torch_ms = None
        torch.cuda.empty_cache()
        row = {
            "B": B, "L": L, "ms_per_step": ms, "tflops": flops / ms / 1e9,
            "activation_bytes": eng.train_activation_bytes(B, L), "torch_fp32_ms_per_step": torch_ms,
            "kernel_ms": {k: round(v[0], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])},
            "card": card,
        }
        results.append(row)
        print(json.dumps(row))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
