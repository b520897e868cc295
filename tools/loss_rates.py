"""Time bt_beat_loss (forward, two launches) and bt_beat_loss_backward (one launch) against the reference's torch
modules composed on the same GPU (beat_this_b200's restatement of loss.py is not used: the torch arm is the same
max_pool1d / binary_cross_entropy_with_logits graph the reference builds, run eagerly).

    python tools/loss_rates.py [--out loss_rates.json]

Workloads: B = 64 rows of T = 1500 frames (a training batch of the reference) and a ragged set of 64 pieces of 500 to
15 000 frames (the torch arm scores those one piece at a time, as the reference's test_step does).  CUDA events around
`--iters` calls after `--warmup` calls; the card's name, power limit and SM clock are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from beat_this_b200 import loss as L  # noqa: E402


def torch_shift_tolerant(preds, targets, mask, t, pw):
    """ShiftTolerantBCELoss.forward (reference loss.py:76-92) in plain torch."""
    spread = lambda x, f: F.max_pool1d(x, 1 + 2 * f * t, 1)  # noqa: E731
    crop = lambda x, f: x[..., f * t : -f * t or None]  # noqa: E731
    look_at = crop(targets, 2) + (1 - spread(targets, 2))
    look_at = look_at * crop(mask, 2)
    return F.binary_cross_entropy_with_logits(crop(spread(preds, 1), 1), crop(targets, 2), weight=look_at, pos_weight=pw)


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
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("loss_rates needs a CUDA device")
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    t, pw = 3, 4.5
    pw_t = torch.tensor(pw, device=dev)
    res = {}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res["gpu"] = smi

    # B x T batch
    B, T = 64, 1500
    x = torch.tensor(rng.standard_normal((B, T)) * 3, dtype=torch.float32, device=dev, requires_grad=True)
    y = torch.tensor(rng.random((B, T)) < 0.05, dtype=torch.float32, device=dev)
    m = torch.ones(B, T, device=dev)
    ours = L.ShiftTolerantBCELoss(pw, t)
    g = torch.ones((), device=dev)
    res["batch_fwd_ms"] = time_ms(lambda: ours(x, y, m), args.warmup, args.iters)
    res["torch_batch_fwd_ms"] = time_ms(lambda: torch_shift_tolerant(x, y, m, t, pw_t), args.warmup, args.iters)
    res["batch_fwd_bwd_ms"] = time_ms(lambda: torch.autograd.grad(ours(x, y, m), x, g), args.warmup, args.iters)
    res["torch_batch_fwd_bwd_ms"] = time_ms(lambda: torch.autograd.grad(torch_shift_tolerant(x, y, m, t, pw_t), x, g),
                                            args.warmup, args.iters)
    ours_v = float(ours(x, y, m).detach())
    ref_v = float(torch_shift_tolerant(x, y, m, t, pw_t).detach())
    res["batch_loss_ours_vs_torch"] = [ours_v, ref_v]

    # ragged pieces: one call for all of them against one torch call per piece
    lens = rng.integers(500, 15001, 64)
    off = np.concatenate([[0], np.cumsum(lens)]).tolist()
    xr = torch.tensor(rng.standard_normal(off[-1]) * 3, dtype=torch.float32, device=dev)
    yr = torch.tensor(rng.random(off[-1]) < 0.05, dtype=torch.float32, device=dev)
    mr = torch.ones(off[-1], device=dev)
    spec = L.loss_spec(ours)
    res["ragged_frames"] = int(off[-1])
    res["ragged_fwd_ms"] = time_ms(lambda: L.beat_loss_rows(xr, yr, mr, off, *spec), args.warmup, args.iters)
    pieces = [(xr[a:b][None], yr[a:b][None], mr[a:b][None]) for a, b in zip(off[:-1], off[1:])]
    res["torch_ragged_fwd_ms"] = time_ms(lambda: [torch_shift_tolerant(a, b, c, t, pw_t) for a, b, c in pieces],
                                         max(2, args.warmup // 4), max(5, args.iters // 10))
    rows, _ = L.beat_loss_rows(xr, yr, mr, off, *spec)
    want = torch.stack([torch_shift_tolerant(a, b, c, t, pw_t) for a, b, c in pieces]).double()
    res["ragged_max_rel_diff"] = float(((rows - want).abs() / want.abs()).max())
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
