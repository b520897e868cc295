"""Rates of the training loop (beat_this_b200.train.fit) and its AdamW update on one GPU.

    python tools/fit_rates.py [--pieces 64] [--rounds 5] [--micro 32] [--launches 200] [--out fit_rates.json]

The shape: final0 in training mode, B 8, L 1500, accumulate 8, over a seeded float16 bundle written to a temporary
directory as tools/batch_rates.py writes it (pitch, tempo and permute-mask augmentation).  It reports:
* the micro-batch time of the loop's body (a batch from TrainingBatches, forward, the loss pair, backward of the
  scaled sum, and every 8th micro-batch AdamW, the schedule and zero_grad) against bare forward and backward on a
  fixed batch of the same shape, in alternating rounds of `--micro` micro-batches, host clock ending in a device
  synchronise; medians over `--rounds`;
* the adamw_kernel time of one update of final0's 139 trainable tensors (CUDA events around `--launches` launches of
  a prepared table, so the host's table building is outside), the bytes it must move (28 per element) over that time
  against 3.35 TB/s; and, on the same tensors, optim.AdamW.step() and torch.optim.AdamW with foreach=True and with
  fused=True (CUDA events around `--launches` steps).
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from batch_rates import AUG, write_dataset  # noqa: E402
from beat_this_b200 import _lib, synthetic  # noqa: E402
from beat_this_b200 import dataset as D  # noqa: E402
from beat_this_b200 import train as T  # noqa: E402
from beat_this_b200.engine import Engine  # noqa: E402
from beat_this_b200.loss import loss_from_hparams  # noqa: E402
from beat_this_b200.optim import AdamW, CosineWarmupScheduler, param_groups  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
DEV = "cuda:0"


def timed(fn, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pieces", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--micro", type=int, default=32)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    torch.manual_seed(0)
    np.random.seed(0)
    B, L, acc = 8, 1500, 8
    hp = synthetic.model_hparams("final0")
    module = T.BeatThisModule(hp, DEV, train_mode=True).reset_parameters()
    module.train()
    trainable = [p for p in module.parameters() if p.requires_grad]
    res = {"card": card, "shape": {"model": "final0", "B": B, "L": L, "accumulate": acc},
           "tensors": len(trainable), "elements": sum(p.numel() for p in trainable),
           "decay_tensors": sum(p.ndim >= 2 for p in trainable),
           "decay_elements": sum(p.numel() for p in trainable if p.ndim >= 2)}

    with tempfile.TemporaryDirectory() as tmp:
        names = write_dataset(Path(tmp), args.pieces)
        ds = D.BeatTrackingDataset(names, tmp, 50, L, augmentations=AUG, length_based_oversampling_factor=0.65)
        batches = D.TrainingBatches(ds, B, seed=0, device=DEV)
        loss_pair = loss_from_hparams(hp)
        opt = AdamW(param_groups(module, 0.01), lr=8e-4)
        sched = CosineWarmupScheduler(opt, 1000, 100000)

        def stream():
            while True:
                yield from batches

        it = stream()
        k = [0]

        def loop_micro():
            batch = next(it)
            out = module(batch["spect"])
            lb, ld = T._losses(loss_pair, out, batch)
            ((lb + ld) / acc).backward()
            k[0] += 1
            if k[0] % acc == 0:
                opt.step()
                sched.step()
                opt.zero_grad(set_to_none=True)

        x = (torch.rand(B, L, 128, generator=torch.Generator().manual_seed(1)) * 4).to(DEV)
        gb, gd = torch.randn(2, B, L, device=DEV)

        def bare_micro():
            out = module(x)
            torch.autograd.backward((out["beat"], out["downbeat"]), (gb, gd))

        def rounds(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.micro):
                fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / args.micro * 1e3

        for fn in (loop_micro, bare_micro):  # warm-up of every shape
            for _ in range(acc):
                fn()
        loop_ms, bare_ms = [], []
        for _ in range(args.rounds):
            loop_ms.append(rounds(loop_micro))
            bare_ms.append(rounds(bare_micro))
        res["loop_micro_batch_ms"] = float(np.median(loop_ms))
        res["bare_fwd_bwd_ms"] = float(np.median(bare_ms))
        res["loop_overhead_ms"] = res["loop_micro_batch_ms"] - res["bare_fwd_bwd_ms"]
        res["rounds"] = {"loop_ms": loop_ms, "bare_ms": bare_ms}

    # the update alone, on the same 139 tensors with fresh gradients
    g = torch.Generator(DEV).manual_seed(2)
    for p in trainable:
        p.grad = torch.randn(p.shape, device=DEV, generator=g) * 1e-3
    opt = AdamW(param_groups(module, 0.01), lr=8e-4)
    opt.step()
    eng = Engine.shared(DEV)
    entries = [_lib.bt_adamw_entry(p.data_ptr(), p.grad.data_ptr(), opt.state[p]["exp_avg"].data_ptr(),
                                   opt.state[p]["exp_avg_sq"].data_ptr(), p.numel(), 8e-4, 0.9, 0.999, 1e-8,
                                   0.01 if p.ndim >= 2 else 0.0, 10) for p in trainable]
    table = (_lib.bt_adamw_entry * len(entries))(*entries)
    launch = lambda: eng._call("bt_adamw_step", table, len(entries))  # noqa: E731
    for _ in range(20):
        launch()
    kernel_ms = timed(launch, args.launches)
    nbytes = 28 * res["elements"]
    res["adamw_kernel_ms"] = kernel_ms
    res["adamw_bytes"] = nbytes
    res["adamw_bytes_per_s"] = nbytes / (kernel_ms * 1e-3)
    res["adamw_share_of_3_35_TBps"] = res["adamw_bytes_per_s"] / HBM_BYTES_PER_S
    res["optim_AdamW_step_ms"] = timed(opt.step, args.launches)
    for kind in ("foreach", "fused"):
        ref = torch.optim.AdamW(param_groups(module, 0.01), lr=8e-4, **{kind: True})
        for _ in range(5):
            ref.step()
        res[f"torch_AdamW_{kind}_step_ms"] = timed(ref.step, args.launches)
    print(json.dumps(res))
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
