"""Optimizer-step rates of data-parallel training (beat_this_b200.train) at W = 1, 2, 4 and 8 ranks, as many as the
machine has GPUs.

    python tools/train_dp_rates.py [--pieces 64] [--rounds 3] [--steps 4] [--warmup 1] [--out train_dp_rates.json]

The shape: final0 in training mode, B 8, L 1500, accumulate 8, over a seeded float16 bundle written to a temporary
directory as tools/batch_rates.py writes it.  Each round launches one torchrun job per W, in turn (alternating
rounds); a job runs passes over the data as fit's epochs do and times `--steps` optimizer steps of 8 micro-batches
after `--warmup`, each a host clock around one step of fit's loop (W = 1: the one-process loop; W > 1: the owned
micro-batches, the gather, the ordered sum, the replay and AdamW) ending in a device synchronise.  It reports per W the median step time over the rounds and the speed-up over W = 1, and, by CUDA
events in the W > 1 jobs, the all_gather of one step's send buffer, one bt_grad_pack and one bt_grad_ordered_sum of 8
rows.  The cards' names, power limits and the GPU interconnect (nvidia-smi topo -m) are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import socket
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

B, L, ACC = 8, 1500, 8


def event_ms(fn, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def worker(args):
    import numpy as np
    import torch.distributed as dist

    from batch_rates import AUG
    from beat_this_b200 import dataset as D
    from beat_this_b200 import synthetic
    from beat_this_b200 import train as T
    from beat_this_b200.distributed import init_from_env
    from beat_this_b200.loss import loss_from_hparams
    from beat_this_b200.optim import AdamW, param_groups

    rank, world, local = init_from_env()
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    np.random.seed(0)
    torch.manual_seed(0)
    names = json.loads(Path(args.data, "names.json").read_text())
    ds = D.BeatTrackingDataset(names, args.data, 50, L, deterministic=False, augmentations=AUG,
                               length_based_oversampling_factor=0.65)
    batches = D.TrainingBatches(ds, B, shuffle=True, drop_last=True, seed=0, device=device)
    # passes over the data as fit's epochs run them, as many as the steps take; only full steps are timed
    groups = T.micro_batch_owners(len(batches), ACC, world)
    if len(groups[0]) < ACC:
        raise SystemExit(f"{len(batches)} batches make no step of {ACC} micro-batches: raise --pieces")
    owners = [r for g in groups for r, _ in g]
    if world > 1:
        batches.shard = lambda k: owners[k] == rank
    hp = dict(synthetic.model_hparams("final0"), pos_weights={"beat": 1, "downbeat": 1})
    module = T.BeatThisModule(hp, device, train_mode=True).reset_parameters().train()
    loss_pair = loss_from_hparams(hp)
    opt = AdamW(param_groups(module, 0.01), lr=1e-4)
    exchange = T._GradientExchange(module, opt, world, ACC) if world > 1 else None
    times = []
    while len(times) < args.warmup + args.steps:
        times += one_pass(module, batches, groups, rank, exchange, loss_pair, opt, T)
    res = {"world": world, "step_s": statistics.median(times[args.warmup : args.warmup + args.steps])}
    if exchange is not None:
        eng, grads = module.engine, exchange.grads
        rows = [exchange.recv[j % world, j // world] for j in range(ACC)]
        res["all_gather_ms"] = event_ms(lambda: dist.all_gather(list(exchange.recv.unbind(0)), exchange.send), 5)
        res["grad_pack_ms"] = event_ms(lambda: eng.grad_pack(grads, exchange.send[0]), 20)
        res["grad_ordered_sum_ms"] = event_ms(lambda: eng.grad_ordered_sum(grads, rows), 20)
        res["P"], res["Q"] = exchange.P, exchange.Q
    if rank == 0:
        Path(args.result).write_text(json.dumps(res))
    if world > 1:
        dist.destroy_process_group()


def one_pass(module, batches, groups, rank, exchange, loss_pair, opt, T):
    """One pass over the batches, a step per group as fit runs them: the times of the steps of ACC micro-batches."""
    it = iter(batches)
    times = []
    for group in groups:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for owner, slot in group:
            batch = next(it)
            if owner != rank:
                module.dropout_mode()
                continue
            out = module(batch["spect"], batch_stats=None if exchange is None else exchange.stats(slot))
            lb, ld = T._losses(loss_pair, out, batch)
            ((lb + ld) / ACC).backward()
            if exchange is not None:
                exchange.pack(slot, lb, ld, batch["spect"].shape)
        if exchange is not None:
            exchange.reduce(len(group))
        opt.step()
        opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        if len(group) == ACC:
            times.append(time.perf_counter() - t0)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pieces", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default="train_dp_rates.json")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--data", help=argparse.SUPPRESS)
    ap.add_argument("--result", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    if not torch.cuda.is_available():
        raise SystemExit("train_dp_rates measures on CUDA devices; there is none")
    from batch_rates import write_dataset

    n_gpus = torch.cuda.device_count()
    worlds = [w for w in (1, 2, 4, 8) if w <= n_gpus]
    query = ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]
    cards = subprocess.run(query, capture_output=True, text=True).stdout.strip().splitlines()
    topo = subprocess.run(["nvidia-smi", "topo", "-m"], capture_output=True, text=True).stdout
    runs = {w: [] for w in worlds}
    with tempfile.TemporaryDirectory() as tmp:
        names = write_dataset(Path(tmp), args.pieces)
        Path(tmp, "names.json").write_text(json.dumps(names))
        for _ in range(args.rounds):
            for w in worlds:
                result = os.path.join(tmp, f"w{w}.json")
                cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={w}",
                       "--master-addr", "127.0.0.1", "--master-port", str(free_port()), os.path.abspath(__file__),
                       "--worker", "--data", tmp, "--result", result, "--steps", str(args.steps), "--warmup",
                       str(args.warmup)]
                subprocess.run(cmd, check=True, cwd=ROOT)
                runs[w].append(json.loads(Path(result).read_text()))
    base = statistics.median(r["step_s"] for r in runs[1])
    out = {"gpus": cards, "interconnect": topo, "shape": dict(model="final0", B=B, L=L, accumulate=ACC), "worlds": {}}
    for w in worlds:
        step = statistics.median(r["step_s"] for r in runs[w])
        row = {"step_s": step, "speedup": base / step, "rounds": [r["step_s"] for r in runs[w]]}
        for k in ("all_gather_ms", "grad_pack_ms", "grad_ordered_sum_ms"):
            if k in runs[w][0]:
                row[k] = statistics.median(r[k] for r in runs[w])
        out["worlds"][w] = row
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(out, indent=1))
    print(json.dumps({k: v for k, v in out.items() if k != "interconnect"}, indent=1))
    print(topo)


if __name__ == "__main__":
    main()
