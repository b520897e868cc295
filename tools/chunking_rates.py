"""Launches and time of split_predict_aggregate on one long piece: the batched path (one bt_spect2frames_chunked call,
every chunk in one wave) against the per-chunk route (one bt_forward_chunks call per chunk, stitched by
aggregate_prediction), with the same chunking.

    python tools/chunking_rates.py [--minutes 10] [--chunk 1500] [--border 0] [--mode keep_first] [--float32]
                                   [--model final0] [--out chunking_rates.json]

The piece is the log-mel spectrogram of synth_clip(0, minutes * 60) on the seeded checkpoint of beat_this_b200.synthetic.
Times are CUDA events around --iters calls after --warmup calls; the two routes alternate, and their outputs must be
bitwise equal.  The card's name, power limit and SM clocks are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from beat_this_b200 import synthetic  # noqa: E402
from beat_this_b200.inference import Spect2Frames, split_predict_aggregate  # noqa: E402


def time_ms(fn, iters):
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
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--chunk", type=int, default=1500)
    ap.add_argument("--border", type=int, default=0)
    ap.add_argument("--mode", default="keep_first", choices=["keep_first", "keep_last"])
    ap.add_argument("--model", default="final0")
    ap.add_argument("--float32", action="store_true", help="fp32 CUDA-core path instead of the 16-bit tensor-core path")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("chunking_rates needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = synthetic.write_checkpoint(os.path.join(tmp, f"{args.model}.ckpt"), args.model, 0)
        s2f = Spect2Frames(ckpt, "cuda:0", float16=not args.float32)
    model, eng = s2f.model, s2f.model.engine
    spect = eng.logmel([synthetic.synth_clip(0, args.minutes * 60.0)])[0]
    c, b, mode = args.chunk, args.border, args.mode
    per_chunk = lambda x: model(x)  # noqa: E731  (not a BeatThisB200: the per-chunk route)
    routes = {"batched": lambda: split_predict_aggregate(spect, c, b, mode, model),
              "per_chunk": lambda: split_predict_aggregate(spect, c, b, mode, per_chunk)}
    res = {"gpu": smi, "frames": int(spect.shape[0]), "chunking": [c, b, mode], "model": args.model,
           "dtype": "f32" if args.float32 else eng.act_dtype}
    outs = {}
    for name, fn in routes.items():
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        n0 = eng.launches
        outs[name] = fn()
        torch.cuda.synchronize()
        res[f"{name}_launches"] = eng.launches - n0
    res["bitwise_equal"] = all(torch.equal(outs["batched"][k], outs["per_chunk"][k]) for k in ("beat", "downbeat"))
    for name in routes:
        res[f"{name}_ms"] = []
    for _ in range(args.rounds):
        for name, fn in routes.items():
            res[f"{name}_ms"].append(round(time_ms(fn, args.iters), 3))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
