"""Time per piece of split_predict_aggregate on one 10-minute piece (30 001 frames) at chunk lengths 1500, 3000, 6000
and the whole piece, on a model loaded with max_chunk_size = 30 001.

    python tools/long_chunk_rates.py [--minutes 10] [--chunks 1500,3000,6000,0] [--border 0] [--float32]
                                     [--model final0] [--out long_chunk_rates.json]

A chunk length of 0 stands for the whole piece.  The piece is the log-mel spectrogram of synth_clip(0, minutes * 60) on
the seeded checkpoint of beat_this_b200.synthetic.  Per chunk length: ms per piece (CUDA events around --iters calls
after --warmup calls, --rounds times, the lengths alternating), the time-direction and frequency-direction attention
ms per piece (the library's per-kernel-class device timing, bt_profile_*, in a separate run), the chunks, waves and
padded frames of the call, and the device memory the context holds after it (its workspace is sized once, for the frame
budget max(128 x 1500, max_chunk_size) frames).  The card's name, power limit and SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from beat_this_b200 import _lib, synthetic  # noqa: E402
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


def smi(fields):
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--chunks", default="1500,3000,6000,0", help="chunk lengths; 0 = the whole piece")
    ap.add_argument("--border", type=int, default=0)
    ap.add_argument("--model", default="final0")
    ap.add_argument("--float32", action="store_true", help="fp32 CUDA-core path instead of the 16-bit tensor-core path")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("long_chunk_rates needs a CUDA device")
    res = {"gpu": smi("name,power.limit,clocks.max.sm")}
    free0 = torch.cuda.mem_get_info()[0]
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = synthetic.write_checkpoint(os.path.join(tmp, f"{args.model}.ckpt"), args.model, 0)
        audio = synthetic.synth_clip(0, args.minutes * 60.0)
        T = 1 + len(audio) // 441
        s2f = Spect2Frames(ckpt, "cuda:0", float16=not args.float32, max_chunk_size=T)
    model, eng = s2f.model, s2f.model.engine
    spect = eng.logmel([audio])[0]
    b = args.border
    lengths = [int(c) or T for c in args.chunks.split(",")]
    res.update({"frames": T, "model": args.model, "dtype": "f32" if args.float32 else eng.act_dtype, "border": b,
                "max_chunk_size": model.max_chunk_size})
    routes = {c: (lambda c=c: split_predict_aggregate(spect, c, b, "keep_first", model)) for c in lengths}
    rows = {}
    for c, fn in routes.items():
        ck = _lib.bt_chunking(c, b, 0)
        n = int(eng.lib.bt_plan_chunking_max(T, ctypes.byref(ck), model.max_chunk_size, None, None, None, None, 0))
        for _ in range(args.warmup):
            out = fn()
        torch.cuda.synchronize()
        assert all(torch.isfinite(out[k]).all() for k in ("beat", "downbeat")), c
        eng.profile_reset()
        eng.profile_enable(True)
        fn()
        prof = eng.profile_results()
        eng.profile_enable(False)
        rows[c] = {"chunks": n, "waves": prof["stem"][1], "padded_frames": n * c,
                   "attn_time_ms": round(sum(ms for k, (ms, _) in prof.items() if k.startswith("attn_time")), 3),
                   "attn_freq_ms": round(prof.get("attn_freq", (0.0, 0))[0], 3), "ms": []}
    res["ctx_device_mb"] = round((free0 - torch.cuda.mem_get_info()[0]) / 2**20, 1)
    for _ in range(args.rounds):
        for c, fn in routes.items():
            rows[c]["ms"].append(round(time_ms(fn, args.iters), 3))
    res["sm_clock_after"] = smi("clocks.sm")
    res["by_chunk"] = {str(c): r for c, r in rows.items()}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
