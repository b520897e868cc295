"""Time the minimal peak picker's kernel at 50 and 100 frames per second.

    python tools/peakpick_rates.py [--clips 64] [--secs 30] [--iters 200] [--out peakpick_rates.json]

Workloads, each `--clips` clips of `--secs` seconds of seeded sinusoid-plus-noise logits (a beat period of 0.4-0.8 s):
- bt_peakpick on the 50 fps logits (1 + 50 secs frames per clip);
- bt_peakpick_fps with fps = 50 on the same logits (the same kernel: any difference is noise);
- bt_peakpick_fps with fps = 100 on the same logits (only the divisor changes);
- bt_peakpick_fps with fps = 100 on logits of clips of the same length at 100 fps (twice the frames; the noise makes
  more local maxima in the +-3 frame window, so more peaks).
Each row is the kernel's device time from the library's profile (CUDA events around each launch): the median of five
means over `--iters` launches each, after `--warmup`, with the smallest and largest of the five.  The card's name, power limit and
SM clocks are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from beat_this_b200.engine import Engine  # noqa: E402


def logits(clips, secs, fps, seed=0):
    rng = np.random.default_rng(seed)
    n = 1 + int(secs * fps)
    t = np.arange(n) / fps
    out = []
    for _ in range(clips):
        period = rng.uniform(0.4, 0.8)
        out.append((2.5 * np.sin(2 * np.pi * t / period + rng.uniform(0, 6)) + 0.7 * rng.standard_normal(n)).astype(np.float32))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--secs", type=float, default=30.0)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    eng = Engine.mel_only("cuda")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    data = {}
    for fps in (50, 100):
        b = logits(a.clips, a.secs, fps, 1)
        d = logits(a.clips, a.secs, fps, 2)
        fo = np.cumsum([0] + [len(x) for x in b]).tolist()
        data[fps] = (torch.tensor(np.concatenate(b), device=eng.device), torch.tensor(np.concatenate(d), device=eng.device), fo)
    b50, d50, fo50 = data[50]
    b100, d100, fo100 = data[100]
    work = [
        ("bt_peakpick_50fps_logits", True, b50, d50, fo50, None),
        ("bt_peakpick_fps_50_50fps_logits", False, b50, d50, fo50, 50.0),
        ("bt_peakpick_fps_100_50fps_logits", False, b50, d50, fo50, 100.0),
        ("bt_peakpick_fps_100_100fps_logits", False, b100, d100, fo100, 100.0),
    ]
    from ctypes import c_void_p

    from beat_this_b200._lib import check, i64_array

    rows = {}
    outs = {}
    for name, legacy, beat, down, fo, fps in work:
        n = len(fo) - 1
        width = max(b - a_ for a_, b in zip(fo[:-1], fo[1:]))
        times = torch.empty((2, n, width), dtype=torch.float64, device=eng.device)
        cnt = torch.empty((2, n), dtype=torch.int32, device=eng.device)
        head = (eng.ctx, c_void_p(beat.data_ptr()), c_void_p(down.data_ptr()), i64_array(fo), n)
        tail = (c_void_p(times[0].data_ptr()), c_void_p(cnt[0].data_ptr()), c_void_p(times[1].data_ptr()),
                c_void_p(cnt[1].data_ptr()), width, eng._stream())

        def call():
            code = eng.lib.bt_peakpick(*head, *tail) if legacy else eng.lib.bt_peakpick_fps(*head, fps, *tail)
            check(eng.lib, eng.ctx, code)

        for _ in range(a.warmup):
            call()
        means = []
        for _ in range(5):
            eng.profile_enable(True)
            eng.profile_reset()
            for _ in range(a.iters):
                call()
            prof = eng.profile_results()
            eng.profile_enable(False)
            ms, launches = prof["peakpick"]
            assert launches == a.iters and set(prof) == {"peakpick"}
            means.append(ms / launches * 1e3)
        torch.cuda.synchronize()
        outs[name] = (times.cpu().numpy(), cnt.cpu().numpy())
        rows[name] = {"us": float(np.median(means)), "us_min": min(means), "us_max": max(means),
                      "peaks_per_clip": float(cnt[0].float().mean().item())}
        print(f"{name:36s} {rows[name]['us']:8.2f} us  [{min(means):.2f}, {max(means):.2f}]  "
              f"{rows[name]['peaks_per_clip']:.1f} beats / clip")
    same = outs["bt_peakpick_50fps_logits"][0].tobytes() == outs["bt_peakpick_fps_50_50fps_logits"][0].tobytes()
    res = {"gpu": smi, "clips": a.clips, "secs": a.secs, "iters": a.iters, "rows": rows, "fps50_bitwise_bt_peakpick": same}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
