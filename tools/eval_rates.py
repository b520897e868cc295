"""Speed of the device beat metrics (bt_beat_metrics) against the numpy restatement of the same contract
(tests/beat_metrics_reference.py), on the same seeded sets: --pieces pieces of 30 s to 10 min, beats and downbeats
(2 x --pieces sets), jittered, with dropped and inserted beats and tempo-doubled, halved or off-beat estimates.

    python tools/eval_rates.py [--pieces 10000] [--reps 20]

Prints one JSON line:
  gpu           name, power limit and SM clock read from nvidia-smi in this run
  sets, beats   sets scored and estimates + references in them
  device_ms     CUDA events around the bt_beat_metrics launch alone (mean / min over --reps, after a warm-up), and
                beat_metrics() wall time including the input checks, the packing, the H2D and the D2H copies
  numpy_s       the restatement's wall time (host clock, one run)
  agree         the two tables are equal (Cemgil within 1e-12)
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info(index: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl, sm, smax = [f.strip() for f in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_mhz": float(sm), "sm_max_mhz": float(smax)}
    except Exception as e:  # the numbers still stand, without the card's state
        return {"name": torch.cuda.get_device_name(index), "error": f"nvidia-smi: {e}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pieces", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()

    import beat_metrics_reference as BM
    from beat_this_b200 import _lib
    from beat_this_b200.engine import Engine
    from beat_this_b200.evaluate import beat_metrics

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    est, ref = BM.pieces(2024, args.pieces)
    n = len(est)

    beat_metrics(est[:64], ref[:64], device=dev)  # warm-up: context, module load
    t0 = time.perf_counter()
    got = beat_metrics(est, ref, device=dev)
    call_ms = (time.perf_counter() - t0) * 1e3

    # the launch alone, on inputs already on the device
    eng = Engine.shared(dev)
    offs = np.concatenate(([0], np.cumsum([len(a) for a in est + ref]))).astype(np.int64)
    packed = torch.from_numpy(np.concatenate(est + ref)).to(dev)
    out = torch.empty((n, 12), dtype=torch.float64, device=dev)
    p = _lib.bt_beat_metric_params(5.0, 0.07, 0.04, 0.175, 0.175)
    eo, ro = _lib.i64_array(offs[: n + 1]), _lib.i64_array(offs[n:])
    base = ctypes.c_void_p(packed.data_ptr())

    def launch():
        _lib.check(eng.lib, eng.ctx, eng.lib.bt_beat_metrics(eng.ctx, base, eo, base, ro, n, ctypes.byref(p),
                                                             ctypes.c_void_p(out.data_ptr()), eng._stream()))

    launch()
    torch.cuda.synchronize(dev)
    times = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        launch()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    assert np.array_equal(out.cpu().numpy(), got)

    t0 = time.perf_counter()
    want = BM.beat_metrics(est, ref)
    numpy_s = time.perf_counter() - t0
    exact = [i for i in range(12) if i not in (6, 7)]
    agree = bool(np.array_equal(got[:, exact], want[:, exact]) and np.max(np.abs(got[:, 6:8] - want[:, 6:8])) <= 1e-12)
    print(json.dumps({
        "gpu": gpu_info(0),
        "sets": n,
        "beats": int(offs[-1]),
        "device_ms": {"kernel_mean": float(np.mean(times)), "kernel_min": float(np.min(times)), "beat_metrics_call": call_ms},
        "numpy_s": numpy_s,
        "agree": agree,
    }))
    return 0 if agree else 1


if __name__ == "__main__":
    sys.exit(main())
