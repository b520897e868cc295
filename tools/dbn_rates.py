"""Speed of the device DBN (bt_dbn_track_device) against the host C++ tracker (bt_dbn_track) on the bench.py config-4
material: 64 seeded 30 s clips (seeds 7000..7063), final0-shaped synthetic checkpoint, 16-bit kernels.

    python tools/dbn_rates.py [--reps 20] [--clips 1000] [--runs 3]

Prints one JSON line:
  gpu            name, power limit and SM clock read from nvidia-smi in this run
  device_ms      the device DBN on the group's logits, CUDA events around one call (its three kernels and the copy of
                 the beat times to pinned memory; mean / min over --reps, after warm-up), and per kernel
  host_ms        bt_dbn_track wall time on the same group with one thread per hardware thread (what
                 Audio2Beats(dbn=True) uses) and with 1 thread
  e2e_clips_s    Audio2Beats(dbn=True).batch clips/s over --clips clips, dbn_impl "native" and "device" alternated
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CACHE = os.environ.get("BT_TEST_CACHE", "/tmp/beat_this_b200_cache")


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
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()

    from beat_this_b200 import synthetic
    from beat_this_b200.inference import Audio2Beats, Audio2Frames, load_model

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ckpt = synthetic.write_checkpoint(os.path.join(CACHE, "final0_s0.ckpt"), "final0", 0)
    model = load_model(ckpt, dev, float16=True)
    base = [synthetic.synth_clip(7000 + i, 30.0) for i in range(64)]
    dev_a2b = Audio2Beats.from_model(model, dbn=True, dbn_impl="device")
    nat_a2b = Audio2Beats.from_model(model, dbn=True, dbn_impl="native")
    eng = model.engine

    # one group's logits: 64 x 30 s
    frames = Audio2Frames.batch(dev_a2b, base, 22050)
    fo = [0]
    for b, _ in frames:
        fo.append(fo[-1] + b.numel())
    beat = torch.cat([b for b, _ in frames]).contiguous()
    down = torch.cat([d for _, d in frames]).contiguous()
    params = dev_a2b.frames2beats.dbn_params
    slot = {}
    for _ in range(3):
        eng.dbn_async(beat, down, fo, slot, params).result()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ms = []
    for _ in range(args.reps):
        e0.record()
        h = eng.dbn_async(beat, down, fo, slot, params)
        e1.record()
        h.result()
        e1.synchronize()
        dev_ms.append(e0.elapsed_time(e1))
    eng.profile_enable(True)
    eng.profile_reset()
    for _ in range(args.reps):
        eng.dbn_async(beat, down, fo, slot, params).result()
    prof = {k: v[0] / v[1] for k, v in eng.profile_results().items() if k.startswith("dbn_") and v[1]}
    eng.profile_enable(False)

    # the host tracker on the same group, on the activations batch_host builds
    trk = nat_a2b.frames2beats
    bh, dh = beat.cpu().numpy(), down.cpu().numpy()
    ref = trk.batch_host(bh, dh, fo)
    got = dev_a2b.frames2beats.batch_host(bh, dh, fo)
    identical = all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(ref, got))
    eps = 1e-5
    bp = torch.from_numpy(bh).double().sigmoid().numpy() * (1 - eps) + eps / 2
    dp = torch.from_numpy(dh).double().sigmoid().numpy() * (1 - eps) + eps / 2
    act = np.ascontiguousarray(np.stack((np.maximum(bp - dp, eps / 2), dp), axis=1))
    # Audio2Beats(dbn=True) calls bt_dbn_track with n_threads=0: one thread per hardware thread of the host
    pipe_threads = os.cpu_count() or 1
    host = {}
    for nt in (0, 1):
        trk.dbn.batch_cat(act, fo, n_threads=nt)
        ts = []
        for _ in range(3 if nt == 1 else 10):
            t0 = time.perf_counter()
            trk.dbn.batch_cat(act, fo, n_threads=nt)
            ts.append((time.perf_counter() - t0) * 1e3)
        host[f"threads_{nt or pipe_threads}"] = {"mean": float(np.mean(ts)), "min": float(np.min(ts)), "runs": len(ts)}

    # end to end, alternated
    clips = [base[i % 64] for i in range(args.clips)]
    for r in (nat_a2b, dev_a2b):
        r.batch(clips[:128], 22050)
    e2e = {"native": [], "device": []}
    for _ in range(args.runs):
        for name, r in (("native", nat_a2b), ("device", dev_a2b)):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            r.batch(clips, 22050)
            torch.cuda.synchronize(dev)
            e2e[name].append(len(clips) / (time.perf_counter() - t0))

    print(json.dumps({
        "gpu": gpu_info(0),
        "group": {"clips": 64, "seconds": 30.0, "frames": fo[-1], "checkpoint": "final0-shaped synthetic, 16-bit kernels"},
        "device_ms": {"mean": float(np.mean(dev_ms)), "min": float(np.min(dev_ms)), "reps": len(dev_ms),
                      "per_kernel_ms": prof},
        "host_ms": host,
        "host_pipeline_threads": pipe_threads,
        "device_equals_native_on_group": identical,
        "e2e_clips_s": {k: [round(v, 1) for v in vs] for k, vs in e2e.items()},
        "e2e_clips": len(clips),
    }))


if __name__ == "__main__":
    main()
