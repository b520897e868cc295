"""Host-side microbenchmarks on the bench box: DBN tracker and audio staging vs thread count."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from beat_this_b200 import _lib
from beat_this_b200.dbn import DBNDownBeatTracker

d = DBNDownBeatTracker(beats_per_bar=[3, 4], min_bpm=55.0, max_bpm=215.0, fps=50, transition_lambda=100)
acts = []
for i in range(64):
    T = 1501; t = np.arange(T)
    b = np.clip(0.5 + 0.5 * np.sin(2 * np.pi * t / (18 + i % 7) + i), 1e-5, 1 - 1e-5) ** 8
    dd = np.clip(0.5 + 0.5 * np.sin(2 * np.pi * t / (72 + 4 * (i % 7)) + i), 1e-5, 1 - 1e-5) ** 8 * 0.5
    acts.append(np.vstack((np.maximum(b - dd, 5e-6), dd)).T.copy())
d.batch(acts[:2])
t0 = time.perf_counter(); d.batch(acts[:1], 1); print("dbn 1 piece 1 thread: %.1f ms" % (1e3 * (time.perf_counter() - t0)))
for nt in (8, 16, 32, 64, 128):
    ts = []
    for _ in range(3):
        t0 = time.perf_counter(); d.batch(acts, nt); ts.append(time.perf_counter() - t0)
    print("dbn 64 pieces, %3d threads: %.1f ms (best of 3)" % (nt, 1e3 * min(ts)))

rng = np.random.default_rng(0)
clips64 = [rng.standard_normal(661500) for _ in range(64)]
clips32 = [c.astype(np.float32) for c in clips64]
dst = torch.empty(64 * 661500, dtype=torch.float32, pin_memory=torch.cuda.is_available())
for name, clips in (("float64", clips64), ("float32", clips32)):
    for nt in (4, 8, 16, 32, 64):
        _lib.stage_audio(clips, dst, nt)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter(); _lib.stage_audio(clips, dst, nt); ts.append(time.perf_counter() - t0)
        print("stage 64 x 30 s %s, %2d threads: %.1f ms" % (name, nt, 1e3 * min(ts)))
