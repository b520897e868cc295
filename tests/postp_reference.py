"""Float64 numpy restatement of the minimal post-processor at any frame rate: the contract of bt_peakpick_fps
(include/beatthis.h), which is the reference's Postprocessor("minimal", fps) (model/postprocessor.py:85-136,176-197)."""
import numpy as np


def peak_frames(x) -> np.ndarray:
    """Frames t with x[t] == max(x[t-3 .. t+3]) (the window cut at the clip's ends) and x[t] > 0."""
    x = np.asarray(x, np.float32)
    padded = np.concatenate([np.full(3, -np.inf, np.float32), x, np.full(3, -np.inf, np.float32)])
    mx = np.lib.stride_tricks.sliding_window_view(padded, 7).max(axis=1) if len(x) else x
    return np.nonzero((x == mx) & (x > 0))[0]


def merge_adjacent(frames) -> np.ndarray:
    """Runs of peaks at most one frame from the running mean of the run become that mean (float64)."""
    out = []
    cur, c = None, 0.0
    for f in map(float, frames):
        if cur is not None and f - cur <= 1.0:
            c += 1.0
            cur += (f - cur) / c
        else:
            if cur is not None:
                out.append(cur)
            cur, c = f, 1.0
    if cur is not None:
        out.append(cur)
    return np.asarray(out, np.float64)


def postp_minimal(beat, down, fps):
    """One clip's fp32 logits -> (beat_times, downbeat_times), float64 seconds."""
    bt = merge_adjacent(peak_frames(beat)) / fps
    dt = merge_adjacent(peak_frames(down)) / fps
    if len(bt):
        dt = np.asarray([bt[np.argmin(np.abs(bt - d))] for d in dt], np.float64)
    return bt, np.unique(dt)
