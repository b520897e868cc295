"""Generate tests/golden/postp_fps.npz by running the UNMODIFIED reference's minimal post-processor
(beat_this/model/postprocessor.py: Postprocessor("minimal", fps) with its own deduplicate_peaks) and framewise truth
builder (prepare_annotations, beat_this/dataset/dataset.py:512-547) at frame rates other than 50.  Both are plain
torch / numpy and run on the CPU.

    BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_postp_fps.py

The reference's dataset module imports pytorch_lightning at the top for its data module, which prepare_annotations does
not use; when the package is absent a stand-in module with an empty LightningDataModule is registered first.

Contents:
- fps: the rates, as float64 (43.06640625 = 22050 / 512; the others are integers and are passed to the reference as
  Python ints, as a checkpoint's hyper-parameter would be).
- beat{k}, down{k}: fp32 logits of case k, shared by every rate: seeded sinusoids with noise, quantised logits (ties,
  plateaus, adjacent peaks), hand-made clips with downbeats halfway between two beats (argmin ties at some rates),
  merged peaks at half frames, downbeats without beats and clips without peaks.
- beat_times{r}_{k}, down_times{r}_{k}: the reference's output for case k at rate fps[r].
- pad_beat, pad_down [B, T], pad_mask [B, T] (trailing padding, large positive logits under it) and
  pad_beat_times{r}_{i}, pad_down_times{r}_{i}: the reference's batched call with the padding mask.
- truth_T{j}, truth_times{j}, truth_values{j}, and per rate truth_beat{r}_{j}, truth_down{r}_{j} (framewise, bool),
  truth_orig_beat{r}_{j}, truth_orig_down{r}_{j} (the unquantised times inside [0, T / fps)): prepare_annotations(item,
  0, T, fps) on times at and one ulp either side of the half-frame boundaries of every rate.
"""
from __future__ import annotations

import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if not os.environ.get("BEAT_THIS_REFERENCE"):
    sys.exit("usage: BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_postp_fps.py")
sys.path.insert(0, os.environ["BEAT_THIS_REFERENCE"])

import numpy as np
import torch

try:
    import pytorch_lightning  # noqa: F401
except ImportError:
    sys.modules["pytorch_lightning"] = types.SimpleNamespace(LightningDataModule=object)

from beat_this.dataset.dataset import prepare_annotations
from beat_this.model.postprocessor import Postprocessor  # the reference

GOLD = os.path.join(ROOT, "tests", "golden")
RATES = (10, 25, 22050 / 512, 86, 100, 200)


def logit_cases(rng):
    cases = []
    for T in (1, 5, 50, 300, 1501, 4000):
        t = np.arange(T)
        b = (2.5 * np.sin(2 * np.pi * t / rng.uniform(18, 40) + rng.uniform(0, 6)) + 0.7 * rng.standard_normal(T))
        d = (2.5 * np.sin(2 * np.pi * t / rng.uniform(70, 160) + rng.uniform(0, 6)) - 1.0 + 0.7 * rng.standard_normal(T))
        cases.append((b.astype(np.float32), d.astype(np.float32)))
    for T in (64, 500, 1501):  # quantised logits: ties, plateaus and runs of adjacent peaks
        cases.append((np.round(rng.standard_normal(T) * 1.5).astype(np.float32),
                      np.round(rng.standard_normal(T) * 1.5 - 0.5).astype(np.float32)))
    neg = np.full(100, -3.0, np.float32)
    cases.append((neg, neg.copy()))  # no peaks at all
    cases.append((np.full(100, 2.0, np.float32), np.full(100, 1.0, np.float32)))  # one plateau: every frame a peak
    # beats at 10, 20, 30 and 43, 44 (merged: 43.5), 100; downbeats halfway between beats, on a merged half frame,
    # next to the first beat and one with no beat nearby
    b = np.full(160, -5.0, np.float32)
    b[[10, 20, 30, 43, 44, 100]] = [3, 3, 3, 2, 2, 1]
    d = np.full(160, -5.0, np.float32)
    d[[15, 25, 37, 65, 72, 150]] = 1.0
    cases.append((b, d))
    for gap in (3, 7, 11, 13):  # every odd gap: downbeats exactly halfway between two beats, at many positions
        b = np.full(400, -4.0, np.float32)
        beats = np.arange(5, 390, 2 * gap)
        b[beats] = 2.0
        d = np.full(400, -4.0, np.float32)
        d[beats[:-1] + gap] = 1.5
        cases.append((b, d))
    b = np.full(50, -5.0, np.float32)
    d = b.copy()
    d[[5, 30]] = 2.0  # downbeats but no beats: nothing to snap to
    cases.append((b, d))
    return cases


def main():
    rng = np.random.default_rng(4306)
    out = {"fps": np.asarray(RATES, np.float64)}
    cases = logit_cases(rng)
    for k, (b, d) in enumerate(cases):
        out[f"beat{k}"], out[f"down{k}"] = b, d
    out["n"] = np.int64(len(cases))
    # a padded batch: trailing padding with logits that would be peaks if they were read
    lens = (700, 1, 333, 0, 1024)
    T = max(lens)
    pb = (2.5 * np.sin(np.arange(T) / rng.uniform(3, 6, (len(lens), 1))) + 0.5 * rng.standard_normal((len(lens), T)))
    pd = (2.5 * np.sin(np.arange(T) / rng.uniform(12, 20, (len(lens), 1))) - 1 + 0.5 * rng.standard_normal((len(lens), T)))
    mask = np.arange(T)[None, :] < np.asarray(lens)[:, None]
    pb = np.where(mask, pb, 50.0).astype(np.float32)
    pd = np.where(mask, pd, 50.0).astype(np.float32)
    out["pad_beat"], out["pad_down"], out["pad_mask"] = pb, pd, mask

    for r, fps in enumerate(RATES):
        fps = int(fps) if float(fps).is_integer() else fps
        post = Postprocessor("minimal", fps)
        for k, (b, d) in enumerate(cases):
            bt, dt = post(torch.tensor(b), torch.tensor(d))
            out[f"beat_times{r}_{k}"] = np.asarray(bt, np.float64)
            out[f"down_times{r}_{k}"] = np.asarray(dt, np.float64)
        bts, dts = post(torch.tensor(pb), torch.tensor(pd), torch.tensor(mask))
        for i, (bt, dt) in enumerate(zip(bts, dts)):
            out[f"pad_beat_times{r}_{i}"] = np.asarray(bt, np.float64)
            out[f"pad_down_times{r}_{i}"] = np.asarray(dt, np.float64)

    # framewise truth: times at and one ulp either side of every rate's half-frame boundaries, before 0 and past the end
    n_truth = 0
    for T in (1, 9, 160):
        parts = [rng.uniform(-0.2, T / 10 + 0.2, 40)]
        for fps in RATES:
            half = (np.arange(-2, T + 3) + 0.5) / fps
            parts += [half, np.nextafter(half, -1), np.nextafter(half, 2), np.arange(-1, T + 2) / fps]
        times = np.sort(np.concatenate(parts))
        values = rng.choice([1, 2, 3], len(times))
        out[f"truth_T{n_truth}"] = np.int64(T)
        out[f"truth_times{n_truth}"] = times
        out[f"truth_values{n_truth}"] = values.astype(np.int64)
        for r, fps in enumerate(RATES):
            fps = int(fps) if float(fps).is_integer() else fps
            beat, down, orig_b, orig_d = prepare_annotations({"beat_time": times, "beat_value": values}, 0, T, fps)
            out[f"truth_beat{r}_{n_truth}"] = np.asarray(beat, bool)
            out[f"truth_down{r}_{n_truth}"] = np.asarray(down, bool)
            out[f"truth_orig_beat{r}_{n_truth}"] = np.frombuffer(orig_b, np.float64)
            out[f"truth_orig_down{r}_{n_truth}"] = np.frombuffer(orig_d, np.float64)
        n_truth += 1
    out["n_truth"] = np.int64(n_truth)
    path = os.path.join(GOLD, "postp_fps.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {len(cases)} logit cases, {len(lens)} padded rows and {n_truth} truth cases at {len(RATES)} rates to {path}")


if __name__ == "__main__":
    main()
