"""Generate tests/golden/loss.npz by running the UNMODIFIED reference's losses (beat_this/model/loss.py) and framewise
truth builder (prepare_annotations, beat_this/dataset/dataset.py:512-534).  Both are plain torch / numpy and run on
the CPU.

    BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_loss.py

The reference's dataset module imports pytorch_lightning at the top for its data module, which prepare_annotations does
not use; when the package is absent a stand-in module with an empty LightningDataModule is registered first.

Per case k the fixture holds the module's inputs (preds, targets, optionally mask) and outputs (loss, preds.grad after
loss.backward()), and spec{k} = [kind, tolerance argument, pos_weight, has mask].  Cases cover the three loss classes,
tolerances 0, 1 and 3, pos_weight 1 and 4.5, no mask, bool, float and [B, 1] masks, binary and label-smoothed targets,
logits drawn from three values (ties everywhere: they pin which frame of a window receives the gradient), rows of
exactly 4t + 1 frames and [B, C, T] input.  truth{k}: prepare_annotations on beat times at and near half-frame
boundaries.
"""
from __future__ import annotations

import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if not os.environ.get("BEAT_THIS_REFERENCE"):
    sys.exit("usage: BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_loss.py")
sys.path.insert(0, os.environ["BEAT_THIS_REFERENCE"])

import numpy as np
import torch

try:
    import pytorch_lightning  # noqa: F401
except ImportError:
    sys.modules["pytorch_lightning"] = types.SimpleNamespace(LightningDataModule=object)

import beat_this.model.loss as ref_loss  # the reference
from beat_this.dataset.dataset import prepare_annotations

GOLD = os.path.join(ROOT, "tests", "golden")
CLASSES = (ref_loss.MaskedBCELoss, ref_loss.ShiftTolerantBCELoss, ref_loss.SplittedShiftTolerantBCELoss)


def main():
    rng = np.random.default_rng(2024)
    out = {}
    k = 0
    for kind, cls in enumerate(CLASSES):
        for t in ((0,) if kind == 0 else (0, 1, 3)):
            for pw in (1.0, 4.5):
                for mask_kind in ("none", "bool", "float", "b1"):
                    if kind == 2 and mask_kind == "none":
                        continue  # SplittedShiftTolerantBCELoss.forward requires the mask
                    for smooth in (False, True):
                        variant = k % 4  # 0: random logits, 1: tie-heavy, 2: rows of 4t + 1 frames, 3: [B, C, T]
                        B = int(rng.integers(1, 4))
                        T = 4 * t + 1 if variant == 2 else int(rng.integers(4 * t + 1, 4 * t + 40))
                        shape = (B, 2, T) if variant == 3 else (B, T)
                        if variant == 1:
                            preds = rng.choice(np.array([-1.5, 0.25, 2.0], np.float32), shape)
                        else:
                            preds = (rng.standard_normal(shape) * 2).astype(np.float32)
                        targets = (rng.random(shape) < 0.15).astype(np.float32)
                        if smooth:
                            targets = targets * 0.9 + 0.05
                        mshape = (B, 1) + ((1,) if variant == 3 else ()) if mask_kind == "b1" else shape
                        if mask_kind == "bool":
                            mask = torch.tensor(rng.random(mshape) < 0.8)
                        elif mask_kind == "float":
                            mask = torch.tensor(np.where(rng.random(mshape) < 0.2, 0.0, rng.random(mshape)).astype(np.float32))
                        elif mask_kind == "b1":
                            mask = torch.tensor(rng.random(mshape) < 0.6).float()
                            if kind == 2 or (kind == 1 and t > 0):  # these crop the mask's last dimension
                                mask = torch.ones(shape) * mask  # as _compute_loss forms it (pl_module.py:101)
                        else:
                            mask = None
                        module = cls(pos_weight=pw) if kind == 0 else cls(pos_weight=pw, tolerance=t)
                        x = torch.tensor(preds, requires_grad=True)
                        loss = module(x, torch.tensor(targets), mask) if mask is not None else module(x, torch.tensor(targets))
                        loss.backward()
                        out[f"spec{k}"] = np.array([kind, t, pw, mask is not None], np.float64)
                        out[f"preds{k}"] = preds
                        out[f"targets{k}"] = targets
                        if mask is not None:
                            out[f"mask{k}"] = mask.numpy()
                        out[f"loss{k}"] = np.float32(loss.item())
                        out[f"grad{k}"] = x.grad.numpy()
                        k += 1
    out["n"] = np.int64(k)
    # framewise truth: beat times at and one ulp either side of half-frame boundaries, before 0 and past the end
    n_truth = 0
    for T in (1, 7, 120):
        half = (np.arange(-2, T + 3) + 0.5) / 50
        times = np.sort(np.concatenate([half, np.nextafter(half, -1), np.nextafter(half, 2), rng.uniform(-0.1, T / 50 + 0.1, 20)]))
        values = rng.choice([1, 2, 3], len(times))
        item = {"beat_time": times, "beat_value": values}
        beat, down, _, _ = prepare_annotations(item, 0, T, 50)
        out[f"truth_T{n_truth}"] = np.int64(T)
        out[f"truth_times{n_truth}"] = times
        out[f"truth_values{n_truth}"] = values.astype(np.int64)
        out[f"truth_beat{n_truth}"] = np.asarray(beat, bool)
        out[f"truth_down{n_truth}"] = np.asarray(down, bool)
        n_truth += 1
    out["n_truth"] = np.int64(n_truth)
    np.savez_compressed(os.path.join(GOLD, "loss.npz"), **out)
    print(f"wrote {k} loss cases and {n_truth} truth cases to {os.path.join(GOLD, 'loss.npz')}")


if __name__ == "__main__":
    main()
