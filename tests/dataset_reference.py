"""The seeded data tree of the training-batch fixture (tests/golden/train_batches.npz, oracle/make_golden_train_batches.py)
and a numpy restatement of bt_train_batch's contract (include/beatthis.h).

``write_tree(root)`` writes the reference's prepared layout with every case its dataset code distinguishes: four
datasets (one without downbeats, one named ``rwc`` with sub-collections, one as loose .npy files instead of a bundle,
``gtzan`` as the test set), a one-column annotation file in a downbeat dataset, a piece that lacks one variant, pieces
shorter than, as long as and longer than TRAIN_LENGTH, beat times on half-frame boundaries and past a piece's end, and
both split files.  The same seed writes the same bytes.
"""
from __future__ import annotations

import contextlib
import io
import json
from pathlib import Path

import numpy as np

FPS = 50
TRAIN_LENGTH = 200
AUGMENTATIONS = {"pitch": {"min": -1, "max": 1}, "tempo": {"min": -4, "max": 4, "stride": 4}}
VARIANTS = ["track", "track_ps-1", "track_ps1", "track_ts-4", "track_ts4"]
ZERO_MASK = {"kind": "zero", "min_count": 1, "max_count": 3, "min_len": 0.1, "max_len": 1.0, "min_parts": 1,
             "max_parts": 1}
PERMUTE_MASK = {"kind": "permute", "min_count": 1, "max_count": 4, "min_len": 0.02, "max_len": 1.0, "min_parts": 1,
                "max_parts": 40}
# fixture configurations: (BeatTrackingDataset keyword arguments, number of items drawn)
CONFIGS = {
    "det": (dict(deterministic=True, augmentations={}), 8),
    "pt": (dict(augmentations=AUGMENTATIONS), 8),
    "zero": (dict(augmentations={"mask": ZERO_MASK}), 8),
    "permute": (dict(augmentations={"mask": PERMUTE_MASK}), 10),
    "all": (dict(augmentations={**AUGMENTATIONS, "mask": PERMUTE_MASK}), 8),
    "over": (dict(augmentations=AUGMENTATIONS, length_based_oversampling_factor=2), 6),
    "full": (dict(deterministic=True, augmentations={}, train_length=None), 4),
}
# BeatDataModule.setup arguments recorded by the fixture
SPLITS = {"single": {}, "fold0": {"fold": 0}, "fold3": {"fold": 3}, "hung": {"hung_data": True},
          "noval": {"no_val": True}}

# dataset -> (has_downbeats, stored as a bundle, pieces: (stem, frames, split part, fold))
DATASETS = {
    "ballroom": (True, True, [("Albums-Cafe_1", 150, "train", 0), ("Albums-Cafe_2", 200, "train", 1),
                              ("Albums-Cafe_3", 350, "val", 3), ("Albums-Cafe_4", 455, "train", 3),
                              ("Albums-Cafe_5", 240, "test", 2), ("Albums-Cafe_6", 300, "train", 0)]),
    "beatles": (False, False, [("01_Help", 260, "train", 0), ("02_Yesterday", 199, "val", 1),
                               ("03_Something", 420, "train", 3)]),
    "rwc": (True, True, [("rwc_popular_001", 330, "train", 0), ("rwc_popular_002", 201, "val", 0),
                         ("rwc_jazz_001", 280, "train", 3), ("rwc_classical_001", 120, "train", 5)]),
    "gtzan": (True, True, [("gtzan_rock_00001", 310, "test", 0), ("gtzan_jazz_00002", 180, "test", 1)]),
}
ONE_COLUMN = "ballroom/Albums-Cafe_6"  # a downbeat dataset piece annotated with beats only: skipped
MISSING_VARIANT = ("ballroom/Albums-Cafe_4", "track_ts4")  # skipped whenever tempo augmentation is on


def variant_frames(frames: int, variant: str) -> int:
    if "_ts" in variant:
        return int(round(frames / (1 + int(variant.split("_ts")[1]) / 100)))
    return frames


def spectrogram(rng, frames) -> np.ndarray:
    """Low-entropy float16 values (multiples of 1/4 in [-2, 2)), so the fixture compresses well."""
    return (rng.integers(-8, 8, (frames, 128)) / 4).astype(np.float16)


def beat_times(rng, frames):
    """(times, positions in the bar): a jittered grid from 0 s to past the end, some times on half-frame boundaries."""
    step = rng.uniform(0.3, 0.6)
    t = np.arange(0.0, frames / FPS + 1.0, step) + rng.uniform(0, 0.01)
    t[1::3] = np.floor(t[1::3] * FPS) / FPS + 0.5 / FPS  # k + 1/2 frames: numpy rounds half to even
    t = np.round(np.sort(t), 6)
    pos = 1 + (np.arange(len(t)) + int(rng.integers(0, 4))) % 4
    return t, pos


def write_tree(root, seed=0) -> Path:
    root = Path(root)
    rng = np.random.default_rng(seed)
    ann, spects = root / "annotations", root / "audio" / "spectrograms"
    for dataset, (has_down, bundled, pieces) in DATASETS.items():
        (ann / dataset / "annotations" / "beats").mkdir(parents=True, exist_ok=True)
        (ann / dataset / "info.json").write_text(json.dumps({"has_downbeats": has_down}))
        members = {}
        for stem, frames, part, fold in pieces:
            t, pos = beat_times(rng, frames)
            name = f"{dataset}/{stem}"
            path = ann / dataset / "annotations" / "beats" / f"{stem}.beats"
            if has_down and name != ONE_COLUMN:
                path.write_text("".join(f"{a}\t{b}\n" for a, b in zip(t, pos)))
            else:
                path.write_text("".join(f"{a}\n" for a in t))
            for v in VARIANTS:
                s = spectrogram(rng, variant_frames(frames, v))
                if (name, v) == MISSING_VARIANT:
                    continue
                if bundled:
                    members[f"{stem}/{v}"] = s
                else:
                    (spects / dataset / stem).mkdir(parents=True, exist_ok=True)
                    np.save(spects / dataset / stem / f"{v}.npy", s)
        if bundled:
            spects.mkdir(parents=True, exist_ok=True)
            np.savez(spects / f"{dataset}.npz", **members)
        if dataset != "gtzan":
            (ann / dataset / "single.split").write_text("".join(f"{s}\t{p}\n" for s, _, p, _ in pieces))
        (ann / dataset / "8-folds.split").write_text("".join(f"{s}\t{f}\n" for s, _, _, f in pieces))
    return root


# ---- bt_train_batch restated -----------------------------------------------------------------------------------------
def gather(window, row_map, length):
    """One item of a batch from its drawn window (n rows of 16-bit values, any dtype viewed as uint16) and row map (None:
    identity): ([length, 128] uint16 bits, with 0 for -1 rows and rows >= n)."""
    w = np.asarray(window).view(np.uint16)
    n = len(w)
    out = np.zeros((length, w.shape[1]), np.uint16)
    m = np.arange(n) if row_map is None else np.asarray(row_map)
    keep = m >= 0
    out[:n][keep] = w[m[keep]]
    return out


def targets(frames, n, length):
    """(framewise target, padding mask) of one item: bool [length]."""
    y = np.zeros(length, bool)
    y[np.asarray(frames, np.int64)] = True
    pad = np.arange(length) < n
    return y, pad


def apply_mask_reference(spect, mask, fps, rng):
    """augment_mask_ (reference augment.py:129-201) restated literally on an array, in place: the operations the row
    map must reproduce."""
    count = rng.randint(mask["min_count"], mask["max_count"] + 1)
    lo, hi = int(mask["min_len"] * fps), int(mask["max_len"] * fps)
    for _ in range(count):
        length = rng.randint(lo, hi + 1)
        start = rng.randint(0, len(spect) - length)
        ex = spect[start : start + length]
        if mask["kind"] == "permute":
            k = min(rng.randint(mask["min_parts"], mask["max_parts"] + 1), len(ex) + 1)
            pos = rng.choice(len(ex), k - 1, replace=False)
            pos.sort()
            parts = np.split(ex, pos)
            ex[:] = np.concatenate([parts[i] for i in rng.permutation(k)])
        else:
            ex[:] = 0
    return spect


# ---- the fixture's draws: the seed, the items and the datasets the dataset tests build
SEED = 4000  # oracle/make_golden_train_batches.py


def _items():
    return sorted(f"{d}/{p[0]}" for d, (_, _, ps) in DATASETS.items() if d != "gtzan" for p in ps)


def _tests():
    return sorted(f"gtzan/{p[0]}" for p in DATASETS["gtzan"][2])


def _dataset(tree, cfg):
    from beat_this_b200.dataset import BeatTrackingDataset

    kw = {"train_length": TRAIN_LENGTH, **CONFIGS[cfg][0]}
    log = io.StringIO()
    with contextlib.redirect_stdout(log):
        ds = BeatTrackingDataset(_tests() if cfg == "full" else _items(), tree, spect_fps=FPS, **kw)
    return ds, log.getvalue()
