"""Generate tests/golden/train_batches.npz by running the UNMODIFIED reference's BeatDataModule and BeatTrackingDataset
(beat_this/dataset/dataset.py, dataset/augment.py) on the CPU over the seeded tree of tests/dataset_reference.py.

    python oracle/make_golden_train_batches.py <beat_this source tree>

(or BEAT_THIS_REFERENCE=<tree>).  pytorch_lightning comes from oracle/shims (the data module only calls
save_hyperparameters from it); pandas reads the split files as in the reference.  Under numpy 2 the two private
numpy.lib.format helpers the reference's memory-mapped .npz reader calls are re-exported from where numpy 2 keeps them.

Recorded:
* split/<name>/{train,val,test}: the item lists of BeatDataModule(...).setup("fit") / setup("test") for each entry of
  SPLITS, split/<name>/train_len the train dataset's length, split/<name>/log everything the module printed, and
  split/<name>/pos_weights get_train_positive_weights() (beat, downbeat).
* for each entry of CONFIGS (dataset keyword arguments over ITEMS, or the test items for "full"):
  <cfg>/items the dataset's spect_path per item after skipping and oversampling, <cfg>/log its messages,
  <cfg>/seq the index sequence, and per drawn item j (np.random.seed(SEED + k) before the first):
  <cfg>/<j>/{spect (uint16 bits), truth_beat, truth_downbeat, padding_mask, start_frame, downbeat_mask, spect_path,
  dataset, truth_orig_beat, truth_orig_downbeat (float64)}.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys
import tempfile
from pathlib import Path

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("BEAT_THIS_REFERENCE")
if not REF:
    sys.exit("usage: python oracle/make_golden_train_batches.py <beat_this source tree>")
sys.path.insert(0, os.path.join(HERE, "shims"))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np

# numpy 2 moved the two private helpers the reference's MemmappedNpzFile calls (mmnpz.py:68-69) to _format_impl
if not hasattr(np.lib.format, "_check_version"):
    from numpy.lib import _format_impl

    np.lib.format._check_version = _format_impl._check_version
    np.lib.format._read_array_header = _format_impl._read_array_header

from beat_this.dataset.dataset import BeatDataModule, BeatTrackingDataset  # the reference

import dataset_reference as D

GOLD = os.path.join(ROOT, "tests", "golden")
SEED = 4000


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        root = D.write_tree(Path(tmp) / "data")
        for name, kw in D.SPLITS.items():
            log = io.StringIO()
            with contextlib.redirect_stdout(log):
                dm = BeatDataModule(root, train_length=D.TRAIN_LENGTH, augmentations=D.AUGMENTATIONS, **kw)
                dm.setup("fit")
                dm.setup("test")
                pw = dm.get_train_positive_weights()
            out[f"split/{name}/train"] = np.array(dm.train_items, dtype=str)
            out[f"split/{name}/val"] = np.array(dm.val_items, dtype=str)
            out[f"split/{name}/test"] = np.array(dm.test_items, dtype=str)
            out[f"split/{name}/train_len"] = np.int64(len(dm.train_dataset))
            out[f"split/{name}/pos_weights"] = np.array([pw["beat"], pw["downbeat"]], np.int64)
            out[f"split/{name}/log"] = np.array(log.getvalue())
        items = sorted(f"{d}/{p[0]}" for d, (_, _, ps) in D.DATASETS.items() if d != "gtzan" for p in ps)
        tests = sorted(f"gtzan/{p[0]}" for p in D.DATASETS["gtzan"][2])
        for k, (cfg, (kw, count)) in enumerate(D.CONFIGS.items()):
            kw = {"train_length": D.TRAIN_LENGTH, **kw}
            log = io.StringIO()
            with contextlib.redirect_stdout(log):
                ds = BeatTrackingDataset(tests if cfg == "full" else items, data_folder=root, spect_fps=D.FPS, **kw)
            out[f"{cfg}/items"] = np.array([str(it["spect_path"]) for it in ds.items], dtype=str)
            out[f"{cfg}/log"] = np.array(log.getvalue())
            seq = np.random.RandomState(k).randint(0, len(ds), count)
            out[f"{cfg}/seq"] = seq
            np.random.seed(SEED + k)
            for j, i in enumerate(seq):
                it = ds[int(i)]
                p = f"{cfg}/{j}/"
                out[p + "spect"] = np.ascontiguousarray(it["spect"]).view(np.uint16)
                for key in ("truth_beat", "truth_downbeat", "padding_mask"):
                    out[p + key] = np.asarray(it[key], bool)
                out[p + "start_frame"] = np.int64(it["start_frame"])
                out[p + "downbeat_mask"] = np.bool_(bool(it["downbeat_mask"]))
                out[p + "spect_path"] = np.array(it["spect_path"])
                out[p + "dataset"] = np.array(it["dataset"])
                out[p + "truth_orig_beat"] = np.frombuffer(it["truth_orig_beat"], np.float64)
                out[p + "truth_orig_downbeat"] = np.frombuffer(it["truth_orig_downbeat"], np.float64)
    path = os.path.join(GOLD, "train_batches.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes, {len(out)} arrays)")


if __name__ == "__main__":
    main()
