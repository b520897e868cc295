"""Generate tests/golden/chunking_modes.npz by running the UNMODIFIED reference's split_piece, aggregate_prediction
and split_predict_aggregate (beat_this/inference.py:100-230) on the CPU.

    BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_chunking_modes.py

Plans: for every chunk size c in {1500, 1000, 64, 2b + 1}, border b in {0, 1, 6, 100} with 2b < c, piece length
T in {1, 2b, c - 2b, c - 2b + 1, c, c + 1, 3c + 7} and both overlap modes, case k holds
case{k} = [T, c, b, mode (0 keep_first, 1 keep_last)], the chunk starts and lengths split_piece returns, and owner{k}:
aggregate_prediction over "predictions" that hold each chunk's own index, i.e. the chunk every frame is taken from
(-1000 would mark a frame no chunk covers).

Logits: split_predict_aggregate with the reference model of the seeded small0-shaped checkpoint
(beat_this_b200.synthetic) on the reference log-mel spectrogram of synth_clip(seed, seconds), for each (chunk_size,
border_size, overlap_mode) of LOGIT_SETTINGS and each clip of LOGIT_CLIPS.
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "shims"))
if not os.environ.get("BEAT_THIS_REFERENCE"):
    sys.exit("usage: BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_chunking_modes.py")
sys.path.insert(0, os.environ["BEAT_THIS_REFERENCE"])
sys.path.insert(0, ROOT)

import numpy as np
import torch

import beat_this.inference as ref_inf  # the reference
from beat_this.preprocessing import LogMelSpect as RefLogMelSpect

from beat_this_b200 import synthetic
from oracle import beat_this_oracle as O

GOLD = os.path.join(ROOT, "tests", "golden")
MODES = ("keep_first", "keep_last")
LOGIT_SETTINGS = [(1500, 0, "keep_first"), (1000, 6, "keep_last")]
LOGIT_CLIPS = [(40, 30.0), (41, 61.0)]  # (synth_clip seed, seconds): 1501 and 3051 frames


def sweep():
    """(T, chunk_size, border) of the plan sweep, each once."""
    out = []
    for b in (0, 1, 6, 100):
        for c in (1500, 1000, 64, 2 * b + 1):
            if 2 * b >= c:
                continue
            for T in sorted({1, 2 * b, c - 2 * b, c - 2 * b + 1, c, c + 1, 3 * c + 7}):
                if (T, c, b) not in out:
                    out.append((T, c, b))
    return out


def main():
    torch.set_num_threads(8)
    gold = {}
    k = 0
    for T, c, b in sweep():
        chunks, starts = ref_inf.split_piece(torch.zeros(T, 1), c, b, avoid_short_end=True)
        preds = [{"beat": torch.full((len(ch),), float(i)), "downbeat": torch.zeros(len(ch))} for i, ch in enumerate(chunks)]
        for m, mode in enumerate(MODES):
            owner, _ = ref_inf.aggregate_prediction(preds, starts, T, c, b, mode, "cpu")
            gold[f"case{k}"] = np.array([T, c, b, m], np.int64)
            gold[f"starts{k}"] = np.asarray(starts, np.int64)
            gold[f"lens{k}"] = np.array([len(ch) for ch in chunks], np.int64)
            gold[f"owner{k}"] = owner.numpy().astype(np.int32)
            k += 1
    gold["n"] = np.int64(k)

    path = synthetic.write_checkpoint("/tmp/bt_golden/small0_s0.ckpt", "small0", 0)
    model = ref_inf.load_model(path, "cpu")
    sd = O.strip_prefix(torch.load(path, weights_only=True)["state_dict"])
    gold["small0_ckpt_sum"] = np.float64(synthetic.tensor_checksum(sd))
    mel = RefLogMelSpect()
    gold["settings"] = np.array([[c, b, MODES.index(m)] for c, b, m in LOGIT_SETTINGS], np.int64)
    gold["clips"] = np.array(LOGIT_CLIPS, np.float64)
    for j, (seed, secs) in enumerate(LOGIT_CLIPS):
        spect = mel(torch.tensor(synthetic.synth_clip(seed, secs), dtype=torch.float32))
        for i, (c, b, mode) in enumerate(LOGIT_SETTINGS):
            with torch.inference_mode():
                pred = ref_inf.split_predict_aggregate(spect, c, b, mode, model)
            assert (pred["beat"] > -1000).all()
            gold[f"beat_s{i}_c{j}"] = pred["beat"].numpy()
            gold[f"down_s{i}_c{j}"] = pred["downbeat"].numpy()
    np.savez_compressed(os.path.join(GOLD, "chunking_modes.npz"), **gold)
    print(f"wrote {k} plan cases and {len(LOGIT_SETTINGS) * len(LOGIT_CLIPS)} logit cases to "
          f"{os.path.join(GOLD, 'chunking_modes.npz')}")


if __name__ == "__main__":
    main()
