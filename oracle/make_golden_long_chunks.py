"""Generate tests/golden/long_chunks.npz by running the UNMODIFIED reference's split_piece, aggregate_prediction,
split_predict_aggregate (beat_this/inference.py:100-230) and BeatThis.forward (model/beat_tracker.py:188-192) on the
CPU with chunks longer than 1500 frames: the sequence length of a model trained with another --train-length.

    BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_long_chunks.py

Plans: for every chunk size c in {1501, 3000, 4500, 8000}, border b in {0, 6, 100} and piece length T in
{1, c - 2b, c - 2b + 1, c, c + 1, 3c + 7} (and 30 001 frames, a 10-minute piece, at c = 8000), both overlap modes:
case{k} = [T, c, b, mode (0 keep_first, 1 keep_last)], the chunk starts and lengths split_piece returns, and owner{k},
aggregate_prediction over "predictions" that hold each chunk's own index.

Logits: for the seeded small0- and final0-shaped checkpoints (beat_this_b200.synthetic) and the reference log-mel
spectrogram of synth_clip(seed, seconds) for each clip of CLIPS (3 051 and 7 501 frames), split_predict_aggregate at
each (chunk_size, border_size, overlap_mode) of SETTINGS; the last one is longer than both pieces, so each runs as one
sequence.  Forward: BeatThis.forward on torch.rand(2, 3000, 128, generator=manual_seed(FORWARD_SEED)) * 7.  The fixture
holds seeds and lengths instead of the inputs, which the tests rebuild from them.
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "shims"))
if not os.environ.get("BEAT_THIS_REFERENCE"):
    sys.exit("usage: BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_long_chunks.py")
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
MODELS = ("small0", "final0")
SETTINGS = [(3000, 6, "keep_first"), (3000, 0, "keep_last"), (4500, 12, "keep_first"), (8000, 0, "keep_first")]
CLIPS = [(80, 61.0), (81, 150.0)]  # (synth_clip seed, seconds): 3 051 and 7 501 frames
FORWARD_SEED, FORWARD_SHAPE = 82, (2, 3000, 128)


def sweep():
    """(T, chunk_size, border) of the plan sweep, each once."""
    out = []
    for c in (1501, 3000, 4500, 8000):
        for b in (0, 6, 100):
            Ts = {1, c - 2 * b, c - 2 * b + 1, c, c + 1, 3 * c + 7} | ({30001} if c == 8000 else set())
            out += [(T, c, b) for T in sorted(Ts)]
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

    mel = RefLogMelSpect()
    spects = [mel(torch.tensor(synthetic.synth_clip(seed, secs), dtype=torch.float32)) for seed, secs in CLIPS]
    gold["settings"] = np.array([[c, b, MODES.index(m)] for c, b, m in SETTINGS], np.int64)
    gold["clips"] = np.array(CLIPS, np.float64)
    gold["clip_frames"] = np.array([s.shape[0] for s in spects], np.int64)
    gold["forward_seed"] = np.int64(FORWARD_SEED)
    x = torch.rand(*FORWARD_SHAPE, generator=torch.Generator().manual_seed(FORWARD_SEED)) * 7
    for name in MODELS:
        path = synthetic.write_checkpoint(f"/tmp/bt_golden/{name}_s0.ckpt", name, 0)
        model = ref_inf.load_model(path, "cpu")
        sd = O.strip_prefix(torch.load(path, weights_only=True)["state_dict"])
        gold[f"{name}_ckpt_sum"] = np.float64(synthetic.tensor_checksum(sd))
        with torch.inference_mode():
            out = model(x)
            gold[f"{name}_forward_beat"] = out["beat"].numpy()
            gold[f"{name}_forward_down"] = out["downbeat"].numpy()
            for j, spect in enumerate(spects):
                for i, (c, b, mode) in enumerate(SETTINGS):
                    pred = ref_inf.split_predict_aggregate(spect, c, b, mode, model)
                    assert (pred["beat"] > -1000).all()
                    gold[f"{name}_beat_s{i}_c{j}"] = pred["beat"].numpy()
                    gold[f"{name}_down_s{i}_c{j}"] = pred["downbeat"].numpy()
        print(f"{name}: forward and {len(SETTINGS) * len(CLIPS)} logit cases done", flush=True)
    path = os.path.join(GOLD, "long_chunks.npz")
    np.savez_compressed(path, **gold)
    print(f"wrote {k} plan cases and the logits of {len(MODELS)} models to {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
