"""Generate tests/golden/cli_beats.npz: the `.beats` files the UNMODIFIED reference writes for int16 WAV material.

Needs the reference's source tree, given by BEAT_THIS_REFERENCE:

    python oracle/make_golden_cli.py

The reference's own `load_audio` (beat_this/preprocessing.py:6-24) has no working decoder in this container
(torchcodec / soundfile / madmom are absent), so the decode step is the one every one of those backends performs for
16-bit PCM -- samples / 32768 as float64, channels last; everything after it is the reference:
`Audio2Beats(ckpt, "cpu", float16=False, dbn=False)(signal, sr)` (inference.py:215-322) and `save_beat_tsv`
(utils.py:85-102).  The test side regenerates the same WAV files from seeds, runs `python -m beat_this_b200.cli` on
them and compares the bytes of the files.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "shims"))
if not os.environ.get("BEAT_THIS_REFERENCE"):
    sys.exit("usage: BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_cli.py")
sys.path.insert(0, os.environ["BEAT_THIS_REFERENCE"])
sys.path.insert(0, ROOT)

import numpy as np
import torch

import beat_this.inference as ref_inf  # the reference
import beat_this.utils as ref_utils

from beat_this_b200 import synthetic

GOLD = os.path.join(ROOT, "tests", "golden")
torch.set_num_threads(8)

CLI_CASES, pcm16 = synthetic.CLI_CASES, synthetic.pcm16


def main():
    out = {}
    for model_name in ("small0", "final0"):
        path = synthetic.write_checkpoint(os.path.join("/tmp/bt_golden", f"{model_name}_s0.ckpt"), model_name, 0)
        a2b = ref_inf.Audio2Beats(path, "cpu", False, False)
        for k, (name, seed, secs, ch) in enumerate(CLI_CASES):
            signal = pcm16(seed, secs, ch).astype(np.float64) / 32768.0
            beats, downbeats = a2b(signal, 22050)
            with tempfile.TemporaryDirectory() as td, contextlib.redirect_stdout(io.StringIO()):
                ref_utils.save_beat_tsv(beats, downbeats, os.path.join(td, "x.beats"))
                text = open(os.path.join(td, "x.beats"), "rb").read()
            out[f"{model_name}_text{k}"] = np.frombuffer(text, dtype=np.uint8)
            out[f"{model_name}_beats{k}"] = np.asarray(beats, dtype=np.float64)
            out[f"{model_name}_downbeats{k}"] = np.asarray(downbeats, dtype=np.float64)
            print(f"{model_name} {name}: {len(beats)} beats, {len(downbeats)} downbeats, {len(text)} bytes")
        sd = torch.load(path, weights_only=True)["state_dict"]
        out[f"{model_name}_ckpt_sum"] = np.float64(synthetic.tensor_checksum({k.replace("model.", "").replace("_orig_mod.", ""): v for k, v in sd.items()}))
    np.savez_compressed(os.path.join(GOLD, "cli_beats.npz"), **out)


if __name__ == "__main__":
    main()
