"""Generate tests/golden/*.npz by running the UNMODIFIED reference (a beat_this source tree).

    BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden.py [live]

(`live`: only tests/golden/live_reference.npz, the reference model's forward on a random batch and its chunk
planner.)

It (1) imports the reference through the two import shims in oracle/shims/ (packages absent
offline: rotary_embedding_torch, soxr), (2) checks the oracle restatement
(oracle/beat_this_oracle.py) against the reference modules on the same seeded inputs and
prints the max-abs differences, and (3) writes the reference's own outputs as fixtures.

Inputs are regenerated from seeds by beat_this_b200.synthetic on the test side; every
fixture stores the checkpoint checksum so a generator drift is detected, not silently
compared.
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "shims"))
if not os.environ.get("BEAT_THIS_REFERENCE"):
    sys.exit("usage: BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden.py [live]")
sys.path.insert(0, os.environ["BEAT_THIS_REFERENCE"])
sys.path.insert(0, ROOT)

import numpy as np
import torch

import beat_this.inference as ref_inf  # the reference
from beat_this.model.postprocessor import Postprocessor as RefPostprocessor
from beat_this.preprocessing import LogMelSpect as RefLogMelSpect

from beat_this_b200 import synthetic
from oracle import beat_this_oracle as O

GOLD = os.path.join(ROOT, "tests", "golden")
os.makedirs(GOLD, exist_ok=True)
torch.set_num_threads(8)


def ref_model_from(name, seed, tmpdir="/tmp/bt_golden"):
    path = synthetic.write_checkpoint(os.path.join(tmpdir, f"{name}_s{seed}.ckpt"), name, seed)
    model = ref_inf.load_model(path, "cpu")  # strict load_state_dict: pins the ckpt layout
    sd = O.strip_prefix(torch.load(path, weights_only=True)["state_dict"])
    return path, model, sd


def main():
    report = {}
    # ---- 1. log-mel -------------------------------------------------------------------
    ref_mel = RefLogMelSpect()
    mels = {}
    for idx, secs in ((0, 3.0), (1, 10.0)):
        x = synthetic.synth_clip(idx, secs)
        xt = torch.tensor(x, dtype=torch.float32)
        m_ref = ref_mel(xt)
        m_or = O.logmel(xt)
        m64 = O.logmel(xt, torch.float64)
        report[f"mel{idx} oracle-vs-ref"] = float((m_ref - m_or).abs().max())
        report[f"mel{idx} ref-vs-f64"] = float((m_ref.double() - m64).abs().max())
        mels[f"clip{idx}_secs"] = np.float64(secs)
        mels[f"clip{idx}_mel"] = m_ref.numpy()
    fb_ref = ref_mel.spect_class.mel_scale.fb
    report["fb oracle-vs-ref"] = float((fb_ref - O.mel_filterbank()).abs().max())
    mels["fb_nnz"] = np.int64((fb_ref != 0).sum())
    np.savez_compressed(os.path.join(GOLD, "logmel.npz"), **mels)

    # ---- 2. chunking table (split_piece) ---------------------------------------------------
    Ts = [1, 7, 250, 251, 1488, 1489, 1494, 1500, 1501, 2976, 2977, 2982, 3001, 4464, 4465, 15001]
    table = {}
    for T in Ts:
        chunks, starts = ref_inf.split_piece(torch.zeros(T, 2), 1500, 6, True)
        table[f"starts_{T}"] = np.asarray(starts, dtype=np.int64)
        table[f"lens_{T}"] = np.asarray([len(c) for c in chunks], dtype=np.int64)
        assert np.array_equal(starts, O.split_starts(T)), T
        assert [len(c) for c in chunks] == [len(c) for c in O.split_piece(torch.zeros(T, 2))[0]]
    table["Ts"] = np.asarray(Ts, dtype=np.int64)
    np.savez_compressed(os.path.join(GOLD, "chunking.npz"), **table)

    # ---- 2b. function-level API: split_piece chunk CONTENTS and aggregate_prediction (both overlap modes), other
    # chunk sizes than 1500 / 6 included.  "Predictions" are the chunk's own first two columns, so the fixtures pin
    # exactly which chunk every output frame is taken from.
    host = {}
    cases = [(37, 16, 2), (100, 16, 2), (1501, 1500, 6), (3001, 1500, 6), (250, 1500, 6), (64, 20, 0), (95, 32, 5)]
    for k, (T, cs, bs) in enumerate(cases):
        g = torch.Generator().manual_seed(100 + k)
        sp = torch.rand(T, 3, generator=g) + 1.0
        chunks, starts = ref_inf.split_piece(sp, cs, bs, True)
        preds = [{"beat": c[:, 0] * (i + 1), "downbeat": c[:, 1] - i} for i, c in enumerate(chunks)]
        host[f"case{k}"] = np.asarray([T, cs, bs], dtype=np.int64)
        host[f"spect{k}"] = sp.numpy()
        host[f"starts{k}"] = np.asarray(starts, dtype=np.int64)
        host[f"chunks{k}"] = torch.cat(chunks).numpy()
        host[f"lens{k}"] = np.asarray([len(c) for c in chunks], dtype=np.int64)
        for mode in ("keep_first", "keep_last"):
            b, d = ref_inf.aggregate_prediction(preds, starts, T, cs, bs, mode, "cpu")
            host[f"{mode}_beat{k}"] = b.numpy()
            host[f"{mode}_down{k}"] = d.numpy()
    host["n"] = np.int64(len(cases))
    np.savez_compressed(os.path.join(GOLD, "host_api.npz"), **host)

    # ---- 2c. .beats writer (reference beat_this/utils.py:26-102): beat numbers and the exact file text for seeded
    # beat / downbeat sets incl. pickup bars, a pickup longer than the first bar, fewer than two downbeats, no beats
    import contextlib
    import io
    import tempfile

    import beat_this.utils as ref_utils

    rng = np.random.default_rng(21)
    tsv = {}
    sets = []
    for _ in range(6):  # regular material: random tempo, random bar length, random pickup
        n = int(rng.integers(8, 60))
        beats = np.cumsum(rng.uniform(0.3, 0.9, n)).round(2)
        bar = int(rng.integers(2, 6))
        first = int(rng.integers(0, bar + 3))
        sets.append((beats, beats[first::bar]))
    b = np.arange(12) * 0.5
    sets += [(b, b[5:6]), (b, b[:0]), (b, b[7::2]), (b[:0], b[:0]), (b, b[[0, 3, 7, 9]]), (b[:1], b[:1])]
    for k, (beats, downs) in enumerate(sets):
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            numbers = ref_utils.infer_beat_numbers(beats, downs)
        with tempfile.TemporaryDirectory() as td, contextlib.redirect_stdout(io.StringIO()):
            ref_utils.save_beat_tsv(beats, downs, os.path.join(td, "x.beats"))
            text = open(os.path.join(td, "x.beats")).read()
        tsv[f"beats{k}"] = np.asarray(beats, dtype=np.float64)
        tsv[f"downs{k}"] = np.asarray(downs, dtype=np.float64)
        tsv[f"numbers{k}"] = np.asarray(numbers, dtype=np.int64)
        tsv[f"text{k}"] = np.frombuffer(text.encode(), dtype=np.uint8)
        tsv[f"warned{k}"] = np.int64(1 if out.getvalue().strip() else 0)
    tsv["n"] = np.int64(len(sets))
    np.savez_compressed(os.path.join(GOLD, "beats_tsv.npz"), **tsv)

    # ---- 3. minimal postprocessor known-answer cases --------------------------------------------
    post = RefPostprocessor("minimal")
    rng = np.random.default_rng(7)
    cases = {}
    n_case = 0

    def add_case(b, d):
        nonlocal n_case
        bt, dt = post(torch.tensor(b), torch.tensor(d))
        ob, od = O.postp_minimal(torch.tensor(b), torch.tensor(d))
        assert np.array_equal(bt, ob) and np.array_equal(dt, od), n_case
        cases[f"beat_{n_case}"] = b
        cases[f"down_{n_case}"] = d
        cases[f"beat_times_{n_case}"] = np.asarray(bt, dtype=np.float64)
        cases[f"down_times_{n_case}"] = np.asarray(dt, dtype=np.float64)
        n_case += 1

    for T in (1, 5, 50, 300, 1501, 1501, 4000):
        t = np.arange(T)
        b = (2.5 * np.sin(2 * np.pi * t / rng.uniform(18, 40) + rng.uniform(0, 6))
             + 0.7 * rng.standard_normal(T)).astype(np.float32)
        d = (2.5 * np.sin(2 * np.pi * t / rng.uniform(70, 160) + rng.uniform(0, 6)) - 1.0
             + 0.7 * rng.standard_normal(T)).astype(np.float32)
        add_case(b, d)
    # ties / plateaus / adjacent peaks (quantised logits), all-negative, all-positive-constant
    for T in (64, 500, 1501):
        b = np.round(rng.standard_normal(T) * 1.5).astype(np.float32)
        d = np.round(rng.standard_normal(T) * 1.5 - 0.5).astype(np.float32)
        add_case(b, d)
    add_case(np.full(100, -3.0, np.float32), np.full(100, -3.0, np.float32))
    add_case(np.full(100, 2.0, np.float32), np.full(100, 1.0, np.float32))
    b = np.full(200, -5.0, np.float32); d = b.copy()
    b[[10, 11, 12, 40, 41, 90, 150]] = [3, 3, 3, 2, 2, 1, 4]
    d[[9, 60, 61, 62, 63, 149]] = 1.0  # snapping incl. equidistant tie and a downbeat without beats nearby
    add_case(b, d)
    b = np.full(50, -5.0, np.float32); d = b.copy(); d[[5, 30]] = 2.0  # downbeats but no beats
    add_case(b, d)
    cases["n"] = np.int64(n_case)
    np.savez_compressed(os.path.join(GOLD, "postp_minimal.npz"), **cases)

    # ---- 4. model / end-to-end ---------------------------------------------------------
    gold = {}
    # 4a. BASELINE config 1: Spect2Frames small0, one random 1500-frame spectrogram (2 chunks)
    path, model, sd = ref_model_from("small0", 0)
    torch.manual_seed(0)
    spect = torch.rand(1500, 128) * 7
    s2f = ref_inf.Spect2Frames(path, "cpu", False)
    rb, rd = s2f(spect)
    ob, od = O.spect2frames(sd, spect)
    report["small0 spect2frames oracle-vs-ref"] = float(max((rb - ob).abs().max(), (rd - od).abs().max()))
    gold["small0_ckpt_sum"] = np.float64(synthetic.tensor_checksum(sd))
    gold["small0_spect1500_beat"] = rb.numpy()
    gold["small0_spect1500_down"] = rd.numpy()

    # per-stage check of the oracle against reference module hooks (one short chunk)
    taps = {}
    xs = torch.rand(1, 200, 128) * 7
    with torch.inference_mode():
        ref_out = model(xs)
        b2, d2 = O.forward(sd, xs, taps)
        e_b, e_d = O.forward(sd, xs, explicit=True)
        ref_front = model.frontend(xs)
    report["small0 forward oracle-vs-ref"] = float(max((ref_out["beat"] - b2).abs().max(), (ref_out["downbeat"] - d2).abs().max()))
    report["small0 explicit-softmax vs sdpa"] = float((e_b - b2).abs().max())
    report["small0 frontend tap vs ref"] = float((ref_front - taps["frontend"]).abs().max())

    # 4a'. ablation families (reference README.md:86-101): Head instead of SumHead, no partial transformers
    for variant in ("small0-nosum", "small0-nopartial"):
        vpath, vmodel, vsd = ref_model_from(variant, 0)
        vhp = synthetic.model_hparams(variant)
        torch.manual_seed(5)
        vspect = torch.rand(1700, 128) * 7  # 2 chunks
        vb, vd = ref_inf.Spect2Frames(vpath, "cpu", False)(vspect)
        vob, vod = O.spect2frames(vsd, vspect, sum_head=vhp["sum_head"])
        report[f"{variant} spect2frames oracle-vs-ref"] = float(max((vb - vob).abs().max(), (vd - vod).abs().max()))
        key = variant.replace("-", "_")
        gold[f"{key}_ckpt_sum"] = np.float64(synthetic.tensor_checksum(vsd))
        gold[f"{key}_spect1700_beat"] = vb.numpy()
        gold[f"{key}_spect1700_down"] = vd.numpy()

    # 4b. final0-shaped: Audio2Frames / Audio2Beats on a 10 s clip (1 short chunk) and a 30 s clip (2 chunks)
    path, model, sd = ref_model_from("final0", 0)
    a2b = ref_inf.Audio2Beats(path, "cpu", False, False)
    gold["final0_ckpt_sum"] = np.float64(synthetic.tensor_checksum(sd))
    for idx, secs in ((1, 10.0), (2, 30.0)):
        x = synthetic.synth_clip(idx, secs)
        rb, rd = ref_inf.Audio2Frames.__call__(a2b, x, 22050)
        bt, dt = a2b.frames2beats(rb, rd)
        ob, od = O.spect2frames(sd, O.signal2spect(x, 22050))
        report[f"final0 clip{idx} ({secs}s) frames oracle-vs-ref"] = float(max((rb - ob).abs().max(), (rd - od).abs().max()))
        obt, odt = O.postp_minimal(ob, od)
        report[f"final0 clip{idx} beats identical"] = bool(np.array_equal(bt, obt) and np.array_equal(dt, odt))
        gold[f"final0_clip{idx}_secs"] = np.float64(secs)
        gold[f"final0_clip{idx}_beat"] = rb.numpy()
        gold[f"final0_clip{idx}_down"] = rd.numpy()
        gold[f"final0_clip{idx}_beat_times"] = np.asarray(bt, dtype=np.float64)
        gold[f"final0_clip{idx}_down_times"] = np.asarray(dt, dtype=np.float64)
    # stereo input (mono mix path, inference.py:270-271)
    x = synthetic.synth_clip(3, 4.0)
    xs2 = np.stack([x, 0.5 * x[::-1]], axis=1)
    rb, rd = ref_inf.Audio2Frames.__call__(a2b, xs2, 22050)
    gold["final0_stereo4s_beat"] = rb.numpy()
    gold["final0_stereo4s_down"] = rd.numpy()
    np.savez_compressed(os.path.join(GOLD, "model.npz"), **gold)

    with open(os.path.join(GOLD, "REPORT.txt"), "w") as f:
        f.write("oracle restatement vs UNMODIFIED reference (max-abs), written by oracle/make_golden.py\n")
        for k, v in report.items():
            line = f"{k}: {v}"
            print(line)
            f.write(line + "\n")


def write_live_reference(tmpdir="/tmp/bt_golden"):
    """The reference model (small0) on a seeded random [2, 100, 128] batch, and its chunk starts for a few lengths:
    what tests/test_cpu_oracle.py::test_oracle_against_reference_forward compares the oracle with."""
    _, model, sd = ref_model_from("small0", 0, tmpdir)
    torch.manual_seed(4)
    x = torch.rand(2, 100, 128) * 7
    with torch.inference_mode():
        ref = model(x)
    gold = {"small0_ckpt_sum": np.float64(synthetic.tensor_checksum(sd)), "beat": ref["beat"].numpy(),
            "downbeat": ref["downbeat"].numpy(), "Ts": np.array([1, 1488, 1489, 3001], dtype=np.int64)}
    for T in gold["Ts"]:
        _, starts = ref_inf.split_piece(torch.zeros(int(T), 1), 1500, 6, True)
        gold[f"starts_{T}"] = np.asarray(starts, dtype=np.int64)
    np.savez_compressed(os.path.join(GOLD, "live_reference.npz"), **gold)


if __name__ == "__main__":
    if sys.argv[1:] == ["live"]:
        write_live_reference()
    else:
        main()
        write_live_reference()
