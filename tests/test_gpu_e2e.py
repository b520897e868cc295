"""End-to-end GPU parity against the reference's own outputs (tests/golden/model.npz, written by
oracle/make_golden.py from the UNMODIFIED reference) and against the CPU oracle on ragged batches."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from numerics import F32_TOL, H16_TOL

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _gold():
    return np.load(os.path.join(GOLDEN, "model.npz"))


def _check_ckpt(path, key):
    from beat_this_b200 import synthetic
    from oracle import beat_this_oracle as O

    sd = O.strip_prefix(torch.load(path, weights_only=True)["state_dict"])
    assert abs(synthetic.tensor_checksum(sd) - float(_gold()[key])) < 1e-6 * abs(float(_gold()[key])), (
        "synthetic checkpoint drifted from the one the golden fixtures were generated with"
    )


def _assert_timestamps(ref_logits, our_logits, ref_times, our_times, err, what):
    """north_star: "beat/downbeat timestamp arrays identical after the deterministic postprocessor".  The peak
    picker is bit exact on identical logits (test_peakpick_golden_bit_exact); with logits that differ by `err`, a frame
    may only change its peak decision where the REFERENCE's own decision margin at that frame (distance to the `> 0`
    threshold or to the competing maximum in the +-3 window, postprocessor.py:95-99) is below 2*err.  Anything else is
    a failure; where no such frame exists the arrays must be identical."""
    import sys

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import peak_mismatch_report

    rep = peak_mismatch_report(np.asarray(ref_logits), np.asarray(our_logits), ref_times, our_times, err)
    print(f"  {what}: timestamps identical {rep['times_identical']}, peak frames differing {rep['frames_differing']}, "
          f"not explained by the margin {rep['unexplained']} (logit err {err:.2e})")
    assert rep["unexplained"] == 0, (what, rep)
    if rep["frames_differing"] == 0:
        assert rep["times_identical"], (what, rep)
    return rep


@pytest.mark.parametrize("float16", [False, True])
def test_config1_spect2frames_small0(small0_ckpt, lib_built, float16):
    """BASELINE config 1: Spect2Frames small0 on one random 1500-frame spectrogram (2 chunks)."""
    from beat_this_b200.inference import Spect2Frames

    _check_ckpt(small0_ckpt, "small0_ckpt_sum")
    g = _gold()
    torch.manual_seed(0)
    spect = torch.rand(1500, 128) * 7
    s2f = Spect2Frames(small0_ckpt, "cuda:0", float16)
    beat, down = s2f(spect.cuda())
    assert isinstance(beat, torch.Tensor) and beat.dtype == torch.float32 and beat.shape == (1500,) and beat.is_cuda
    eb = np.abs(beat.cpu().numpy() - g["small0_spect1500_beat"]).max()
    ed = np.abs(down.cpu().numpy() - g["small0_spect1500_down"]).max()
    print(f"small0 spect1500 float16={float16}: max abs err beat {eb:.3e} downbeat {ed:.3e}")
    assert max(eb, ed) < (H16_TOL if float16 else F32_TOL)


@pytest.mark.parametrize("float16", [False, True])
@pytest.mark.parametrize("variant", ["small0-nosum", "small0-nopartial"])
def test_ablation_checkpoint_families_golden(variant, lib_built, float16):
    """Checkpoints trained without the SumHead / without the partial transformers (reference README.md:86-101)
    load and match the reference's Spect2Frames output (fixture from oracle/make_golden.py)."""
    from conftest import ckpt_path
    from beat_this_b200.inference import Spect2Frames

    path = ckpt_path(variant)
    key = variant.replace("-", "_")
    _check_ckpt(path, f"{key}_ckpt_sum")
    g = _gold()
    torch.manual_seed(5)
    spect = torch.rand(1700, 128) * 7
    beat, down = Spect2Frames(path, "cuda:0", float16)(spect.cuda())
    eb = np.abs(beat.cpu().numpy() - g[f"{key}_spect1700_beat"]).max()
    ed = np.abs(down.cpu().numpy() - g[f"{key}_spect1700_down"]).max()
    print(f"{variant} spect1700 float16={float16}: max abs err beat {eb:.3e} downbeat {ed:.3e}")
    assert max(eb, ed) < (H16_TOL if float16 else F32_TOL)


@pytest.mark.parametrize("float16", [False, True])
def test_final0_audio2beats_golden(final0_ckpt, lib_built, float16):
    """Audio2Frames / Audio2Beats, final0-shaped checkpoint, 10 s (one short chunk) and 30 s
    (two 1500-frame chunks) clips, against the reference's own logits and timestamps."""
    from beat_this_b200 import synthetic
    from beat_this_b200.inference import Audio2Beats, Audio2Frames

    _check_ckpt(final0_ckpt, "final0_ckpt_sum")
    g = _gold()
    a2b = Audio2Beats(final0_ckpt, "cuda:0", float16)
    for idx in (1, 2):
        x = synthetic.synth_clip(idx, float(g[f"final0_clip{idx}_secs"]))
        beat, down = Audio2Frames.__call__(a2b, x, 22050)
        rb, rd = g[f"final0_clip{idx}_beat"], g[f"final0_clip{idx}_down"]
        assert beat.shape == rb.shape
        eb = np.abs(beat.cpu().numpy() - rb).max()
        ed = np.abs(down.cpu().numpy() - rd).max()
        print(f"final0 clip{idx} float16={float16}: max abs err beat {eb:.3e} downbeat {ed:.3e}")
        assert max(eb, ed) < (H16_TOL if float16 else F32_TOL)
        bt, dt = a2b(x, 22050)
        assert bt.dtype == np.float64 and dt.dtype == np.float64
        rep_b = _assert_timestamps(rb, beat.cpu().numpy(), g[f"final0_clip{idx}_beat_times"], bt, eb, f"clip{idx} beats ({len(bt)})")
        rep_d = _assert_timestamps(rd, down.cpu().numpy(), g[f"final0_clip{idx}_down_times"], dt, ed, f"clip{idx} downbeats ({len(dt)})")
        if not float16:  # fp32 path: identical, full stop
            assert rep_b["times_identical"] and rep_d["times_identical"]
    # stereo input -> mono mix (inference.py:270-271)
    x = synthetic.synth_clip(3, 4.0)
    xs2 = np.stack([x, 0.5 * x[::-1]], axis=1)
    beat, down = Audio2Frames.__call__(a2b, xs2, 22050)
    e = max(np.abs(beat.cpu().numpy() - g["final0_stereo4s_beat"]).max(), np.abs(down.cpu().numpy() - g["final0_stereo4s_down"]).max())
    print(f"final0 stereo 4 s float16={float16}: max abs err {e:.3e}")
    assert e < (H16_TOL if float16 else F32_TOL)
    with pytest.raises(ValueError):
        a2b(np.zeros((10, 2, 2)), 22050)


@pytest.mark.parametrize("float16", [False, True])
def test_ragged_batch_vs_oracle(small0_ckpt, lib_built, float16):
    """Variable-length clips in one call (BASELINE config 5 shape, small): 1..3 chunks per
    clip, short (T+12) and full chunks mixed; compared with the CPU oracle clip by clip."""
    from beat_this_b200 import synthetic
    from beat_this_b200.inference import Audio2Beats, Audio2Frames
    from oracle import beat_this_oracle as O

    sd = O.strip_prefix(torch.load(small0_ckpt, weights_only=True)["state_dict"])
    secs = [5.0, 29.7, 30.0, 61.3, 12.34, 5.0]
    clips = [synthetic.synth_clip(10 + i, s) for i, s in enumerate(secs)]
    a2b = Audio2Beats(small0_ckpt, "cuda:0", float16)
    frames = Audio2Frames.batch(a2b, clips, 22050)
    beats = a2b.batch(clips, 22050)
    worst = 0.0
    for x, (b, d), (bt, dt) in zip(clips, frames, beats):
        ob, od = O.spect2frames(sd, O.signal2spect(x, 22050))
        assert b.shape == ob.shape
        e = max((b.cpu() - ob).abs().max().item(), (d.cpu() - od).abs().max().item())
        worst = max(worst, e)
        obt, odt = O.postp_minimal(b.cpu(), d.cpu())  # oracle postprocessor on OUR logits: must be bit exact
        assert np.array_equal(bt, obt) and np.array_equal(dt, odt)
    print(f"ragged batch float16={float16}: worst max abs logit err {worst:.3e}")
    assert worst < (H16_TOL if float16 else F32_TOL)


@pytest.mark.parametrize("float16", [False, True])
def test_wave_size_does_not_change_results(small0_ckpt, lib_built, float16):
    """Chunks are processed in waves of equal-length chunks (bt_set_wave_chunks): 1-, 2- and 128-chunk waves
    over a ragged batch (9 chunks of two lengths) must give bit-identical logits -- every chunk is independent
    and the persistent kernels walk the tiles in a fixed order."""
    from beat_this_b200 import synthetic
    from beat_this_b200.inference import Audio2Frames

    secs = [61.3, 5.0, 30.0, 95.0, 12.34]
    clips = [synthetic.synth_clip(30 + i, s) for i, s in enumerate(secs)]
    a2f = Audio2Frames(small0_ckpt, "cuda:0", float16)
    ref = None
    for wave in (128, 2, 1):
        a2f.model.engine.set_wave_chunks(wave)
        out = [(b.cpu().clone(), d.cpu().clone()) for b, d in a2f.batch(clips, 22050)]
        if ref is None:
            ref = out
            continue
        for (b, d), (rb, rd) in zip(out, ref):
            assert torch.equal(b, rb) and torch.equal(d, rd), wave


def test_audio_at_44k1_goes_through_the_device_resampler(small0_ckpt, lib_built):
    """Audio2Beats with sr != 22050 (reference inference.py:274-275): device resampler + the usual path must equal
    the oracle pipeline run on the float64 direct-form resampling of the same signal."""
    from beat_this_b200 import synthetic
    from beat_this_b200.inference import Audio2Beats, Audio2Frames
    from oracle import beat_this_oracle as O

    sd = O.strip_prefix(torch.load(small0_ckpt, weights_only=True)["state_dict"])
    x = synthetic.synth_clip(77, 12.0, sr=44100)
    stereo = np.stack([x, 0.25 * x[::-1]], axis=1)
    a2b = Audio2Beats(small0_ckpt, "cuda:0", False)
    for sig in (x, stereo):
        beat, down = Audio2Frames.__call__(a2b, sig, 44100)
        mono = sig if sig.ndim == 1 else sig.mean(1)
        ob, od = O.spect2frames(sd, O.signal2spect(O.resample_direct(mono, 44100), 22050))
        assert beat.shape == ob.shape
        e = max((beat.cpu() - ob).abs().max().item(), (down.cpu() - od).abs().max().item())
        print(f"44.1 kHz clip ndim={sig.ndim}: max abs logit err vs oracle pipeline {e:.3e}")
        assert e < F32_TOL
        bt, dt = a2b(sig, 44100)
        obt, odt = O.postp_minimal(beat.cpu(), down.cpu())
        assert np.array_equal(bt, obt) and np.array_equal(dt, odt)


def test_no_cpu_fallback(small0_ckpt, lib_built):
    from beat_this_b200.inference import Spect2Frames

    with pytest.raises(RuntimeError):
        Spect2Frames(small0_ckpt, "cpu")


def test_grouped_pipeline_equals_single_calls(small0_ckpt, lib_built, monkeypatch):
    """batch() cuts a call into groups that flow through the staging / copy / compute ring (pipeline.py); group
    boundaries, ring reuse and input dtype / layout must not change any result: tiny groups (2 clips) over 9 clips ==
    one clip per call."""
    import beat_this_b200.inference as I
    from beat_this_b200 import synthetic

    a2b = I.Audio2Beats(small0_ckpt, "cuda:0", True)
    base = [synthetic.synth_clip(30 + i, 6.0 + 1.7 * i) for i in range(9)]
    clips = [c if i % 3 else c.astype(np.float32) for i, c in enumerate(base)]
    clips[4] = np.stack([clips[4], 0.5 * clips[4][::-1]], axis=1)  # one stereo clip
    single = [a2b(c, 22050) for c in clips]
    monkeypatch.setattr(I, "GROUP_CHUNKS", 2)
    grouped = a2b.batch(clips, 22050)
    frames_g = I.Audio2Frames.batch(a2b, clips, 22050)
    for c, (b, d), (gb, gd), (fb, fd) in zip(clips, single, grouped, frames_g):
        assert np.array_equal(b, gb) and np.array_equal(d, gd)
        sb, sd_ = I.Audio2Frames.__call__(a2b, c, 22050)
        assert torch.equal(sb, fb) and torch.equal(sd_, fd)
    # an error inside a group surfaces and leaves the pipeline usable
    with pytest.raises(Exception):
        a2b.batch(clips[:3] + [np.zeros(100)], 22050)
    again = a2b.batch(clips[:2], 22050)
    assert np.array_equal(again[0][0], single[0][0]) and np.array_equal(again[1][1], single[1][1])


def test_file2beats_and_file2file(small0_ckpt, lib_built, tmp_path):
    """File2Beats / File2File on int16 WAV files (BASELINE config 3 shape, tiny): same beats as feeding
    the decoded samples to Audio2Beats, and the .beats TSV the reference's save_beat_tsv would write."""
    from scipy.io import wavfile

    from beat_this_b200 import synthetic
    from beat_this_b200.inference import Audio2Beats, File2Beats, File2File
    from beat_this_b200.preprocessing import load_audio

    paths = []
    for i, secs in enumerate((6.0, 9.5)):
        x = synthetic.synth_clip(40 + i, secs)
        p = tmp_path / f"clip{i}.wav"
        wavfile.write(p, 22050, np.round(x * 32767).astype(np.int16))
        paths.append(p)
    f2b = File2Beats(small0_ckpt, "cuda:0", float16=False)
    a2b = Audio2Beats(small0_ckpt, "cuda:0", float16=False)
    batch = f2b.batch(paths)
    for p, (bb, bd) in zip(paths, batch):
        sig, sr = load_audio(p)
        assert sr == 22050 and sig.dtype == np.float64
        b1, d1 = f2b(p)
        b2, d2 = a2b(sig, sr)
        assert np.array_equal(b1, b2) and np.array_equal(d1, d2)
        assert np.array_equal(b1, bb) and np.array_equal(d1, bd)
    # mixed tree through the native WAV front door: stereo, another sample rate, a broken file with on_error="skip"
    x = synthetic.synth_clip(45, 5.0, sr=44100)
    stereo = np.stack([np.round(x * 32767), np.round(0.3 * x[::-1] * 32767)], axis=1).astype(np.int16)
    wavfile.write(tmp_path / "st44.wav", 44100, stereo)
    (tmp_path / "broken.wav").write_bytes(b"RIFF0000WAVEjunk")
    mixed = f2b.batch([paths[1], tmp_path / "st44.wav", tmp_path / "broken.wav", paths[0]], on_error="skip")
    assert mixed[2] is None
    sig, sr = load_audio(tmp_path / "st44.wav")
    b44, d44 = a2b(sig, sr)
    assert np.array_equal(mixed[1][0], b44) and np.array_equal(mixed[1][1], d44)
    assert np.array_equal(mixed[0][0], batch[1][0]) and np.array_equal(mixed[3][1], batch[0][1])
    with pytest.raises(Exception):
        f2b.batch([paths[0], tmp_path / "broken.wav"])
    out = tmp_path / "out" / "clip0.beats"
    File2File(small0_ckpt, "cuda:0", float16=False)(paths[0], out)
    lines = out.read_text().splitlines()
    assert len(lines) == len(batch[0][0]) and all("\t" in ln for ln in lines)
    with pytest.raises(RuntimeError):
        f2b(tmp_path / "missing.wav")


def test_cli_directory_tree(small0_ckpt, lib_built, tmp_path):
    """`python -m beat_this_b200.cli <dir> -o <out> --activations` (reference cli.py semantics on the batched engine):
    mixed sample rates / channel counts in one tree, .beats identical to File2Beats, .npy = vstack([beat, downbeat]),
    --skip-existing leaves present outputs alone."""
    from scipy.io import wavfile

    from beat_this_b200 import cli, synthetic
    from beat_this_b200.inference import File2Beats

    src = tmp_path / "in"
    (src / "sub").mkdir(parents=True)
    specs = [("a.wav", 22050, 6.0, 1), ("sub/b.wav", 44100, 7.5, 2), ("sub/c.wav", 22050, 3.2, 1)]
    for name, sr, secs, ch in specs:
        x = synthetic.synth_clip(60 + len(name), secs, sr=sr)
        data = np.round(x * 32767).astype(np.int16)
        wavfile.write(src / name, sr, data if ch == 1 else np.stack([data, data // 2], axis=1))
    out = tmp_path / "out"
    assert cli.main([str(src), "-o", str(out), "--model", small0_ckpt, "--activations", "--batch", "2"]) == 0
    f2b = File2Beats(small0_ckpt, "cuda:0", float16=False)
    for name, sr, secs, ch in specs:
        dst = (out / name).with_suffix(".beats")
        beats, downbeats = f2b(src / name)
        lines = dst.read_text().splitlines()
        assert [float(ln.split("\t")[0]) for ln in lines] == [float(f"{b}") for b in beats]
        assert sum(ln.endswith("\t1") for ln in lines) == len(downbeats)
        act = np.load(dst.with_suffix(".npy"))
        assert act.shape[0] == 2 and act.shape[1] == 1 + int(round(secs * sr)) * 22050 // sr // 441
    stamp = (out / "a.beats").stat().st_mtime_ns
    (out / "sub" / "b.beats").unlink()
    assert cli.main([str(src), "-o", str(out), "--model", small0_ckpt, "--skip-existing"]) == 0
    assert (out / "a.beats").stat().st_mtime_ns == stamp and (out / "sub" / "b.beats").exists()


@pytest.mark.parametrize("model_name", ["small0", "final0"])
def test_cli_beats_files_equal_the_reference_bytes(model_name, small0_ckpt, final0_ckpt, lib_built, tmp_path):
    """`python -m beat_this_b200.cli <tree> -o <out>` on int16 WAV files (mono, stereo, a 2-chunk file) against the
    bytes of the `.beats` files the UNMODIFIED reference writes for the same material (tests/golden/cli_beats.npz,
    oracle/make_golden_cli.py: reference Audio2Beats on samples / 32768 + reference save_beat_tsv)."""
    from scipy.io import wavfile

    from beat_this_b200 import cli, synthetic
    from oracle import beat_this_oracle as O
    from beat_this_b200.synthetic import CLI_CASES, pcm16

    g = np.load(os.path.join(GOLDEN, "cli_beats.npz"))
    ckpt = small0_ckpt if model_name == "small0" else final0_ckpt
    sd = O.strip_prefix(torch.load(ckpt, weights_only=True)["state_dict"])
    want = float(g[f"{model_name}_ckpt_sum"])
    assert abs(synthetic.tensor_checksum(sd) - want) < 1e-6 * abs(want), "checkpoint drifted from the fixture's"
    src = tmp_path / "in"
    (src / "sub").mkdir(parents=True)
    for name, seed, secs, ch in CLI_CASES:
        wavfile.write(src / name, 22050, pcm16(seed, secs, ch))
    out = tmp_path / "out"
    assert cli.main([str(src), "-o", str(out), "--model", ckpt, "--batch", "2"]) == 0
    for k, (name, seed, secs, ch) in enumerate(CLI_CASES):
        got = (out / name).with_suffix(".beats").read_bytes()
        ref = g[f"{model_name}_text{k}"].tobytes()
        assert got == ref, (model_name, name, len(got), len(ref))


def test_config4_audio2beats_dbn_on_host(small0_ckpt, lib_built):
    """BASELINE config 4 shape (Audio2Beats --dbn, DBN on the host): frames from the device, post-processing by the
    host DBN (madmom if installed, else beat_this_b200/dbn.py).  The host side must equal running the same tracker
    on the oracle-style activations of OUR logits (postprocessor.py:138-173 arithmetic)."""
    from beat_this_b200 import synthetic
    from beat_this_b200.inference import Audio2Beats, Audio2Frames

    a2b = Audio2Beats(small0_ckpt, "cuda:0", False, True)
    clips = [synthetic.synth_clip(90 + i, s) for i, s in enumerate((20.0, 8.0))]
    res = a2b.batch(clips, 22050)
    frames = Audio2Frames.batch(a2b, clips, 22050)
    for (beats, downbeats), (bl, dl) in zip(res, frames):
        eps = 1e-5
        bp = bl.double().sigmoid().cpu().numpy() * (1 - eps) + eps / 2
        dp = dl.double().sigmoid().cpu().numpy() * (1 - eps) + eps / 2
        out = a2b.frames2beats.dbn(np.vstack((np.maximum(bp - dp, eps / 2), dp)).T)
        assert np.array_equal(beats, out[:, 0]) and np.array_equal(downbeats, out[out[:, 1] == 1][:, 0])
        assert np.all(np.diff(beats) > 0) and np.all(np.isin(downbeats, beats))
    single = a2b(clips[1], 22050)
    assert np.array_equal(single[0], res[1][0]) and np.array_equal(single[1], res[1][1])
