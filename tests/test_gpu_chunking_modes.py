"""GPU tests of split_predict_aggregate with any chunk size, border and overlap mode as one batched call
(bt_spect2frames_chunked / bt_audio2frames_chunked): bitwise against the per-chunk route, against the reference's own
logits (tests/golden/chunking_modes.npz, oracle/make_golden_chunking_modes.py), and bitwise against the plain entry
points for 1500 / 6 / keep_first."""
import ctypes
import os
import wave

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from numerics import F32_TOL, H16_TOL

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

MODES = ("keep_first", "keep_last")
# (chunk_size, border_size, overlap_mode): short chunks of many waves, a border-0 family, the widest border
SETTINGS = [(64, 6, "keep_last"), (13, 6, "keep_first"), (1000, 0, "keep_first"), (1500, 100, "keep_last")]


def sweep_lengths(c, b):
    return sorted({T for T in (1, 2 * b, c - 2 * b, c - 2 * b + 1, c, c + 1, 3 * c + 7) if T >= 1})


def n_chunks(T, c, b, mode):
    from beat_this_b200 import _lib

    ck = _lib.bt_chunking(c, b, _lib.OVERLAP_MODES[mode])
    return int(_lib.load().bt_plan_chunking(T, ctypes.byref(ck), None, None, None, None, 0))


def ragged_pieces(c, b, mode, seed, min_chunks=129):
    """Random spectrograms of the sweep lengths, repeated until one call holds more than 128 chunks (several waves)."""
    g = torch.Generator().manual_seed(seed)
    pieces, chunks = [], 0
    while chunks < min_chunks:
        for T in sweep_lengths(c, b):
            pieces.append(torch.rand(T, 128, generator=g) * 7)
            chunks += n_chunks(T, c, b, mode)
    return pieces, chunks


@pytest.mark.parametrize("float16", [False, True])
@pytest.mark.parametrize("model_name", ["small0", "final0"])
def test_batched_equals_per_chunk_route_bitwise(model_name, float16, lib_built):
    """Every chunk of every piece in one call, in waves of up to 128 chunks padded to their longest member, against
    one bt_forward_chunks call per chunk (BeatThisB200.__call__) stitched by aggregate_prediction: bit-identical, as
    each chunk's logits do not depend on the wave it rides in."""
    from conftest import ckpt_path
    from beat_this_b200.inference import Spect2Frames, split_predict_aggregate

    s2f = Spect2Frames(ckpt_path(model_name), "cuda:0", float16)
    model = s2f.model
    per_chunk = lambda x: model(x)  # noqa: E731  (not a BeatThisB200: split_predict_aggregate walks the chunks)
    for k, (c, b, mode) in enumerate(SETTINGS):
        pieces, chunks = ragged_pieces(c, b, mode, seed=10 * k + (model_name == "final0"))
        assert chunks > 128
        launches = model.engine.launches
        out = s2f.spects2frames([p.cuda() for p in pieces], c, b, mode)
        batched_launches = model.engine.launches - launches
        launches = model.engine.launches
        for i, (p, (beat, down)) in enumerate(zip(pieces, out)):
            ref = split_predict_aggregate(p.cuda(), c, b, mode, per_chunk)
            assert (ref["beat"] > -1000).all(), (c, b, mode, i)
            assert torch.equal(beat, ref["beat"]) and torch.equal(down, ref["downbeat"]), (c, b, mode, i, p.shape[0])
        print(f"{model_name} float16={float16} chunking {c}/{b}/{mode}: {len(pieces)} pieces, {chunks} chunks, "
              f"{batched_launches} launches batched, {model.engine.launches - launches} per chunk")


@pytest.mark.parametrize("float16", [False, True])
def test_reference_logits(small0_ckpt, lib_built, float16):
    """split_predict_aggregate on a BeatThisB200 against the reference's on the CPU: border 0 and keep_last with
    chunk_size 1000, on a 30 s and a 61 s clip (our log-mel of the same samples in front)."""
    from beat_this_b200 import synthetic
    from beat_this_b200.inference import Spect2Frames, split_predict_aggregate
    from oracle import beat_this_oracle as O

    g = np.load(os.path.join(GOLDEN, "chunking_modes.npz"))
    sd = O.strip_prefix(torch.load(small0_ckpt, weights_only=True)["state_dict"])
    assert abs(synthetic.tensor_checksum(sd) - float(g["small0_ckpt_sum"])) < 1e-6 * abs(float(g["small0_ckpt_sum"]))
    s2f = Spect2Frames(small0_ckpt, "cuda:0", float16)
    worst = 0.0
    for j, (seed, secs) in enumerate(g["clips"]):
        spect = s2f.model.engine.logmel([synthetic.synth_clip(int(seed), float(secs))])[0]
        for i, (c, b, m) in enumerate(g["settings"]):
            out = split_predict_aggregate(spect, int(c), int(b), MODES[int(m)], s2f.model)
            rb, rd = g[f"beat_s{i}_c{j}"], g[f"down_s{i}_c{j}"]
            assert out["beat"].shape == rb.shape
            e = max(np.abs(out["beat"].cpu().numpy() - rb).max(), np.abs(out["downbeat"].cpu().numpy() - rd).max())
            print(f"float16={float16} clip {secs:.0f} s, chunking {c}/{b}/{MODES[int(m)]}: max abs logit err {e:.3e}")
            worst = max(worst, e)
    assert worst < (H16_TOL if float16 else F32_TOL)


@pytest.mark.parametrize("float16", [False, True])
def test_default_chunking_equals_plain_entry_points(small0_ckpt, lib_built, float16):
    """{1500, 6, keep_first} through bt_spect2frames_chunked / bt_audio2frames_chunked (the Engine's route, by default
    and given explicitly) == bt_spect2frames / bt_audio2frames, bitwise, on a ragged batch of more than 128 chunks."""
    from beat_this_b200 import _lib, synthetic
    from beat_this_b200.engine import Engine
    from beat_this_b200.inference import Spect2Frames

    eng = Spect2Frames(small0_ckpt, "cuda:0", float16).model.engine
    secs = [0.5, 5.0, 29.7, 30.0, 61.3, 95.0, 1500.0]
    clips = [synthetic.synth_clip(50 + i, s).astype(np.float32) for i, s in enumerate(secs)]
    clips += [synthetic.synth_clip(57, 600.0).astype(np.float32)] * 4
    so = np.concatenate([[0], np.cumsum([len(x) for x in clips])]).tolist()
    audio = torch.from_numpy(np.concatenate(clips)).cuda()
    fo = Engine.frame_offsets(so)
    assert sum(n_chunks(fo[i + 1] - fo[i], 1500, 6, "keep_first") for i in range(len(clips))) > 128
    p = eng._dev_ptr
    b0, d0 = torch.empty(fo[-1], device="cuda:0"), torch.empty(fo[-1], device="cuda:0")
    _lib.check(eng.lib, eng.ctx, eng.lib.bt_audio2frames(eng.ctx, p(audio), _lib.i64_array(so), len(clips), p(b0), p(d0),
                                                         _lib.i64_array(fo), eng._stream()))
    b1, d1, fo1 = eng.audio2frames_cat(audio, so, (1500, 6, "keep_first"))
    bd, dd, fod = eng.audio2frames_cat(audio, so)
    assert fo == fo1 == fod and torch.equal(b0, b1) and torch.equal(d0, d1) and torch.equal(b0, bd) and torch.equal(d0, dd)
    spect, _ = eng.logmel_cat(audio, so)
    b2, d2 = torch.empty_like(b0), torch.empty_like(d0)
    _lib.check(eng.lib, eng.ctx, eng.lib.bt_spect2frames(eng.ctx, p(spect), _lib.i64_array(fo), len(clips), p(b2), p(d2),
                                                         eng._stream()))
    b3, d3 = eng.spect2frames_cat(spect, fo, (1500, 6, "keep_first"))
    assert torch.equal(b2, b3) and torch.equal(d2, d3) and torch.equal(b0, b2) and torch.equal(d0, d2)
    assert all(torch.equal(a, b) for a, b in zip((b2, d2), eng.spect2frames_cat(spect, fo)))


def _write_wav(path, pcm):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(22050)
        w.writeframes(pcm.tobytes())


def test_frames_batch_equals_spects2frames(small0_ckpt, lib_built, tmp_path):
    """File2Beats.frames_batch with a chunking (native WAV decode, audio2frames route of the pipeline) == the same
    chunking through spects2frames on the log-mel of the same samples, bitwise; the default keywords are 1500 / 6 /
    keep_first."""
    from beat_this_b200 import synthetic
    from beat_this_b200.inference import File2Beats

    f2b = File2Beats(small0_ckpt, "cuda:0", True)
    secs = [5.0, 30.0, 61.3, 12.34]
    pcms = [np.round(synthetic.synth_clip(60 + i, s) * 32767).astype(np.int16) for i, s in enumerate(secs)]
    paths = []
    for i, pcm in enumerate(pcms):
        paths.append(tmp_path / f"clip{i}.wav")
        _write_wav(paths[-1], pcm)
    spects = [f2b.signal2spect(pcm, 22050) for pcm in pcms]
    for c, b, mode in SETTINGS + [(1500, 6, "keep_first")]:
        frames = f2b.frames_batch(paths, chunk_size=c, border_size=b, overlap_mode=mode)
        want = f2b.spects2frames(spects, c, b, mode)
        for (fb, fd), (wb, wd) in zip(frames, want):
            assert torch.equal(fb, wb) and torch.equal(fd, wd), (c, b, mode)
    plain = f2b.frames_batch(paths)
    for (pb, pd), (fb, fd) in zip(plain, f2b.frames_batch(paths, 1500, 6, "keep_first")):
        assert torch.equal(pb, fb) and torch.equal(pd, fd)


BAD = [(1501, 6, "keep_first"), (0, 0, "keep_first"), (64, -1, "keep_last"), (64, 32, "keep_first"),
       (1500, 6, "keep_middle")]


def test_bad_arguments_raise_before_any_launch(small0_ckpt, lib_built, tmp_path):
    from beat_this_b200 import _lib, synthetic
    from beat_this_b200.inference import File2Beats, split_predict_aggregate

    f2b = File2Beats(small0_ckpt, "cuda:0", False)
    eng = f2b.model.engine
    spect = torch.rand(3000, 128, device="cuda:0") * 7
    path = tmp_path / "clip.wav"
    pcm = np.round(synthetic.synth_clip(70, 5.0) * 32767).astype(np.int16)
    _write_wav(path, pcm)
    f2b.frames_batch([path])  # workspace and staging ring in place
    torch.cuda.synchronize()
    n0 = eng.launches
    for c, b, mode in BAD:
        with pytest.raises(ValueError):
            split_predict_aggregate(spect, c, b, mode, f2b.model)
        with pytest.raises(ValueError):
            f2b.spects2frames([spect], c, b, mode)
        with pytest.raises(ValueError):
            f2b.frames_batch([path], c, b, mode)
        with pytest.raises(ValueError):
            eng.spect2frames_cat(spect, [0, 3000], (c, b, mode))
    with pytest.raises(ValueError):  # the beat routes keep the reference's fixed chunking
        f2b.pipeline.submit_signals([pcm], 22050, "beats", (64, 6, "keep_last"))
    # the C ABI refuses on its own, before anything is enqueued
    out = torch.empty(2, 3000, device="cuda:0")
    audio = torch.from_numpy(pcm.astype(np.float32) / 32768).cuda()
    so, fo = [0, len(pcm)], eng.frame_offsets([0, len(pcm)])
    for c, b, m in [(1501, 6, 0), (0, 0, 0), (64, -1, 1), (64, 32, 0), (1500, 6, 2)]:
        ck = _lib.bt_chunking(c, b, m)
        st = eng._stream()
        assert eng.lib.bt_spect2frames_chunked(eng.ctx, ctypes.c_void_p(spect.data_ptr()), _lib.i64_array([0, 3000]), 1,
                                               ctypes.c_void_p(out[0].data_ptr()), ctypes.c_void_p(out[1].data_ptr()),
                                               ctypes.byref(ck), st) == -1
        assert eng.lib.bt_audio2frames_chunked(eng.ctx, ctypes.c_void_p(audio.data_ptr()), _lib.i64_array(so), 1,
                                               ctypes.c_void_p(out[0].data_ptr()), ctypes.c_void_p(out[1].data_ptr()),
                                               _lib.i64_array(fo), ctypes.byref(ck), st) == -1
        assert b"chunk_size" in eng.lib.bt_last_error(eng.ctx)
    assert eng.lib.bt_spect2frames_chunked(eng.ctx, ctypes.c_void_p(spect.data_ptr()), _lib.i64_array([0, 3000]), 1,
                                           ctypes.c_void_p(out[0].data_ptr()), ctypes.c_void_p(out[1].data_ptr()), None,
                                           eng._stream()) == -1
    assert eng.launches == n0
    assert f2b.pipeline.free and not f2b.pipeline.inflight  # nothing was left in the ring
