"""CPU tests of the host front door and of the function-level API against fixtures written by the UNMODIFIED
reference (oracle/make_golden.py): split_piece / aggregate_prediction (tests/golden/host_api.npz), the .beats writer
(tests/golden/beats_tsv.npz), the native staging of signals and WAV files (bt_stage_audio / bt_stage_wav_files)
against the reference's numpy arithmetic (inference.py:269-276, preprocessing.py:6-24)."""
import contextlib
import ctypes
import io
import os
import wave

import numpy as np
import pytest
import torch

from conftest import GOLDEN


def test_split_piece_and_aggregate_match_reference_fixtures():
    import beat_this_b200.inference as I

    g = np.load(os.path.join(GOLDEN, "host_api.npz"))
    for k in range(int(g["n"])):
        T, cs, bs = (int(v) for v in g[f"case{k}"])
        sp = torch.tensor(g[f"spect{k}"])
        chunks, starts = I.split_piece(sp, cs, bs, True)
        assert np.array_equal(np.asarray(starts), g[f"starts{k}"]), k
        assert [len(c) for c in chunks] == g[f"lens{k}"].tolist(), k
        assert np.array_equal(torch.cat(chunks).numpy(), g[f"chunks{k}"]), k
        preds = [{"beat": c[:, 0] * (i + 1), "downbeat": c[:, 1] - i} for i, c in enumerate(chunks)]
        for mode in ("keep_first", "keep_last"):
            b, d = I.aggregate_prediction(preds, starts, T, cs, bs, mode, "cpu")
            assert np.array_equal(b.numpy(), g[f"{mode}_beat{k}"]), (k, mode)
            assert np.array_equal(d.numpy(), g[f"{mode}_down{k}"]), (k, mode)
        # the generic split_predict_aggregate (callable model) goes through the same two functions
        out = I.split_predict_aggregate(sp, cs, bs, "keep_first", lambda c: {"beat": c[..., 0], "downbeat": c[..., 1]})
        assert np.array_equal(out["beat"].numpy(), sp[:, 0].numpy()) and np.array_equal(out["downbeat"].numpy(), sp[:, 1].numpy())


def test_chunk_starts_equal_native_planner(lib_built):
    from beat_this_b200.inference import chunk_starts

    for T in [1, 2, 1487, 1488, 1489, 1500, 1501, 2976, 2977, 3000, 4465, 15001, 40000]:
        n = lib_built.bt_plan_chunks(T, None, None, 0)
        st = (ctypes.c_int64 * n)()
        ln = (ctypes.c_int64 * n)()
        lib_built.bt_plan_chunks(T, st, ln, n)
        assert list(st) == chunk_starts(T, 1500, 6).tolist(), T


def test_beats_writer_matches_reference_fixtures(tmp_path):
    from beat_this_b200.utils import infer_beat_numbers, save_beat_tsv

    g = np.load(os.path.join(GOLDEN, "beats_tsv.npz"))
    for k in range(int(g["n"])):
        beats, downs = g[f"beats{k}"], g[f"downs{k}"]
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            numbers = infer_beat_numbers(beats, downs)
        assert np.array_equal(numbers, g[f"numbers{k}"]), k
        assert bool(out.getvalue().strip()) == bool(int(g[f"warned{k}"])), k
        path = tmp_path / f"{k}.beats"
        with contextlib.redirect_stdout(io.StringIO()):
            save_beat_tsv(beats, downs, str(path))
        assert path.read_bytes() == g[f"text{k}"].tobytes(), k


def test_beats_writer_on_the_reference_cli_fixtures(tmp_path):
    """Writer half of tests/golden/cli_beats.npz (the GPU test runs the whole CLI): the reference's beats -> its bytes."""
    from beat_this_b200.utils import save_beat_tsv

    g = np.load(os.path.join(GOLDEN, "cli_beats.npz"))
    for model_name in ("small0", "final0"):
        for k in range(3):
            path = tmp_path / f"{model_name}{k}.beats"
            with contextlib.redirect_stdout(io.StringIO()):
                save_beat_tsv(g[f"{model_name}_beats{k}"], g[f"{model_name}_downbeats{k}"], str(path))
            assert path.read_bytes() == g[f"{model_name}_text{k}"].tobytes(), (model_name, k)


def _stage(arrays, threads=3):
    from beat_this_b200 import _lib

    n = sum(a.shape[0] for a in arrays)
    dst = torch.zeros(n, dtype=torch.float32)
    so = _lib.stage_audio(arrays, dst, threads)
    return dst.numpy(), so


def test_stage_audio_equals_numpy_mix(lib_built):
    """bt_stage_audio == the reference's host half of signal2spect: numpy mean(1) in the array's own dtype, then the
    fp32 cast of torch.tensor(..., dtype=float32) -- bit for bit, for every accepted layout."""
    from beat_this_b200.pipeline import as_signal_array

    rng = np.random.default_rng(5)
    sigs = [rng.standard_normal(300_001), rng.standard_normal((1000, 2)), rng.standard_normal((777, 3)),
            rng.standard_normal(513).astype(np.float32), rng.standard_normal((4000, 2)).astype(np.float32),
            (rng.standard_normal((2500, 2)) * 9000).astype(np.int16), (rng.standard_normal(100) * 9000).astype(np.int16),
            rng.standard_normal((50, 2))[:, ::-1], list(rng.standard_normal(20)), rng.standard_normal((64, 5)).astype(np.float32)]
    arrays = [as_signal_array(s) for s in sigs]
    got, so = _stage(arrays)
    for i, s in enumerate(sigs):
        a = np.asarray(s)
        if a.dtype == np.int16:
            a = a.astype(np.float64) / 32768.0
        ref = a.mean(1) if a.ndim == 2 else a
        ref = torch.tensor(ref, dtype=torch.float32).numpy()
        assert np.array_equal(got[so[i] : so[i + 1]], ref), i
    with pytest.raises(ValueError):
        as_signal_array(np.zeros((3, 2, 2)))


def _write_wav(path, data, sr, sampwidth):
    """PCM writer for the test (stdlib wave): data int array [T] or [T, ch] already scaled to the sample width."""
    data = np.asarray(data)
    ch = 1 if data.ndim == 1 else data.shape[1]
    with wave.open(str(path), "wb") as w:
        w.setnchannels(ch); w.setsampwidth(sampwidth); w.setframerate(sr)
        if sampwidth == 2:
            raw = data.astype("<i2").tobytes()
        elif sampwidth == 3:
            v = data.astype(np.int32).reshape(-1)
            raw = np.stack([v & 255, (v >> 8) & 255, (v >> 16) & 255], 1).astype(np.uint8).tobytes()
        elif sampwidth == 4:
            raw = data.astype("<i4").tobytes()
        else:
            raw = data.astype(np.uint8).tobytes()
        w.writeframes(raw)


def test_native_wav_front_door_equals_load_audio(lib_built, tmp_path):
    """bt_wav_probe + bt_stage_wav_files == load_audio (float64, [T, ch]) -> mean(1) -> float32, for PCM 8/16/24/32
    and IEEE float files, mono and multi-channel; non-WAV input is reported as BT_ERR_FORMAT."""
    from scipy.io import wavfile

    from beat_this_b200._lib import bt_wav_info
    from beat_this_b200.preprocessing import load_audio

    rng = np.random.default_rng(9)
    files = []
    x = rng.standard_normal((30000, 2))
    _write_wav(tmp_path / "s16.wav", np.clip(x * 8000, -32768, 32767), 22050, 2); files.append("s16.wav")
    _write_wav(tmp_path / "m16.wav", np.clip(x[:, 0] * 8000, -32768, 32767), 44100, 2); files.append("m16.wav")
    _write_wav(tmp_path / "s24.wav", np.clip(x[:9000] * 2_000_000, -8388608, 8388607), 48000, 3); files.append("s24.wav")
    _write_wav(tmp_path / "m32.wav", np.clip(x[:5000, 1] * 5e8, -2**31, 2**31 - 1), 22050, 4); files.append("m32.wav")
    _write_wav(tmp_path / "m8.wav", np.clip(x[:4000, 0] * 40 + 128, 0, 255), 8000, 1); files.append("m8.wav")
    wavfile.write(tmp_path / "f32.wav", 22050, (x[:7000] * 0.3).astype(np.float32)); files.append("f32.wav")
    wavfile.write(tmp_path / "f64.wav", 22050, x[:600, 0] * 0.3); files.append("f64.wav")
    paths = [str(tmp_path / f) for f in files]
    infos = (bt_wav_info * len(paths))()
    for i, p in enumerate(paths):
        assert lib_built.bt_wav_probe(p.encode(), ctypes.byref(infos[i])) == 0, p
    so = [0]
    for i in range(len(paths)):
        so.append(so[-1] + infos[i].frames)
    dst = torch.full((so[-1],), 7.0, dtype=torch.float32)
    status = (ctypes.c_int32 * len(paths))()
    code = lib_built.bt_stage_wav_files((ctypes.c_char_p * len(paths))(*[p.encode() for p in paths]), infos, len(paths),
                                        ctypes.c_void_p(dst.data_ptr()), (ctypes.c_int64 * len(so))(*so), 4, status)
    assert code == 0 and list(status) == [0] * len(paths)
    for i, p in enumerate(paths):
        wav, sr = load_audio(p)
        assert sr == infos[i].sample_rate and wav.shape[0] == infos[i].frames, p
        ref = torch.tensor(wav.mean(1) if wav.ndim == 2 else wav, dtype=torch.float32).numpy()
        assert np.array_equal(dst.numpy()[so[i] : so[i + 1]], ref), p
    (tmp_path / "notwav.bin").write_bytes(b"ID3" + bytes(100))
    info = bt_wav_info()
    assert lib_built.bt_wav_probe(str(tmp_path / "notwav.bin").encode(), ctypes.byref(info)) == -6
    assert lib_built.bt_wav_probe(str(tmp_path / "missing.wav").encode(), ctypes.byref(info)) == -5


def test_plan_groups_and_padded_frames_known_answers():
    from beat_this_b200.pipeline import plan_groups

    assert plan_groups([10] * 5, 25, 64) == [(0, 2), (2, 4), (4, 5)]
    assert plan_groups([100, 1, 1], 25, 64) == [(0, 1), (1, 3)]
    assert plan_groups([1] * 10, 1000, 4) == [(0, 4), (4, 8), (8, 10)]
    assert plan_groups([], 10, 4) == []
    from beat_this_b200.pipeline import padded_frames

    lengths = (22050 * 5, 656082, 656083 + 441, 661500, 22050 * 300)
    assert [padded_frames(n, 22050, 1500, 6) for n in lengths] == [1500 * k for k in (1, 1, 2, 2, 11)]
    assert padded_frames(44100 * 30, 44100, 1500, 6) == 2 * 1500
