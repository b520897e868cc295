"""GPU tests of native MP3 input: bt_mp3_decode against the float64 decoder of mp3_reference.py in both output modes
and in one call, and every path that reads audio -- load_audio, File2Beats and its .batch / .frames_batch, the CLI,
prepare and evaluate -- on MP3 files against the in-memory path on load_audio's array.  Corrupt files end as
statuses, never as faults."""
import ctypes
import os

import numpy as np
import pytest
import torch

import mp3_reference as M
from beat_this_b200 import _lib
from support import DEV, dev  # noqa: F401
import mp3_support as S
from mp3_support import FIXTURE, assert_close, probe, write

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng(lib_built, dev):  # noqa: F811
    from beat_this_b200.engine import Engine

    return Engine.mel_only(DEV)


@pytest.fixture(scope="module")
def fixture_bytes():
    return open(FIXTURE, "rb").read()


def _variants(tmp_path, fixture_bytes):
    """(path, float64 decode) of the fixture and of streams covering stereo coding, tags and a gapless trim."""
    frames = M.split_frames(fixture_bytes)
    out = [(FIXTURE, M.decode(fixture_bytes).pcm)]
    for ext in (1, 2, 3):
        data = b"".join(M.with_header(f, mode_ext=ext) for f in frames[50:110])
        out.append((write(tmp_path, f"ext{ext}.mp3", M.id3v2(300) + data + M.id3v1()), M.decode(data).pcm))
    body = b"".join(frames[:40])
    full = M.decode(body).pcm
    out.append((write(tmp_path, "gapless.mp3", M.xing_frame(frames[0], 40, 576, 1000) + body),
                full[576 + 529 : 1152 * 40 - 1000 + 529]))
    for name, data in S.variants():  # mono, CRC, 32 / 48 kHz, mixed blocks, gains, scfsi, reservoir, VBR, tables
        pcm = M.decode(data).pcm
        out.append((write(tmp_path, f"{name}.mp3", data), pcm if pcm.shape[1] > 1 else pcm[:, 0]))
    return out


def _device_decode(eng, paths, mode, corrupt=None, preset_status=None):
    infos = [probe(p)[1] for p in paths]
    fo, status_at, bo, total = _lib.mp3_layout(infos)
    host = np.zeros(total, dtype=np.uint8)
    nf, mb, status = _lib.stage_mp3_files(paths, infos, host.ctypes.data, 1)
    if corrupt:
        corrupt(host, fo, bo)
    if preset_status is not None:
        np.frombuffer(host, dtype=np.uint8)[status_at : status_at + 4 * len(paths)] = np.array(
            preset_status, dtype=np.int32).view(np.uint8)
    per = [1 if mode == _lib.BT_MP3_MONO_F32 else i.channels for i in infos]
    oo = _lib.offsets(i.n_samples * p for i, p in zip(infos, per))
    buf = torch.from_numpy(host).to(DEV)
    out = torch.full((max(oo[-1], 1),), float("nan"), dtype=torch.float32 if mode == _lib.BT_MP3_MONO_F32 else torch.float64,
                     device=DEV)
    launches = eng.launches
    eng.mp3_decode(buf, _lib.mp3_streams(infos, nf, mb, oo[:-1]), mode, out, status_at)
    torch.cuda.synchronize()
    n_launch = eng.launches - launches
    st = buf[status_at : status_at + 4 * len(paths)].view(torch.int32).tolist()
    o = out.cpu().numpy()
    res = [o[oo[i] : oo[i + 1]].reshape(-1, per[i]) if per[i] > 1 else o[oo[i] : oo[i + 1]] for i in range(len(paths))]
    return res, st, n_launch


def test_every_variant_decodes_in_one_call(eng, tmp_path, fixture_bytes):
    vs = _variants(tmp_path, fixture_bytes)
    chans, st, n = _device_decode(eng, [p for p, _ in vs], _lib.BT_MP3_CHANNELS_F64)
    assert st == [0] * len(vs) and n == 3
    for (_, want), got in zip(vs, chans):
        assert got.shape == want.shape
        assert_close(got, want)
    mono, st, n = _device_decode(eng, [p for p, _ in vs], _lib.BT_MP3_MONO_F32)
    assert st == [0] * len(vs) and n == 3
    for c, m in zip(chans, mono):
        want = ((c[:, 0] + c[:, 1]) / 2).astype(np.float32) if c.ndim == 2 else c.astype(np.float32)
        assert np.array_equal(m.view(np.int32), want.view(np.int32))


def test_streams_that_are_not_decoded_are_zero_filled(eng, tmp_path, fixture_bytes):
    """A file whose staging failed (no frames at all) and a file marked bad on entry: zeros over their whole output
    in a NaN-filled buffer, in both modes; the good file beside them is unchanged."""
    frames = M.split_frames(fixture_bytes)
    good = write(tmp_path, "good.mp3", b"".join(frames[:20]))
    lost = write(tmp_path, "lost.mp3", b"".join(frames[:10]) + bytes(100) + b"".join(frames[10:20]))
    for mode in (_lib.BT_MP3_CHANNELS_F64, _lib.BT_MP3_MONO_F32):
        ref, st, _ = _device_decode(eng, [good], mode)
        got, st, n = _device_decode(eng, [good, lost, good], mode, preset_status=[0, -5, -5])
        assert st == [0, -5, -5]
        assert np.array_equal(got[0], ref[0])
        assert np.array_equal(got[1], np.zeros_like(got[1])) and np.array_equal(got[2], np.zeros_like(got[2]))
        only, st, n = _device_decode(eng, [lost], mode)  # no stream has a frame: the output is still written
        assert st == [-5] and n == 1 and np.array_equal(only[0], np.zeros_like(only[0]))


def test_corrupt_files_leave_their_neighbours_alone(eng, tmp_path, fixture_bytes):
    frames = M.split_frames(fixture_bytes)
    paths = [write(tmp_path, f"n{k}.mp3", b"".join(frames[30 * k : 30 * k + 30])) for k in range(4)]
    good, st, _ = _device_decode(eng, paths, _lib.BT_MP3_CHANNELS_F64)
    assert st == [0] * 4

    def corrupt(host, fo, bo):
        t = (_lib.bt_mp3_frame * 30).from_buffer(host, _lib.MP3_FRAME_BYTES * fo[1])
        t[5].main_start = 10**6  # outside the stream's main data
        t = (_lib.bt_mp3_frame * 30).from_buffer(host, _lib.MP3_FRAME_BYTES * fo[2])
        t[7].side_info[2] |= 0x7F  # part2_3_length of granule 0 past its data and big_values over 288 in the next

    got, st, _ = _device_decode(eng, paths, _lib.BT_MP3_CHANNELS_F64, corrupt)
    assert st[0] == st[3] == 0 and st[1] == -5
    assert not np.any(got[1]) and (st[2] == 0 or not np.any(got[2]))
    assert np.array_equal(got[0], good[0]) and np.array_equal(got[3], good[3])


def test_refusals_launch_nothing(eng):
    lib = _lib.load()
    b = torch.zeros(64, dtype=torch.uint8, device=DEV)
    o = torch.zeros(64, dtype=torch.float64, device=DEV)
    p, q = ctypes.c_void_p(b.data_ptr()), ctypes.c_void_p(o.data_ptr())

    def table(**kw):
        t = (_lib.bt_mp3_stream * 1)(_lib.bt_mp3_stream(0, 10, 0, 1, 0, 10, 0, 2, 44100))
        for k, v in kw.items():
            setattr(t[0], k, v)
        return t

    launches = eng.launches
    bad = [(table(**{f: v}), 1, 0, p) for f, v in (("channels", 0), ("channels", 3), ("sample_rate", 22050),
                                                   ("n_frames", -1), ("n_samples", -1), ("skip", -1),
                                                   ("out_offset", -1), ("byte_offset", -1))]
    bad += [(table(), 1, 2, p), (table(), -1, 0, p), (table(), 65536, 0, p), (table(), 1, 0, None)]
    for t, n, mode, buf in bad:
        assert lib.bt_mp3_decode(eng.ctx, buf, p, t, n, mode, q, p, None) == -1
    torch.cuda.synchronize()
    assert eng.launches == launches


def test_load_audio_equals_the_channels_decode(eng, lib_built):
    from beat_this_b200.preprocessing import load_audio

    a, sr = load_audio(FIXTURE)
    (want,), st, _ = _device_decode(eng, [FIXTURE], _lib.BT_MP3_CHANNELS_F64)
    assert sr == 44100 and st == [0] and a.dtype == np.float64 and np.array_equal(a, want)


def test_the_references_own_test(small0_ckpt, lib_built, dev):  # noqa: F811
    """The reference's test_File2Beat on (the first ten seconds of) its own recording."""
    from beat_this_b200.inference import File2Beats

    beat, downbeat = File2Beats(small0_ckpt, DEV)(FIXTURE)
    assert isinstance(beat, np.ndarray) and isinstance(downbeat, np.ndarray)


@pytest.mark.parametrize("float16", [False, True], ids=["fp32", "h16"])
def test_native_path_equals_the_in_memory_path(small0_ckpt, lib_built, dev, tmp_path, fixture_bytes, float16):  # noqa: F811
    from beat_this_b200.inference import Audio2Beats, Audio2Frames, File2Beats
    from beat_this_b200.preprocessing import load_audio

    frames = M.split_frames(fixture_bytes)
    paths = [FIXTURE, write(tmp_path, "b.mp3", b"".join(M.with_header(f, mode_ext=2) for f in frames[:200]))]
    f2b = File2Beats(small0_ckpt, DEV, float16=float16)
    sigs = [load_audio(p)[0] for p in paths]
    got = f2b.batch(paths)
    want = Audio2Beats.batch(f2b, sigs, 44100)
    for (x, y), (u, v) in zip(got, want):
        assert np.array_equal(x, u) and np.array_equal(y, v)
    fa = f2b.frames_batch(paths)
    fb = Audio2Frames.batch(f2b, sigs, 44100)
    for (x, y), (u, v) in zip(fa, fb):
        assert torch.equal(x.view(torch.int32), u.view(torch.int32)) and torch.equal(y.view(torch.int32), v.view(torch.int32))


def test_bad_files_in_a_group(small0_ckpt, lib_built, dev, tmp_path, fixture_bytes):  # noqa: F811
    from beat_this_b200.inference import File2Beats

    frames = M.split_frames(fixture_bytes)
    good = [write(tmp_path, f"g{k}.mp3", b"".join(frames[100 * k : 100 * k + 100])) for k in range(2)]
    lost = write(tmp_path, "lost.mp3", b"".join(frames[:10]) + bytes(100) + b"".join(frames[10:100]))
    f2b = File2Beats(small0_ckpt, DEV, float16=False)
    ref = f2b.batch(good)
    res = f2b.batch([good[0], lost, good[1]], on_error="skip")
    assert res[1] is None
    assert np.array_equal(res[0][0], ref[0][0]) and np.array_equal(res[2][0], ref[1][0])
    with pytest.raises(RuntimeError, match="lost.mp3.*malformed MP3 frames"):
        f2b.batch([good[0], lost], on_error="raise")


def test_cli_prepare_and_evaluate_read_mp3(small0_ckpt, lib_built, dev, tmp_path, fixture_bytes):  # noqa: F811
    import flac_reference as F
    import flac_support as FS
    from beat_this_b200 import cli, evaluate
    from beat_this_b200.inference import File2Beats
    from beat_this_b200.prepare import prepare

    frames = M.split_frames(fixture_bytes)
    src = tmp_path / "in"
    src.mkdir()
    write(src, "a.mp3", b"".join(frames[:200]))
    v = FS.signal(44100 * 5, 2, 16, 3)
    write(src, "b.flac", F.encode(v, 44100, 16, 4096).data)
    write(src, "c.wav", F.wav_twin(v, 44100, 16))
    out = tmp_path / "out"
    assert cli.main([str(src), "-o", str(out), "--model", small0_ckpt, "--append", "--batch", "4"]) == 0
    for name in ("a.mp3", "b.flac", "c.wav"):
        assert (out / f"{name}.beats").exists(), name
    f2b = File2Beats(small0_ckpt, DEV, float16=False)
    from beat_this_b200.preprocessing import load_audio

    sig, sr = load_audio(src / "a.mp3")
    assert len(sig) == 200 * 1152 and sr == 44100
    # the frame count evaluate takes for the MP3 equals the one of a WAV file holding load_audio's samples
    import wave

    with wave.open(str(src / "twin.wav"), "wb") as w:
        w.setnchannels(2)
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes(np.clip(np.round(sig * 32767), -32768, 32767).astype("<i2").tobytes())
    assert evaluate._frames_of_audio(f2b, str(src / "a.mp3")) == evaluate._frames_of_audio(f2b, str(src / "twin.wav"))
    d = tmp_path / "prep"
    (d / "audio").mkdir(parents=True)
    (d / "ann").mkdir()
    write(d / "audio", "a.mp3", b"".join(frames[:150]))
    (d / "ann" / "a.beats").write_text("".join(f"{0.5 * (i + 1):.3f}\t{i % 4 + 1}\n" for i in range(5)))
    r = prepare([d / "audio"], d / "ann", d / "data", "toy", pitch_shift=(-1, 1), time_stretch=(4, 4), batch=2,
                device=DEV)
    assert r["written"] == ["a"] and os.path.exists(r["bundle"])
