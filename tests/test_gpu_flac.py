"""GPU tests of native FLAC input: bt_flac_decode against the test encoder's integers (flac_reference.py) in both
output modes, the mono output against bt_stage_wav_files on WAV twins of the same samples, and every path that reads
audio -- load_audio, File2Beats.batch / frames_batch, the CLI, prepare and evaluate -- on FLAC files against the same
path on their WAV twins.  Corrupt files end as statuses, never as faults."""
import ctypes

import numpy as np
import pytest
import torch

import flac_reference as F
import flac_support as S
from beat_this_b200 import _lib
from support import DEV, dev  # noqa: F401

pytestmark = pytest.mark.gpu

VARIANTS = S.variants()


@pytest.fixture(scope="module")
def eng(lib_built, dev):  # noqa: F811
    from beat_this_b200.engine import Engine

    return Engine.mel_only(DEV)


def _staged(tmp_path, streams):
    paths = [S.write(tmp_path, f"v{k}", s) for k, s in enumerate(streams)]
    infos = [S.probe(p)[1] for p in paths]
    buf, nf, ns, status, layout = S.stage(paths, infos)
    assert status == [0] * len(paths)
    return paths, infos, buf, nf, ns, layout


def _decode(eng, buf, infos, nf, ns, layout, mode, status=None):
    per = [1 if mode == _lib.BT_FLAC_MONO_F32 else i.channels for i in infos]
    oo = _lib.offsets(s * p for s, p in zip(ns, per))
    b = torch.from_numpy(buf.copy()).to(DEV)
    if status is not None:
        b[layout[1] : layout[1] + 4 * len(infos)] = torch.tensor(status, dtype=torch.int32).view(torch.uint8).to(DEV)
    out = torch.full((max(oo[-1], 1),), float("nan"), device=DEV,
                     dtype=torch.float32 if mode == _lib.BT_FLAC_MONO_F32 else torch.float64)
    eng.flac_decode(b, _lib.flac_streams(infos, nf, ns, oo[:-1]), mode, out, layout[1])
    st = b[layout[1] : layout[1] + 4 * len(infos)].view(torch.int32).tolist()
    return out.cpu().numpy(), oo, st


def test_every_variant_decodes_exactly_in_one_call(eng, tmp_path):
    streams = [v[1] for v in VARIANTS]
    _, infos, buf, nf, ns, layout = _staged(tmp_path, streams)
    launches = eng.launches
    out, oo, st = _decode(eng, buf, infos, nf, ns, layout, _lib.BT_FLAC_CHANNELS_F64)
    assert eng.launches - launches == 2  # flac_frames + flac_output
    assert st == [0] * len(streams)
    for k, (name, s, rate, bits) in enumerate(VARIANTS):
        got = out[oo[k] : oo[k + 1]]
        assert np.array_equal(got, S.expected_channels(s.samples, bits)), name
        ints = np.round(got * (1 << (bits - 1))).astype(np.int64).reshape(s.samples.shape)
        assert np.array_equal(ints, s.samples), name
        if name != "total_zero":
            assert F.md5_of(ints, bits) == bytes(infos[k].md5), name
    out, oo, st = _decode(eng, buf, infos, nf, ns, layout, _lib.BT_FLAC_MONO_F32)
    assert st == [0] * len(streams)
    for k, (name, s, rate, bits) in enumerate(VARIANTS):
        assert np.array_equal(out[oo[k] : oo[k + 1]].view(np.int32), S.expected_mono(s.samples, bits).view(np.int32)), name


def test_mono_equals_the_wav_stager_on_wav_twins(eng, tmp_path):
    picked = [v for v in VARIANTS if v[0].startswith(("lpc_bits", "channels", "mid_side", "wasted"))]
    _, infos, buf, nf, ns, layout = _staged(tmp_path, [v[1] for v in picked])
    out, oo, st = _decode(eng, buf, infos, nf, ns, layout, _lib.BT_FLAC_MONO_F32)
    assert st == [0] * len(picked)
    for k, (name, s, rate, bits) in enumerate(picked):
        p = tmp_path / f"{name}.wav"
        p.write_bytes(F.wav_twin(s.samples, rate, bits))
        w = _lib.bt_wav_info()
        assert _lib.load().bt_wav_probe(str(p).encode(), ctypes.byref(w)) == 0, name
        dst = torch.zeros(w.frames, dtype=torch.float32)
        _lib.stage_wav_files([str(p)], [w], dst, [0, w.frames], 2)
        assert np.array_equal(out[oo[k] : oo[k + 1]].view(np.int32), dst.numpy().view(np.int32)), name


def test_corrupt_files_leave_their_neighbours_alone(eng, tmp_path):
    streams = [F.encode(S.signal(6000, 2, 16, k), 44100, 16, 1024) for k in range(5)]
    _, infos, buf, nf, ns, layout = _staged(tmp_path, streams)
    bo = layout[2]
    buf[bo[1] + streams[1].frames[2][0] + 20] ^= 0x04  # one bit of file 1's third frame
    cut = S.frame_table(buf, layout, 3, nf[3])         # file 3: its last frame's table entry runs past its bytes
    t = (_lib.bt_flac_frame * 1).from_buffer(buf, _lib.FLAC_FRAME_BYTES * (layout[0][3] + nf[3] - 1))
    t[0].bytes = cut[-1][2] + 1000
    out, oo, st = _decode(eng, buf, infos, nf, ns, layout, _lib.BT_FLAC_MONO_F32, status=[0, 0, 0, 0, -5])
    assert st == [0, -5, 0, -5, -5]
    for k in (0, 2):
        assert np.array_equal(out[oo[k] : oo[k + 1]], S.expected_mono(streams[k].samples, 16))
    for k in (1, 3, 4):
        assert not out[oo[k] : oo[k + 1]].any()


def test_refusals_launch_nothing(eng, tmp_path):
    lib = _lib.load()
    s = (_lib.bt_flac_stream * 1)(_lib.bt_flac_stream(0, 10, 0, 1, 10, 0, 2, 16))
    b = torch.zeros(64, dtype=torch.uint8, device=DEV)
    o = torch.zeros(64, dtype=torch.float64, device=DEV)
    p, q = ctypes.c_void_p(b.data_ptr()), ctypes.c_void_p(o.data_ptr())
    lib.bt_profile_enable(eng.ctx, 1)
    lib.bt_profile_reset(eng.ctx)
    launches = eng.launches
    bad = []
    for field, v in (("channels", 0), ("channels", 9), ("bits_per_sample", 3), ("bits_per_sample", 33),
                     ("n_frames", -1), ("n_samples", -1), ("out_offset", -1), ("byte_offset", -1)):
        t = (_lib.bt_flac_stream * 1)(_lib.bt_flac_stream(0, 10, 0, 1, 10, 0, 2, 16))
        setattr(t[0], field, v)
        bad.append((t, 1, 0, p))
    bad += [(s, 1, 2, p), (s, -1, 0, p), (s, 65536, 0, p), (s, 1, 0, None)]
    for t, n, mode, buf in bad:
        assert lib.bt_flac_decode(eng.ctx, buf, p, t, n, mode, q, p, None) == -1
    torch.cuda.synchronize()
    lib.bt_profile_collect(eng.ctx)
    assert eng.launches == launches and lib.bt_profile_count(eng.ctx) == 0
    lib.bt_profile_enable(eng.ctx, 0)


def _clips(tmp_path, n=4, seconds=(6.0, 9.5, 4.0, 12.0)):
    """FLAC files and their WAV twins of synthetic music, stereo 16-bit at 44.1 kHz."""
    from beat_this_b200 import synthetic

    flacs, wavs = [], []
    for k in range(n):
        x = synthetic.synth_clip(200 + k, seconds[k % len(seconds)], sr=44100)
        v = np.round(np.stack([x, 0.6 * x + 0.1 * np.roll(x, 7)], axis=1) * 30000).astype(np.int64)
        s = F.encode(v, 44100, 16, 4096, F.FrameStyle(assignment="mid_side", subframes=F.Subframe(order=12, porder=6)))
        flacs.append(tmp_path / f"c{k}.flac")
        flacs[-1].write_bytes(s.data)
        wavs.append(tmp_path / f"c{k}.wav")
        wavs[-1].write_bytes(F.wav_twin(v, 44100, 16))
    return flacs, wavs


def test_load_audio_equals_the_wav_twin(lib_built, dev, tmp_path):  # noqa: F811
    from beat_this_b200.preprocessing import load_audio

    flacs, wavs = _clips(tmp_path, 2)
    for f, w in zip(flacs, wavs):
        a, sa = load_audio(f)
        b, sb = load_audio(w)
        assert sa == sb == 44100 and a.dtype == b.dtype == np.float64 and a.shape == b.shape
        assert np.array_equal(a, b)
    mono = F.encode(S.signal(5000, 1, 24, 1), 32000, 24, 1000)
    (tmp_path / "m.flac").write_bytes(mono.data)
    (tmp_path / "m.wav").write_bytes(F.wav_twin(mono.samples, 32000, 24))
    a, _ = load_audio(tmp_path / "m.flac")
    b, _ = load_audio(tmp_path / "m.wav")
    assert a.ndim == 1 and np.array_equal(a, b)
    (tmp_path / "bad.flac").write_bytes(mono.data[:-300])
    with pytest.raises(RuntimeError, match="FLAC"):
        load_audio(tmp_path / "bad.flac")


def test_file2beats_on_flac_equals_wav_twins(small0_ckpt, lib_built, dev, tmp_path):  # noqa: F811
    from beat_this_b200.inference import File2Beats

    flacs, wavs = _clips(tmp_path)
    f2b = File2Beats(small0_ckpt, DEV, float16=False)
    a = f2b.batch(flacs)
    b = f2b.batch(wavs)
    for (x, y), (u, v) in zip(a, b):
        assert np.array_equal(x, u) and np.array_equal(y, v)
    fa = f2b.frames_batch(flacs)
    fb = f2b.frames_batch(wavs)
    for (x, y), (u, v) in zip(fa, fb):
        assert torch.equal(x.view(torch.int32), u.view(torch.int32)) and torch.equal(y.view(torch.int32), v.view(torch.int32))
    one = f2b(flacs[0])
    assert np.array_equal(one[0], b[0][0]) and np.array_equal(one[1], b[0][1])
    # a mixed call keeps every file's place
    mixed = f2b.batch([flacs[0], wavs[1], flacs[2]])
    assert all(np.array_equal(m[0], r[0]) for m, r in zip(mixed, [b[0], b[1], b[2]]))
    # corrupt files in a group: their own status, neighbours unaffected
    data = bytearray(flacs[1].read_bytes())
    data[len(data) // 2] ^= 0x20
    bad = tmp_path / "bad.flac"
    bad.write_bytes(bytes(data))
    launches = f2b.model.engine.launches
    res = f2b.batch([flacs[0], bad, flacs[2]], on_error="skip")
    assert res[1] is None
    assert np.array_equal(res[0][0], b[0][0]) and np.array_equal(res[2][0], b[2][0])
    assert f2b.model.engine.launches > launches
    with pytest.raises(RuntimeError, match="bad.flac"):
        f2b.batch([flacs[0], bad], on_error="raise")


def test_one_group_makes_two_decode_launches(small0_ckpt, lib_built, dev, tmp_path):  # noqa: F811
    from beat_this_b200.inference import File2Beats

    flacs, wavs = _clips(tmp_path)
    f2b = File2Beats(small0_ckpt, DEV, float16=False)
    f2b.batch(wavs)
    lib, ctx = _lib.load(), f2b.model.engine.ctx
    lib.bt_profile_enable(ctx, 1)

    def profile(paths):
        lib.bt_profile_reset(ctx)
        f2b.batch(paths)
        torch.cuda.synchronize()
        lib.bt_profile_collect(ctx)
        name, ms, cnt = ctypes.create_string_buffer(64), ctypes.c_double(), ctypes.c_int64()
        out = {}
        for i in range(lib.bt_profile_count(ctx)):
            lib.bt_profile_get(ctx, i, name, 64, ctypes.byref(ms), ctypes.byref(cnt))
            if cnt.value:  # a kernel class keeps its name after a reset
                out[name.value.decode()] = cnt.value
        return out

    pf, pw = profile(flacs), profile(wavs)
    lib.bt_profile_enable(ctx, 0)
    assert pf.pop("flac_frames") == 1 and pf.pop("flac_output") == 1
    assert pf == pw  # the rest of the group is the WAV group's


def test_cli_on_a_mixed_tree_writes_equal_beats(small0_ckpt, lib_built, dev, tmp_path):  # noqa: F811
    from beat_this_b200 import cli

    src = tmp_path / "in"
    src.mkdir()
    _clips(src, 3)
    out = tmp_path / "out"
    assert cli.main([str(src), "-o", str(out), "--model", small0_ckpt, "--append", "--batch", "4"]) == 0
    for k in range(3):
        a = (out / f"c{k}.flac.beats").read_bytes()
        assert a and a == (out / f"c{k}.wav.beats").read_bytes()


def test_prepare_on_flac_equals_wav(lib_built, dev, tmp_path):  # noqa: F811
    from beat_this_b200.prepare import prepare

    (tmp_path / "src").mkdir()
    flacs, wavs = _clips(tmp_path / "src", 2, (4.0, 3.0))
    res = {}
    for kind, files in (("flac", flacs), ("wav", wavs)):
        d = tmp_path / kind
        (d / "audio").mkdir(parents=True)
        (d / "ann").mkdir()
        for f in files:
            (d / "audio" / f.name).write_bytes(f.read_bytes())
            (d / "ann" / f"{f.stem}.beats").write_text("".join(f"{0.5 * (i + 1):.3f}\t{i % 4 + 1}\n" for i in range(5)))
        r = prepare([d / "audio"], d / "ann", d / "data", "toy", pitch_shift=(-1, 1), time_stretch=(4, 4), batch=2,
                    device=DEV)
        res[kind] = (r["written"], np.load(r["bundle"]))
    assert res["flac"][0] == res["wav"][0] == ["c0", "c1"]
    fb, wb = res["flac"][1], res["wav"][1]
    assert fb.files == wb.files
    for m in fb.files:
        assert fb[m].tobytes() == wb[m].tobytes(), m


def test_evaluate_frames_of_flac_equal_wav(small0_ckpt, lib_built, dev, tmp_path):  # noqa: F811
    from beat_this_b200 import evaluate
    from beat_this_b200.inference import File2Beats

    flacs, wavs = _clips(tmp_path, 2)
    f2b = File2Beats(small0_ckpt, DEV, float16=False)
    for f, w in zip(flacs, wavs):
        assert evaluate._frames_of_audio(f2b, str(f)) == evaluate._frames_of_audio(f2b, str(w))
