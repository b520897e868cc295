"""GPU tests of native Ogg Vorbis input: bt_vorbis_decode against the float64 decoder of vorbis_reference.py in both
output modes and in one call, and every path that reads audio -- load_audio, File2Beats and its .batch /
.frames_batch, the CLI, prepare and evaluate -- on Ogg Vorbis files against the in-memory path on load_audio's array.
Corrupt files end as statuses, never as faults."""
import os
import numpy as np
import pytest
import torch

import vorbis_reference as V
import vorbis_support as S
from beat_this_b200 import _lib
from support import DEV, dev  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng(lib_built, dev):  # noqa: F811
    from beat_this_b200.engine import Engine

    return Engine.mel_only(DEV)


@pytest.fixture(scope="module")
def corpus(tmp_path_factory, lib_built):
    d = tmp_path_factory.mktemp("vorbis_gpu")
    out = []
    for name, data in S.corpus():
        p = d / f"{name}.ogg"
        p.write_bytes(data)
        out.append((str(p), data, V.decode(data)))
    return out


def _device_decode(eng, paths, mode, corrupt=None, preset_status=None):
    infos = [S.probe(p)[1] for p in paths]
    fo, status_at, bo, total = _lib.vorbis_layout(infos)
    host = np.zeros(total, dtype=np.uint8)
    npk, pb, bs, status = _lib.stage_vorbis_files(paths, infos, host.ctypes.data, 1)
    if corrupt:
        corrupt(host, fo, bo)
    if preset_status is not None:
        host[status_at:status_at + 4 * len(paths)] = np.array(preset_status, dtype=np.int32).view(np.uint8)
    per = [1 if mode == _lib.BT_VORBIS_MONO_F32 else i.channels for i in infos]
    oo = _lib.offsets(i.n_samples * p for i, p in zip(infos, per))
    buf = torch.from_numpy(host).to(DEV)
    out = torch.full((max(oo[-1], 1),), float("nan"),
                     dtype=torch.float32 if mode == _lib.BT_VORBIS_MONO_F32 else torch.float64, device=DEV)
    launches = eng.launches
    eng.vorbis_decode(buf, _lib.vorbis_streams(infos, npk, pb, bs, oo[:-1]), mode, out, status_at)
    torch.cuda.synchronize()
    n_launch = eng.launches - launches
    st = buf[status_at:status_at + 4 * len(paths)].view(torch.int32).tolist()
    o = out.cpu().numpy()
    res = [o[oo[i]:oo[i + 1]].reshape(-1, per[i]) if per[i] > 1 else o[oo[i]:oo[i + 1]] for i in range(len(paths))]
    return res, st, n_launch


def test_the_corpus_decodes_in_one_call(eng, corpus):
    paths = [p for p, _, _ in corpus]
    chans, st, n = _device_decode(eng, paths, _lib.BT_VORBIS_CHANNELS_F64)
    assert st == [0] * len(corpus) and n == 3
    for (path, _, dec), got in zip(corpus, chans):
        want = dec.pcm if dec.pcm.shape[1] > 1 else dec.pcm[:, 0]
        assert got.shape == want.shape, path
        assert np.abs(got - want).max() <= S.max_err(dec.l1), path
    mono, st, _ = _device_decode(eng, paths, _lib.BT_VORBIS_MONO_F32)
    assert st == [0] * len(corpus)
    for (path, _, dec), got in zip(corpus, mono):
        assert np.abs(got - dec.pcm.mean(axis=1)).max() <= S.max_err(dec.l1) + 2.0**-24, path


def test_launch_profile_names(eng, corpus):
    """The library's own profile names the three launches of one call, once each."""
    eng.profile_enable(True)
    eng.profile_reset()
    try:
        _device_decode(eng, [corpus[1][0], corpus[2][0]], _lib.BT_VORBIS_MONO_F32)
        res = eng.profile_results()
    finally:
        eng.profile_enable(False)
    assert {k: res[k][1] for k in ("vorbis_packets", "vorbis_blocks", "vorbis_output")} == {
        "vorbis_packets": 1, "vorbis_blocks": 1, "vorbis_output": 1}


def test_refusals_launch_nothing(eng, corpus):
    s = _lib.vorbis_streams([S.probe(corpus[0][0])[1]], [1], [1], [256], [0])
    s[0].channels = 9
    buf = torch.zeros(1024, dtype=torch.uint8, device=DEV)
    out = torch.zeros(1 << 16, dtype=torch.float32, device=DEV)
    launches = eng.launches
    with pytest.raises(RuntimeError):
        eng.vorbis_decode(buf, s, _lib.BT_VORBIS_MONO_F32, out, 0)
    out64 = torch.zeros(1 << 16, dtype=torch.float64, device=DEV)
    with pytest.raises(RuntimeError):
        eng.vorbis_decode(buf, _lib.vorbis_streams([S.probe(corpus[0][0])[1]], [1], [1], [256], [0]), 7, out64, 0)
    assert eng.launches == launches


def test_a_corrupt_file_leaves_its_neighbours_unchanged(eng, corpus):
    paths = [p for p, _, _ in corpus[:3]]
    clean, st, _ = _device_decode(eng, paths, _lib.BT_VORBIS_CHANNELS_F64)

    def corrupt(host, fo, bo):  # a mode number past the first file's modes
        host[fo[0] * _lib.VORBIS_PACKET_BYTES + 5 * _lib.VORBIS_PACKET_BYTES + 28] = 63

    got, st2, _ = _device_decode(eng, paths, _lib.BT_VORBIS_CHANNELS_F64, corrupt)
    assert st2 == [-5, 0, 0]
    assert not np.any(got[0])
    for a, b in zip(clean[1:], got[1:]):
        assert np.array_equal(a, b)
    skipped, st3, _ = _device_decode(eng, paths, _lib.BT_VORBIS_MONO_F32, preset_status=[0, -5, 0])
    assert st3 == [0, -5, 0] and not np.any(skipped[1])


def test_load_audio_equals_the_channels_decode(eng, corpus):
    from beat_this_b200.preprocessing import _decode_vorbis_native

    for path, _, dec in corpus[:3]:
        got, sr = _decode_vorbis_native(path, "float64")
        chans, _, _ = _device_decode(eng, [path], _lib.BT_VORBIS_CHANNELS_F64)
        assert sr == 44100 and np.array_equal(got, chans[0])


def _clip(tmp_path, name, seconds, seed, rate=44100):
    setup = V.standard_setup(rate=rate)
    fl = S.flags(int(seconds * rate / 1024) + 4, seed)
    p = tmp_path / name
    p.write_bytes(V.encode(S.signal(int(seconds * rate), 2, seed), V.Plan(setup, fl)))
    return str(p)


@pytest.mark.parametrize("float16", [False, True], ids=["fp32", "h16"])
def test_native_path_equals_the_in_memory_path(small0_ckpt, lib_built, dev, tmp_path, float16):  # noqa: F811
    from beat_this_b200.inference import Audio2Beats, Audio2Frames, File2Beats
    from beat_this_b200.preprocessing import load_audio

    paths = [_clip(tmp_path, "a.ogg", 4, 40), _clip(tmp_path, "b.ogg", 3, 41)]
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


def test_bad_files_in_a_group(small0_ckpt, lib_built, dev, tmp_path):  # noqa: F811
    from beat_this_b200.inference import File2Beats

    good = [_clip(tmp_path, f"g{k}.ogg", 3, 50 + k) for k in range(2)]
    data = bytearray(open(good[0], "rb").read())
    pages, pos = [], 0
    while pos < len(data):
        nseg = data[pos + 26]
        pages.append(pos)
        pos += 27 + nseg + sum(data[pos + 27:pos + 27 + nseg])
    data[pages[4] + 40] ^= 0x55  # an audio page that fails its CRC
    bad = tmp_path / "bad.ogg"
    bad.write_bytes(bytes(data))
    f2b = File2Beats(small0_ckpt, DEV, float16=False)
    ref = f2b.batch(good)
    res = f2b.batch([good[0], str(bad), good[1]], on_error="skip")
    assert res[1] is None
    assert np.array_equal(res[0][0], ref[0][0]) and np.array_equal(res[2][0], ref[1][0])
    with pytest.raises(RuntimeError, match="bad.ogg.*malformed Ogg Vorbis packets"):
        f2b.batch([good[0], str(bad)], on_error="raise")


def test_cli_prepare_and_evaluate_read_vorbis(small0_ckpt, lib_built, dev, tmp_path):  # noqa: F811
    from beat_this_b200 import cli, evaluate
    from beat_this_b200.inference import File2Beats
    from beat_this_b200.prepare import prepare
    from beat_this_b200.preprocessing import load_audio

    src = tmp_path / "in"
    src.mkdir()
    a = _clip(src, "a.ogg", 4, 60)
    out = tmp_path / "out"
    assert cli.main([str(src), "-o", str(out), "--model", small0_ckpt, "--append", "--batch", "4"]) == 0
    assert (out / "a.ogg.beats").exists()
    act = tmp_path / "act"
    assert cli.main([a, "-o", str(act / "a.beats"), "--model", small0_ckpt, "--activations"]) == 0
    f2b = File2Beats(small0_ckpt, DEV, float16=False)
    sig, sr = load_audio(a)
    assert sr == 44100 and sig.shape[1] == 2
    import wave

    with wave.open(str(src / "twin.wav"), "wb") as w:
        w.setnchannels(2)
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes(np.clip(np.round(sig * 32767), -32768, 32767).astype("<i2").tobytes())
    assert evaluate._frames_of_audio(f2b, a) == evaluate._frames_of_audio(f2b, str(src / "twin.wav"))
    d = tmp_path / "prep"
    (d / "audio").mkdir(parents=True)
    (d / "ann").mkdir()
    _clip(d / "audio", "a.ogg", 4, 61)
    (d / "ann" / "a.beats").write_text("".join(f"{0.5 * (i + 1):.3f}\t{i % 4 + 1}\n" for i in range(5)))
    r = prepare([d / "audio"], d / "ann", d / "data", "toy", pitch_shift=(-1, 1), time_stretch=(4, 4), batch=2,
                device=DEV)
    assert r["written"] == ["a"] and os.path.exists(r["bundle"])
