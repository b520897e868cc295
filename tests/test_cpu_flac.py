"""CPU tests of native FLAC input: the probe, the frame tables of the host staging, refusals, the decode kernels'
machine code, and the decoder itself through its host test hook (the same frame decoder the kernels run) against the
integers the test encoder (flac_reference.py) was given."""
import ctypes
import re

import numpy as np
import pytest

import flac_reference as F
import flac_support as S
from beat_this_b200 import _lib
from support import sass

VARIANTS = S.variants()
IDS = [v[0] for v in VARIANTS]


def host_decode(buf, infos, nf, ns, status, layout, mode):
    n = len(infos)
    per = [1 if mode == _lib.BT_FLAC_MONO_F32 else info.channels for info in infos]
    oo = _lib.offsets(s * p for s, p in zip(ns, per))
    out = np.full(max(oo[-1], 1), np.nan, dtype=np.float32 if mode == _lib.BT_FLAC_MONO_F32 else np.float64)
    st = np.array(status, dtype=np.int32)
    streams = _lib.flac_streams(infos, nf, ns, oo[:-1])
    code = _lib.load().bt_debug_flac_decode_host(buf.ctypes.data, buf.ctypes.data, streams, n, mode, out.ctypes.data,
                                                 st.ctypes.data)
    assert code == 0
    return out, oo, st


@pytest.mark.parametrize("name, stream, rate, bits", VARIANTS, ids=IDS)
def test_probe_stage_and_host_decode_are_exact(lib_built, tmp_path, name, stream, rate, bits):
    path = S.write(tmp_path, name, stream)
    code, info = S.probe(path)
    T, ch = stream.samples.shape
    assert code == 0
    assert (info.sample_rate, info.channels, info.bits_per_sample) == (rate, ch, bits)
    assert info.total_samples == (0 if name == "total_zero" else T)
    assert info.frames_offset == stream.frames_offset and info.frames_bytes == len(stream.data) - stream.frames_offset
    assert bytes(info.md5) == F.md5_of(stream.samples, bits)
    buf, nf, ns, status, layout = S.stage([path], [info])
    assert status == [0] and nf == [len(stream.frames)] and ns == [T]
    assert S.frame_table(buf, layout, 0, nf[0]) == stream.frames
    bo = layout[2]
    assert buf[bo[0] : bo[1]].tobytes() == stream.data[stream.frames_offset :]
    out, _, st = host_decode(buf, [info], nf, ns, status, layout, _lib.BT_FLAC_CHANNELS_F64)
    assert st.tolist() == [0]
    assert np.array_equal(out[: T * ch], S.expected_channels(stream.samples, bits))
    back = np.round(out[: T * ch] * (1 << (bits - 1))).astype(np.int64).reshape(T, ch)
    assert F.md5_of(back, bits) == bytes(info.md5) or name == "total_zero"
    out, _, st = host_decode(buf, [info], nf, ns, status, layout, _lib.BT_FLAC_MONO_F32)
    assert st.tolist() == [0]
    assert np.array_equal(out[:T].view(np.int32), S.expected_mono(stream.samples, bits).view(np.int32))


def test_several_streams_in_one_call_and_corrupt_neighbours(lib_built, tmp_path):
    streams = [F.encode(S.signal(3000 + 500 * k, 1 + k % 3, 16, k), 44100, 16, 1024) for k in range(4)]
    paths = [S.write(tmp_path, f"s{k}", s) for k, s in enumerate(streams)]
    infos = [S.probe(p)[1] for p in paths]
    buf, nf, ns, status, layout = S.stage(paths, infos)
    assert status == [0] * 4
    bo = layout[2]
    buf[bo[1] + len(streams[1].data) // 2 - streams[1].frames_offset] ^= 0x10  # one flipped bit in file 1's frames
    buf[bo[3] + streams[3].frames[1][0] + 7] ^= 0x01                          # and in frame 1 of file 3
    out, oo, st = host_decode(buf, infos, nf, ns, status, layout, _lib.BT_FLAC_MONO_F32)
    assert st.tolist() == [0, -5, 0, -5]
    for k in (0, 2):
        assert np.array_equal(out[oo[k] : oo[k + 1]], S.expected_mono(streams[k].samples, 16))
    for k in (1, 3):
        assert not out[oo[k] : oo[k + 1]].any()  # zero-filled
    st_in = np.array([0, -5, 0, 0], dtype=np.int32)  # a stream marked bad on entry is not decoded
    out, oo, st = host_decode(buf, infos, nf, ns, st_in.tolist(), layout, _lib.BT_FLAC_MONO_F32)
    assert st.tolist()[:3] == [0, -5, 0] and not out[oo[1] : oo[2]].any()


def test_malformed_frames_end_as_statuses(lib_built, tmp_path):
    """Reserved codings, CRC mismatches and frames cut short by their table entry: BT_ERR_IO, never a read past the
    frame."""
    base = F.encode(S.signal(4096, 1, 16, 3), 44100, 16, 4096,
                    F.FrameStyle(subframes=F.Subframe(kind="lpc", order=4, porder=2)))
    path = S.write(tmp_path, "base", base)
    _, info = S.probe(path)
    buf, nf, ns, status, layout = S.stage([path], [info])
    bo = layout[2][0]
    off, _, nbytes, _ = base.frames[0]
    hl = len(F.frame_header(0, 4096, 44100, 1, 16, F.FrameStyle(), False))
    def run(b, table_bytes=None):
        b = b.copy()
        if table_bytes is not None:  # a frame table entry that claims fewer bytes: reads stop at its end
            t = (_lib.bt_flac_frame * 1).from_buffer(b)
            t[0].bytes = table_bytes
        return host_decode(b, [info], nf, ns, status, layout, _lib.BT_FLAC_MONO_F32)[2].tolist()

    def fix_crc(b):
        body = b[bo + off : bo + off + nbytes - 2].tobytes()
        crc = F.crc16_many([body])[0]
        b[bo + off + nbytes - 2], b[bo + off + nbytes - 1] = crc >> 8, crc & 0xFF

    # a reserved subframe type with a valid CRC
    b = buf.copy()
    b[bo + off + hl] = 0x02 << 1
    fix_crc(b)
    assert run(b) == [-5]
    # a reserved residual coding method (2) with a valid CRC: the LPC residual header follows 4 warm-up samples, the
    # precision, shift and 4 coefficients; flip the method's top bit wherever it lies
    bitpos = hl * 8 + 8 + 4 * 16 + 4 + 5 + 4 * 12
    b = buf.copy()
    b[bo + off + bitpos // 8] |= 0x80 >> (bitpos % 8)
    fix_crc(b)
    assert run(b) == [-5]
    # CRC mismatch
    b = buf.copy()
    b[bo + off + nbytes - 1] ^= 0xFF
    assert run(b) == [-5]
    # the table claims fewer bytes than the frame has: the CRC and reads stop at the claimed end
    for cut in (1, 8, nbytes // 2, nbytes - 1):
        assert run(buf, table_bytes=cut) == [-5]
    assert run(buf) == [0]


def test_refused_arguments(lib_built):
    lib = _lib.load()
    s = (_lib.bt_flac_stream * 1)(_lib.bt_flac_stream(0, 0, 0, 0, 10, 0, 2, 16))
    buf = np.zeros(64, dtype=np.uint8)
    out = np.zeros(64, dtype=np.float64)
    st = np.zeros(1, dtype=np.int32)
    p = buf.ctypes.data
    assert lib.bt_debug_flac_decode_host(p, p, s, 1, 2, out.ctypes.data, st.ctypes.data) == -1  # unknown mode
    for field, bad in (("channels", 0), ("channels", 9), ("bits_per_sample", 3), ("bits_per_sample", 33),
                       ("n_samples", -1), ("byte_offset", -1)):
        t = (_lib.bt_flac_stream * 1)(_lib.bt_flac_stream(0, 0, 0, 0, 10, 0, 2, 16))
        setattr(t[0], field, bad)
        assert lib.bt_debug_flac_decode_host(p, p, t, 1, 0, out.ctypes.data, st.ctypes.data) == -1, field
    assert lib.bt_debug_flac_decode_host(None, p, s, 1, 0, out.ctypes.data, st.ctypes.data) == -1
    assert lib.bt_debug_flac_decode_host(p, p, s, -1, 0, out.ctypes.data, st.ctypes.data) == -1
    assert lib.bt_flac_decode(None, p, p, s, 1, 0, out.ctypes.data, st.ctypes.data, None) == -1


def test_probe_refuses_what_is_not_flac(lib_built, tmp_path):
    good = F.encode(S.signal(2000, 1, 16, 1), 44100, 16, 1024)
    cases = {
        "notflac.bin": b"RIFF" + bytes(60),
        "empty.flac": b"",
        "marker_only.flac": b"fLaC",
        "no_streaminfo.flac": b"fLaC" + F.metadata_block(1, bytes(10), True) + good.data[good.frames_offset :],
        "short_streaminfo.flac": b"fLaC" + F.metadata_block(0, bytes(20), True),
        "metadata_past_end.flac": F.encode(S.signal(2000, 1, 16, 1), 44100, 16, 1024, extra_metadata=True).data[:60],
        "bad_marker.flac": b"fLaX" + good.data[4:],
        "bits3.flac": None,
    }
    # 3 bits per sample in STREAMINFO: the 5-bit field (bits - 1) sits in bytes 12..13 of the block body
    si_at = 4 + 4
    b = bytearray(good.data)
    b[si_at + 12] = (b[si_at + 12] & 0xFE) | 0
    b[si_at + 13] = (b[si_at + 13] & 0x0F) | (2 << 4)
    cases["bits3.flac"] = bytes(b)
    for name, data in cases.items():
        (tmp_path / name).write_bytes(data)
        code, info = S.probe(tmp_path / name)
        assert code == -6, name
        assert info.frames_bytes == 0
    assert S.probe(tmp_path / "missing.flac")[0] == -5
    (tmp_path / "good.flac").write_bytes(good.data)
    assert S.probe(tmp_path / "good.flac")[0] == 0
    wav = tmp_path / "twin.wav"
    wav.write_bytes(F.wav_twin(good.samples, 44100, 16))
    assert S.probe(wav)[0] == -6  # a WAV file is not this container
    assert [k for k, _ in _lib.probe_audio([str(tmp_path / "good.flac"), str(wav), str(tmp_path / "notflac.bin")])] \
        == ["flac", "wav", None]


def test_staging_refuses_broken_streams(lib_built, tmp_path):
    x = S.signal(5000, 2, 16, 2)
    good = F.encode(x, 44100, 16, 1024)
    path = S.write(tmp_path, "good", good)
    _, info = S.probe(path)

    def staged(data, info=info):
        p = tmp_path / "case.flac"
        p.write_bytes(data)
        return S.stage([str(p)], [info])[3][0]

    fo = good.frames_offset
    assert staged(good.data) == 0
    assert staged(good.data[: fo + good.frames[2][0]]) == -5  # frames missing: the total disagrees
    b = bytearray(good.data)
    b[fo] = 0  # no first frame
    assert staged(bytes(b)) == -5
    b = bytearray(good.data)
    b[fo + 3] |= 1  # reserved header bit
    assert staged(bytes(b)) == -5
    small = _lib.bt_flac_info.from_buffer_copy(info)
    small.max_frames = 2  # more frames than the table holds
    assert staged(good.data, small) == -5
    other = F.encode(x, 48000, 16, 1024)  # frames of another rate than STREAMINFO's
    assert staged(good.data[:fo] + other.data[other.frames_offset :]) == -5
    assert staged(good.data[:fo] + F.encode(x, 44100, 24, 1024).data[fo:]) == -5  # other bits per sample
    # a file that vanished between probe and staging
    nf, ns, status = _lib.stage_flac_files([str(tmp_path / "gone.flac")], [info], np.zeros(info.frames_bytes * 2 + 4096, np.uint8).ctypes.data, 1)
    assert status == [-5] and nf == [0] and ns == [0]


def test_encoder_conventions():
    """The encoder's own codings, stated as RFC 9639 gives them."""
    assert F.coded_number(0) == b"\x00" and F.coded_number(0x7F) == b"\x7f"
    assert F.coded_number(0x80) == b"\xc2\x80"
    assert F.coded_number((1 << 31) - 1) == bytes([0xFD] + [0xBF] * 5)
    assert F.coded_number((1 << 36) - 1) == bytes([0xFE] + [0xBF] * 6)
    w = F.BitWriter()
    w.rice([0, -1, 1, -2, 2], 0)  # zigzag 0, 1, 2, 3, 4 in unary
    assert w.tobytes() == bytes([0b10100100, 0b01000010])
    assert F.crc8(b"123456789") == 0xF4 and F.crc16_many([b"123456789"]) == [0xFEE8]


def test_decode_kernels_have_no_local_memory(lib_built):
    found, local = set(), []
    fn = None
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
            fn = next((k for k in ("flac_frames_kernel", "flac_output_kernel") if k in fn), None)
            if fn:
                found.add(fn)
        elif fn and re.search(r"\b(STL|LDL)(\.\w+)*\b", line):
            local.append((fn, line.strip()))
    assert found == {"flac_frames_kernel", "flac_output_kernel"}, found
    assert not local, local
