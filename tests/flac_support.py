"""The FLAC tests' streams (tests/flac_reference.py) and the calls that stage and decode them."""
import ctypes

import numpy as np

import flac_reference as F
from beat_this_b200 import _lib


def signal(T: int, ch: int, bits: int, seed: int) -> np.ndarray:
    """Integers of `bits` bits [T, ch] that LPC predicts well but not exactly: a few tones plus noise, channels
    correlated, full scale reached."""
    rng = np.random.default_rng(seed)
    t = np.arange(T)[:, None]
    f = rng.uniform(0.001, 0.05, size=(3, 1))
    base = sum(np.sin(2 * np.pi * f[k] * t + k) for k in range(3)) / 3
    x = 0.8 * base + 0.1 * rng.standard_normal((T, ch)) + 0.05 * rng.standard_normal((T, 1))
    top = (1 << (bits - 1)) - 1
    v = np.clip(np.round(x * top), -top - 1, top).astype(np.int64)
    v[0, 0], v[1 % T, 0] = top, -top - 1
    return v


def variants():
    """(name, Stream, sample rate, bits) covering every feature the decoder takes."""
    out = []
    for bits in (4, 8, 12, 16, 20, 24, 32):
        method = 1 if bits > 16 else 0
        st = F.FrameStyle(subframes=F.Subframe(kind="lpc", order=8, precision=15 if bits > 8 else 8, method=method,
                                               porder=3))
        out.append((f"lpc_bits{bits}", F.encode(signal(5000, 2, bits, bits), 44100, bits, 1024, st), 44100, bits))
    for ch in range(1, 9):
        out.append((f"channels{ch}", F.encode(signal(3000, ch, 16, 10 + ch), 48000, 16, 1152), 48000, 16))
    for a in ("left_side", "side_right", "mid_side"):
        for bits in (16, 32):
            st = F.FrameStyle(assignment=a, subframes=F.Subframe(kind="fixed", order=2, method=1))
            out.append((f"{a}_{bits}", F.encode(signal(4500, 2, bits, 7), 44100, bits, 1024, st), 44100, bits))
    for order in range(5):
        st = F.FrameStyle(subframes=F.Subframe(kind="fixed", order=order, porder=2))
        out.append((f"fixed{order}", F.encode(signal(3000, 1, 16, order), 22050, 16, 576, st), 22050, 16))
    for order in (1, 2, 7, 12, 31, 32):
        for precision in (4, 15):
            st = F.FrameStyle(subframes=F.Subframe(kind="lpc", order=order, precision=precision, porder=0))
            out.append((f"lpc{order}_p{precision}", F.encode(signal(2500, 1, 16, order), 16000, 16, 1000, st), 16000, 16))
    const = np.repeat(np.array([[5, -3]]), 2000, axis=0)
    out.append(("constant", F.encode(const, 44100, 16, 512, F.FrameStyle(subframes=F.Subframe(kind="constant"))), 44100, 16))
    out.append(("verbatim", F.encode(signal(2000, 2, 24, 3), 44100, 24, 512,
                                     F.FrameStyle(subframes=F.Subframe(kind="verbatim"))), 44100, 24))
    wasted = signal(3000, 2, 16, 4) & ~np.int64(7)
    wasted[:, 1] &= ~np.int64(0xFF)
    out.append(("wasted", F.encode(wasted, 44100, 16, 1024), 44100, 16))
    out.append(("wasted_mid_side", F.encode(wasted, 44100, 16, 1024, F.FrameStyle(assignment="mid_side")), 44100, 16))
    for method in (0, 1):
        for porder in range(9):
            st = F.FrameStyle(subframes=F.Subframe(kind="lpc", order=4, method=method, porder=porder, escape=True))
            out.append((f"rice{method}_porder{porder}", F.encode(signal(4096, 1, 16, porder), 44100, 16, 4096, st),
                        44100, 16))
    zeros = signal(4096, 1, 16, 1)
    zeros[1024:2048] = 0  # partition 1 of order 2 escapes at width 0
    out.append(("escape_width0", F.encode(zeros, 44100, 16, 4096, F.FrameStyle(subframes=F.Subframe(
        kind="fixed", order=0, porder=2, escape=True, wasted=False))), 44100, 16))
    out.append(("odd_8bit", F.encode(signal(1000, 1, 16, 5), 44100, 16, 100, F.FrameStyle(bs_code="8bit")), 44100, 16))
    out.append(("odd_16bit", F.encode(signal(5000, 1, 16, 6), 44100, 16, 1001), 44100, 16))
    out.append(("short_last", F.encode(signal(4097, 2, 16, 8), 44100, 16, 4096), 44100, 16))
    sizes = [300, 4096, 17, 1000, 2000, 192, 4608]
    out.append(("variable", F.encode(signal(sum(sizes), 2, 16, 9), 44100, 16, sizes, variable=True), 44100, 16))
    # sample numbers past the 1-byte form: sizes adding up beyond 2^7, 2^11 and 2^16
    sizes = [100] * 3 + [4096] * 20
    out.append(("variable_long", F.encode(signal(sum(sizes), 1, 8, 10), 8000, 8, sizes, variable=True), 8000, 8))
    for rate, how in ((44100, "streaminfo"), (44100, "auto"), (88200, "auto"), (176400, "auto"), (192000, "auto"),
                      (8000, "auto"), (16000, "auto"), (22050, "auto"), (24000, "auto"), (32000, "auto"),
                      (48000, "auto"), (96000, "auto"), (11000, "khz"), (11025, "hz"), (100000, "tens")):
        st = F.FrameStyle(rate_code=how, bits_code="streaminfo" if rate == 11025 else "auto")
        out.append((f"rate{rate}_{how}", F.encode(signal(1500, 1, 16, rate % 97), rate, 16, 512, st), rate, 16))
    out.append(("total_zero", F.encode(signal(3000, 2, 16, 11), 44100, 16, 1024, total_zero=True), 44100, 16))
    out.append(("metadata_id3", F.encode(signal(3000, 2, 16, 12), 44100, 16, 1024, extra_metadata=True, id3=True),
                44100, 16))
    fs = signal(4096 * 6, 1, 16, 13)
    for k in range(1, 6, 2):
        fs[4096 * k : 4096 * (k + 1), 0] = F.false_sync_samples(4096, 1, 16, 44100)
    out.append(("false_syncs", F.encode(fs, 44100, 16, 4096, false_syncs=True), 44100, 16))
    return out


def write(tmp_path, name: str, stream) -> str:
    p = tmp_path / f"{name}.flac"
    p.write_bytes(stream.data)
    return str(p)


def probe(path):
    info = _lib.bt_flac_info()
    code = _lib.load().bt_flac_probe(str(path).encode(), ctypes.byref(info))
    return code, info


def stage(paths, infos):
    """stage_flac_files into a numpy byte buffer: (buffer, n_frames, n_samples, status, layout)."""
    layout = _lib.flac_layout(infos)
    buf = np.zeros(max(layout[3], 1), dtype=np.uint8)
    nf, ns, status = _lib.stage_flac_files(paths, infos, buf.ctypes.data, 4)
    return buf, nf, ns, status, layout


def frame_table(buf, layout, i, n):
    fo = layout[0]
    raw = buf[_lib.FLAC_FRAME_BYTES * fo[i] : _lib.FLAC_FRAME_BYTES * (fo[i] + n)]
    t = (_lib.bt_flac_frame * n).from_buffer_copy(raw.tobytes())
    return [(f.offset, f.first_sample, f.bytes, f.block_size) for f in t]


def expected_mono(x, bits: int) -> np.ndarray:
    """bt_stage_wav_files's arithmetic on the integers: float64 v / 2^(bits-1), channel sum in order, one division,
    fp32."""
    v = x.astype(np.float64) * (1.0 / (1 << (bits - 1)))
    if v.shape[1] == 1:
        return v[:, 0].astype(np.float32)
    acc = v[:, 0].copy()
    for c in range(1, v.shape[1]):
        acc += v[:, c]
    return (acc / v.shape[1]).astype(np.float32)


def expected_channels(x, bits: int) -> np.ndarray:
    return (x.astype(np.float64) * (1.0 / (1 << (bits - 1)))).reshape(-1)
