"""The MP3 tests' fixture, error bounds and the calls that probe and stage files (tests/test_cpu_mp3.py,
tests/test_gpu_mp3.py)."""
import ctypes
import os

import numpy as np

import mp3_reference as M
from beat_this_b200 import _lib

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = os.path.join(GOLD, M.FIXTURE)
N_FIXTURE = 383

# ISO/IEC 11172-4 "full accuracy": RMS of the difference below 2^-15 / sqrt(12), maximum at most 2^-14 of full scale.
# The fp32 chain of the decoder (requantisation, 18-term IMDCT sums, 32-term matrixing, 16-tap window sums, each with
# a relative rounding of 2^-24 per operation on values of at most a few units) stays orders of magnitude inside it:
# at most about 40 roundings of 2^-24 on sums of magnitude below 8 give 40 * 8 * 2^-24 < 2^-15, so the bound held here
# is that tighter one, with the ISO limits as a ceiling.
MAX_ERR = 40 * 8 * 2.0**-24
RMS_ERR = 2.0**-15 / np.sqrt(12)
assert MAX_ERR <= 2.0**-14


def probe(path):
    info = _lib.bt_mp3_info()
    code = _lib.load().bt_mp3_probe(str(path).encode(), ctypes.byref(info))
    return code, info


def stage(paths, infos):
    fo, status_at, bo, total = _lib.mp3_layout(infos)
    buf = np.zeros(max(total, 1), dtype=np.uint8)
    nf, mb, status = _lib.stage_mp3_files(paths, infos, buf.ctypes.data, 1)
    return buf, nf, mb, status


def host_decode(paths, mode=_lib.BT_MP3_CHANNELS_F64, corrupt=None, preset_status=None):
    """Probe, stage and decode files through bt_debug_mp3_decode_host into a NaN-filled output: (outputs per file,
    statuses, infos).  corrupt(buf, infos, n_frames, main_bytes) may change the staged data; preset_status replaces
    the staging's statuses (a file marked bad on entry is not decoded)."""
    infos = [probe(p)[1] for p in paths]
    buf, nf, mb, status = stage(paths, infos)
    if corrupt is not None:
        corrupt(buf, infos, nf, mb)
    per = [1 if mode == _lib.BT_MP3_MONO_F32 else i.channels for i in infos]
    oo = _lib.offsets(i.n_samples * p for i, p in zip(infos, per))
    out = np.full(max(oo[-1], 1), np.nan, dtype=np.float32 if mode == _lib.BT_MP3_MONO_F32 else np.float64)
    st = np.array(status if preset_status is None else preset_status, dtype=np.int32)
    streams = _lib.mp3_streams(infos, nf, mb, oo[:-1])
    assert _lib.load().bt_debug_mp3_decode_host(buf.ctypes.data, buf.ctypes.data, streams, len(paths), mode,
                                                out.ctypes.data, st.ctypes.data) == 0
    res = [out[oo[i] : oo[i + 1]].reshape(-1, per[i]) if per[i] > 1 else out[oo[i] : oo[i + 1]] for i in range(len(paths))]
    return res, st.tolist(), infos


def assert_close(got, want):
    d = np.asarray(got, dtype=np.float64) - want
    assert np.all(np.isfinite(got))
    assert np.abs(d).max() <= MAX_ERR and np.sqrt(np.mean(d**2)) < RMS_ERR


def write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return p


def signal(n: int, ch: int, seed: int, level: float = 0.3) -> np.ndarray:
    """Tones, a chirp and noise [n] or [n, ch] in [-1, 1], the channels correlated but not equal."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 44100
    base = np.sin(2 * np.pi * 440 * t) + 0.6 * np.sin(2 * np.pi * (2000 + 3000 * t) * t) + 0.3 * rng.standard_normal(n)
    if ch == 1:
        return level * base / 2
    other = np.sin(2 * np.pi * 660 * t + 1) + 0.3 * rng.standard_normal(n)
    return level * np.stack([base, 0.6 * base + 0.4 * other], axis=1) / 2


G = M.GranuleSpec
SWITCH = [G(), G(block_type=1), G(block_type=2), G(block_type=2), G(block_type=3), G()]


def variants():
    """(name, stream bytes) of synthetic streams, each covering features the fixture does not have."""
    out = []

    def add(name, sig, rate, grans, **kw):
        out.append((name, M.encode(sig, rate, grans, **kw)[0]))

    add("mono_long", signal(1152 * 12, 1, 1), 44100, [G()])
    add("mono_switch_crc", signal(1152 * 12, 1, 2), 44100, SWITCH, crc=True)
    for rate in (32000, 48000):
        add(f"rate{rate}_switch", signal(1152 * 12, 2, 3), rate, SWITCH, ms=True)
        add(f"rate{rate}_mixed", signal(1152 * 8, 2, 4), rate, [G(block_type=2, mixed=1, scalefactors="random",
                                                                       subblock_gain=(1, 0, 2))])
    add("mixed_gains", signal(1152 * 10, 2, 5), 44100,
        [G(block_type=2, mixed=1, scalefactors="random", subblock_gain=(2, 1, 0), scalefac_scale=1)])
    add("short_gains", signal(1152 * 10, 2, 6), 44100,
        [G(block_type=2, scalefactors="random", subblock_gain=(0, 3, 1))])
    add("long_preflag", signal(1152 * 10, 2, 7), 44100, [G(scalefactors="random", preflag=1, scalefac_scale=1)])
    add("scfsi", signal(1152 * 10, 2, 8), 44100, [G(scalefactors="random")], scfsi=(1, 0, 1, 1))
    add("mid_side", signal(1152 * 10, 2, 9), 44100, SWITCH, ms=True)
    # the bit reservoir: a quiet signal leaves free bytes, so main data begins as far back as allowed (511 bytes)
    add("reservoir_511", signal(1152 * 16, 2, 10, 0.05), 44100, [G()], max_is=15)
    add("reservoir_vbr", signal(1152 * 16, 2, 11), 44100, SWITCH, max_is=40, bitrate=[128, 320, 192, 256, 160, 320],
        stuff_to=300)
    add("tables_7_10_13", signal(1152 * 6, 2, 12), 44100, [G(tables=(7, 10, 13), count1=0)], max_is=5)
    add("tables_5_6_9", signal(1152 * 6, 2, 13), 44100, [G(tables=(5, 6, 9), count1=1)], max_is=3)
    add("tables_2_3_8", signal(1152 * 6, 2, 14), 44100, [G(tables=(2, 3, 8))], max_is=1)
    add("tables_11_12_15", signal(1152 * 6, 2, 15), 44100, [G(tables=(11, 12, 15))], max_is=7)
    add("linbits", signal(1152 * 6, 2, 16, 0.9), 44100, [G(tables=(31, 23, 24))], max_is=4000, bitrate=320)
    return out
