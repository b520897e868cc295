"""The Ogg Vorbis tests' corpus, error bound and the calls that probe, stage and decode files (tests/test_cpu_vorbis.py,
tests/test_gpu_vorbis.py)."""
import ctypes

import numpy as np

import vorbis_reference as V
from beat_this_b200 import _lib

# The fp32 chain of one output value: the VQ value and the floor table entry (each rounded once), up to eight cascade
# additions and the coupling's add, the product, the pre-twiddle, log2(N/4) radix passes (each a twiddle product and
# at most three butterfly stages), the post-twiddle, the window and the overlap-add.  Each step rounds by at most 2^-24
# of a value bounded by the L1 norm of the packet's spectrum (V.Decoded.l1, which bounds every partial sum), so one
# output value is off by at most K(N) 2^-24 times the L1 norms of its two packets, K(N) = 4 log2(N) + 20.
def max_err(l1: float, n_max: int = 8192) -> float:
    return (4 * np.log2(n_max) + 20) * 2.0**-24 * 2 * l1


def probe(path):
    info = _lib.bt_vorbis_info()
    code = _lib.load().bt_vorbis_probe(str(path).encode(), ctypes.byref(info))
    return code, info


def stage(paths, infos):
    fo, status_at, bo, total = _lib.vorbis_layout(infos)
    buf = np.zeros(max(total, 1), dtype=np.uint8)
    npk, pb, bs, status = _lib.stage_vorbis_files(paths, infos, buf.ctypes.data, 1)
    return buf, npk, pb, bs, status


def host_decode(paths, mode=_lib.BT_VORBIS_CHANNELS_F64, corrupt=None):
    """Probe, stage and decode files through bt_debug_vorbis_decode_host into a NaN-filled output: (outputs per file,
    statuses, infos).  corrupt(buf, infos, npk) may change the staged data."""
    infos = [probe(p)[1] for p in paths]
    buf, npk, pb, bs, status = stage(paths, infos)
    if corrupt is not None:
        corrupt(buf, infos, npk)
    per = [1 if mode == _lib.BT_VORBIS_MONO_F32 else i.channels for i in infos]
    oo = _lib.offsets(i.n_samples * p for i, p in zip(infos, per))
    out = np.full(max(oo[-1], 1), np.nan, dtype=np.float32 if mode == _lib.BT_VORBIS_MONO_F32 else np.float64)
    st = np.array(status, dtype=np.int32)
    streams = _lib.vorbis_streams(infos, npk, pb, bs, oo[:-1])
    assert _lib.load().bt_debug_vorbis_decode_host(buf.ctypes.data, buf.ctypes.data, streams, len(paths), mode,
                                                   out.ctypes.data, st.ctypes.data) == 0
    res = [out[oo[i]:oo[i + 1]].reshape(-1, per[i]) if per[i] > 1 else out[oo[i]:oo[i + 1]] for i in range(len(paths))]
    return res, st.tolist(), infos


def signal(n: int, ch: int, seed: int, level: float = 0.3) -> np.ndarray:
    """Tones, a chirp and noise [n, ch], the channels correlated but not equal."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 44100
    base = np.sin(2 * np.pi * 440 * t) + 0.6 * np.sin(2 * np.pi * (2000 + 3000 * t) * t) + 0.3 * rng.standard_normal(n)
    chans = [base * (0.6 + 0.4 * c / max(ch, 1)) + 0.3 * rng.standard_normal(n) for c in range(ch)]
    return level * np.stack(chans, axis=1) / 2


def flags(n: int, seed: int):
    """A block-flag sequence with every transition (long-long, long-short, short-short, short-long)."""
    rng = np.random.default_rng(seed)
    return [1, 1, 0, 0, 1, 0, 1] + [int(v) for v in rng.integers(0, 2, n)]


def corpus_signals():
    """(name, signal) of the corpus's streams."""
    return [(name, sig) for name, sig, _ in _specs()]


def corpus():
    """(name, stream bytes) of synthetic streams covering the decoder's features."""
    return [(name, V.encode(sig, plan)) for name, sig, plan in _specs()]


def _specs():
    S = V.standard_setup
    out = []

    def add(name, setup, sig, fl, **kw):
        out.append((name, sig, V.Plan(setup, fl, **kw)))

    add("mono_r1", S(channels=1, residue_type=1, coupled=False), signal(9000, 1, 1), flags(6, 1))
    add("stereo_r2", S(), signal(12000, 2, 2), flags(8, 2))
    add("stereo_r1_lookup2_seq", S(residue_type=1, lookup=2, sequence_p=1), signal(9000, 2, 3), flags(6, 3))
    add("stereo_r0_one_pass", S(residue_type=0, cascade=1, ordered=True), signal(9000, 2, 4), flags(6, 4))
    add("six_r2_submaps", S(channels=6, submaps=2), signal(6000, 6, 5), flags(4, 5))
    add("blocks_64_64", S(bs=(64, 64), sparse=True), signal(3000, 2, 6), [0] * 60)
    add("blocks_512_8192", S(bs=(512, 8192)), signal(30000, 2, 7), flags(4, 7))
    add("many_per_page", S(), signal(12000, 2, 8), flags(8, 8), packets_per_page=9, page_bytes=60000)
    add("spanning_pages", S(), signal(12000, 2, 9), flags(8, 9), page_bytes=300)
    add("front_end_trim", S(), signal(12000, 2, 10), flags(8, 10), trim_front=700, trim_end=300)
    add("cut_packets", S(), signal(12000, 2, 11), flags(8, 11), cut={3: 2, 5: 40, 8: 300})
    return out
