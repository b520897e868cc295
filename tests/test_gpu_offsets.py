"""Host CSR offsets (include/beatthis.h, Conventions): the entry points that take them refuse offsets that start below 0
(or away from 0 where they say so) or decrease.  Each refusal returns BT_ERR_ARG before anything is enqueued: the error
names the entry point, nothing is launched, bt_audio2frames allocates nothing, and a valid call that follows gives
bitwise what a fresh context gives.  Every entry point here also runs once on contexts created with BT_SYNC_DEBUG=1."""
import ctypes
import os
from ctypes import c_void_p

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

BT_ERR_ARG = -1
SO = [0, 3000, 8000]  # two clips: 1 + 3000 // 441 = 7 and 1 + 5000 // 441 = 12 frames
FO = [0, 7, 19]


def p(t):
    return c_void_p(t.data_ptr())


def i64(v):
    return (ctypes.c_int64 * len(v))(*[int(x) for x in v])


def _engines(small0_ckpt):
    from beat_this_b200.engine import Engine
    from beat_this_b200.inference import Spect2Frames

    return {"mel": Engine.mel_only("cuda:0"), "model": Spect2Frames(small0_ckpt, "cuda:0", False).model.engine}


@pytest.fixture(scope="module")
def ctxs(lib_built, small0_ckpt):
    """(used, fresh): contexts that see the refused calls first, and contexts that see only valid ones."""
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device")
    return _engines(small0_ckpt), _engines(small0_ckpt)


@pytest.fixture(scope="module")
def data():
    g = torch.Generator(device="cuda:0").manual_seed(7)
    audio = 0.1 * torch.randn(SO[-1], generator=g, device="cuda:0")
    spect = torch.rand(FO[-1], 128, generator=g, device="cuda:0") * 7
    logits = torch.randn(2, FO[-1], generator=g, device="cuda:0") * 4
    return audio, spect, logits


def _bank():
    from beat_this_b200 import preprocessing as P

    coef, L, M, K = P.resample_filter_bank(44100)
    oo = [0]
    for a, b in zip(SO[:-1], SO[1:]):
        oo.append(oo[-1] + P.resampled_length(b - a, L, M))
    return torch.from_numpy(coef).cuda(), L, M, K, oo


def _calls(data):
    """{entry point: (call(engine, *offsets) -> code, valid offsets, engine key)} writing into scratch outputs."""
    from beat_this_b200.engine import chunking_struct

    audio, spect, (beat, down) = data
    out = torch.empty(4 * SO[-1], device="cuda:0")
    spect_out = torch.empty(FO[-1] + 64, 128, device="cuda:0")
    coef, L, M, K, oo = _bank()
    ck = chunking_struct(1500, 6, "keep_first")
    times = torch.empty(2, 2, FO[-1], dtype=torch.float64, device="cuda:0")
    counts = torch.empty(2, 2, dtype=torch.int32, device="cuda:0")
    peaks = lambda: (p(times[0]), p(counts[0]), p(times[1]), p(counts[1]), FO[-1])  # noqa: E731
    return {
        "bt_logmel": (lambda e, so, fo: e.lib.bt_logmel(e.ctx, p(audio), i64(so), len(so) - 1, p(spect_out), i64(fo), None),
                      (SO, FO), "mel"),
        "bt_resample": (lambda e, so, oo_: e.lib.bt_resample(e.ctx, p(audio), i64(so), len(so) - 1, p(coef), L, M, K, p(out),
                                                             i64(oo_), None), (SO, oo), "mel"),
        "bt_spect2frames": (lambda e, fo: e.lib.bt_spect2frames(e.ctx, p(spect), i64(fo), len(fo) - 1, p(out), p(out[FO[-1]:]),
                                                                None), (FO,), "model"),
        "bt_spect2frames_chunked": (lambda e, fo: e.lib.bt_spect2frames_chunked(e.ctx, p(spect), i64(fo), len(fo) - 1, p(out),
                                                                                p(out[FO[-1]:]), ctypes.byref(ck), None),
                                    (FO,), "model"),
        "bt_audio2frames": (lambda e, so, fo: e.lib.bt_audio2frames(e.ctx, p(audio), i64(so), len(so) - 1, p(out),
                                                                    p(out[FO[-1]:]), i64(fo), None), (SO, FO), "model"),
        "bt_audio2frames_chunked": (lambda e, so, fo: e.lib.bt_audio2frames_chunked(
            e.ctx, p(audio), i64(so), len(so) - 1, p(out), p(out[FO[-1]:]), i64(fo), ctypes.byref(ck), None), (SO, FO), "model"),
        "bt_peakpick": (lambda e, fo: e.lib.bt_peakpick(e.ctx, p(beat), p(down), i64(fo), len(fo) - 1, *peaks(), None),
                        (FO,), "mel"),
        "bt_peakpick_fps": (lambda e, fo: e.lib.bt_peakpick_fps(e.ctx, p(beat), p(down), i64(fo), len(fo) - 1, 100.0, *peaks(),
                                                                None), (FO,), "mel"),
    }


def _bad(name):
    """The refused offsets of an entry point: every check it lacked before (a negative start, offsets that decrease,
    for bt_logmel and bt_audio2frames also frame offsets that do not start at 0), one argument at a time."""
    two = {"bt_logmel", "bt_audio2frames", "bt_audio2frames_chunked"}
    if name in two:
        return [([-441, 2559, 7559], FO), ([0, 8000, 3000], FO), (SO, [1, 8, 20]), (SO, [0, 19, 7])]
    if name == "bt_resample":
        oo = _bank()[4]
        return [([-1, 2999, 7999], oo), (SO, [-1] + oo[1:]), ([0, 8000, 3000], oo), (SO, [0, oo[2], oo[1]])]
    return [([-1, 6, 18],), ([0, 12, 7],)]


def _valid_outputs(eng, name, data):
    """A valid call through the Python layer: its outputs as host arrays."""
    audio, spect, (beat, down) = data
    if name == "bt_logmel":
        out = [eng.logmel_cat(audio, SO)[0]]
    elif name == "bt_resample":
        out = [eng.resample_cat(audio, SO, 44100)[0]]
    elif name.startswith("bt_spect2frames"):
        out = list(eng.spect2frames_cat(spect, FO, (1500, 6, "keep_first") if name.endswith("chunked") else None))
    elif name.startswith("bt_audio2frames"):
        out = list(eng.audio2frames_cat(audio, SO, (1500, 6, "keep_first") if name.endswith("chunked") else None)[:2])
    else:
        fps = 100.0 if name.endswith("fps") else 50.0
        return [a for pair in eng.peakpick_cat(beat, down, FO, fps) for a in pair]
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


NAMES = ["bt_logmel", "bt_resample", "bt_spect2frames", "bt_spect2frames_chunked", "bt_audio2frames",
         "bt_audio2frames_chunked", "bt_peakpick", "bt_peakpick_fps"]


@pytest.mark.parametrize("name", NAMES)
def test_bad_offsets_are_refused_before_anything_is_enqueued(ctxs, data, name):
    used, fresh = ctxs
    call, valid, key = _calls(data)[name]
    eng = used[key]
    assert call(eng, *valid) == 0, eng.lib.bt_last_error(eng.ctx)
    torch.cuda.synchronize()
    for offsets in _bad(name):
        before = eng.launches
        assert call(eng, *offsets) == BT_ERR_ARG, (name, offsets)
        msg = eng.lib.bt_last_error(eng.ctx).decode()
        assert msg.startswith(name + ":"), (offsets, msg)
        assert eng.launches == before, (name, offsets)
    got, want = _valid_outputs(eng, name, data), _valid_outputs(fresh[key], name, data)
    assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want)), name


@pytest.mark.parametrize("name", ["bt_audio2frames", "bt_audio2frames_chunked"])
def test_malformed_audio2frames_allocates_nothing(ctxs, data, name):
    """Frame offsets that claim 2 000 000 frames (a 1 GB spectrogram) and do not match the clips: refused before the
    spectrogram scratch grows, so the device's free memory stays where it was."""
    used, _ = ctxs
    call, _, key = _calls(data)[name]
    eng = used[key]
    torch.cuda.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    for so, fo in [(SO, [0, 7, 2_000_000]), ([-441, 2559, 2_000_000 * 441], [0, 7, 2_000_000])]:
        assert call(eng, so, fo) == BT_ERR_ARG
    torch.cuda.synchronize()
    assert free_before - torch.cuda.mem_get_info()[0] < 2_000_000 * 128 * 4 // 2


def test_every_entry_point_runs_under_sync_debug(lib_built, small0_ckpt, data):
    """One valid call of each entry point above, plus bt_stft, bt_phase_vocoder and bt_istft, on contexts created with
    BT_SYNC_DEBUG=1 (each launch is synchronised and checked as it is made)."""
    from beat_this_b200.augment import StftTables

    old = os.environ.get("BT_SYNC_DEBUG")
    os.environ["BT_SYNC_DEBUG"] = "1"
    try:
        engines = _engines(small0_ckpt)
    finally:
        if old is None:
            del os.environ["BT_SYNC_DEBUG"]
        else:
            os.environ["BT_SYNC_DEBUG"] = old
    for name, (call, valid, key) in _calls(data).items():
        eng = engines[key]
        before = eng.launches
        assert call(eng, *valid) == 0, (name, eng.lib.bt_last_error(eng.ctx))
        assert eng.launches > before, name
    eng = engines["mel"]
    t = StftTables(512, 128, eng.device)
    before = eng.launches
    spec, fo = eng.stft_cat(data[0], SO, t)
    v, vo = eng.phase_vocoder_cat(spec, fo, [0, 1], [1.25, 0.8])
    eng.istft_cat(v, vo, [2400, 6250], t)
    torch.cuda.synchronize()
    assert eng.launches - before == 4  # stft, phase_vocoder, istft, istft_overlap_add
