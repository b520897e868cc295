"""GPU tests of the general log-mel kernel (bt_logmel_config, contract in include/beatthis.h) behind LogMelSpect with
non-default analysis parameters.

Bounds (stated):
  - against the reference's outputs (tests/golden/logmel_params.npz): max-abs <= 2e-3, the log-mel contract of
    DESIGN section 2 (fp32 FFT round-off amplified by log1p(m x) near silence);
  - against the float64 restatement (tests/logmel_reference.py): every element inside device_bound(), whose
    derivation is its docstring (fp32 FFT error charged per radix-2 stage, |.|^p and the band sums mapped as
    intervals, then log1p(m x) applied to the interval ends, which is where m multiplies absolute error near 0).
"""
import ctypes
import json
import os
from ctypes import c_void_p

import numpy as np
import pytest
import torch

import logmel_reference as R
from conftest import GOLDEN
from support import dev  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900), pytest.mark.usefixtures("lib_built")]

REF_TOL = 2e-3


@pytest.fixture(scope="module")
def fixture():
    g = np.load(os.path.join(GOLDEN, "logmel_params.npz"))
    return g, [json.loads(str(g[f"cfg{k}"])) for k in range(int(g["n"]))]


def _check_bound(out, x, fb, c, what):
    lo, hi = R.device_bound(x, fb, c["n_fft"], c["hop_length"], c["normalized"], c["power"], c["log_multiplier"])
    bad = (out < lo) | (out > hi) | ~np.isfinite(out)
    assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the float64 bound, e.g. at {np.argwhere(bad)[:3]}"


def _run(mel, signals, fill=float("nan")):
    """bt_logmel_config (bt_logmel for the defaults, whose LogMelSpect has no tables) into an output pre-filled with
    `fill`, so that a missing store shows."""
    eng, t = mel.engine, mel.tables
    sigs = [torch.as_tensor(s, dtype=torch.float32, device=eng.device) for s in signals]
    so = np.concatenate([[0], np.cumsum([len(s) for s in sigs])]).tolist()
    hop, n_mels = (441, 128) if t is None else (t.hop_length, t.n_mels)
    fo = eng.frame_offsets(so, hop)
    spect = torch.full((fo[-1], n_mels), fill, dtype=torch.float32, device=eng.device)
    audio, so_h, fo_h = torch.cat(sigs), (ctypes.c_int64 * len(so))(*so), (ctypes.c_int64 * len(fo))(*fo)
    if t is None:
        code = eng.lib.bt_logmel(eng.ctx, c_void_p(audio.data_ptr()), so_h, len(sigs), c_void_p(spect.data_ptr()), fo_h,
                                 eng._stream())
    else:
        d = mel.device_tables
        code = eng.lib.bt_logmel_config(
            eng.ctx, ctypes.byref(t.config), *(c_void_p(d[k].data_ptr()) for k in ("window", "twiddle", "fb_start", "fb_ptr", "fb_w")),
            c_void_p(audio.data_ptr()), so_h, len(sigs), c_void_p(spect.data_ptr()), fo_h, eng._stream())
    assert code == 0, eng.lib.bt_last_error(eng.ctx)
    torch.cuda.synchronize()
    return [spect[fo[i]:fo[i + 1]].cpu().numpy() for i in range(len(sigs))]


def _x(g, k, j):
    seed, n = (int(v) for v in g[f"sig{k}_{j}"])
    return R.pcm_signal(seed, n)


def test_every_fixture_configuration(dev, fixture):
    from beat_this_b200.preprocessing import LogMelSpect

    g, cfgs = fixture
    for k, c in enumerate(cfgs):
        mel = LogMelSpect(**c, device=dev, _general=True)
        xs = [_x(g, k, 0), _x(g, k, 1)]
        batched = mel.batch([torch.tensor(x, device=dev) for x in xs])
        for j, x in enumerate(xs):
            single = mel(torch.tensor(x, device=dev)).cpu().numpy()
            out = batched[j].cpu().numpy()
            y = g[f"y{k}_{j}"]
            assert out.shape == y.shape and np.array_equal(single, out), (k, j)
            err = np.abs(out - y).max()
            print(f"config {k} signal {j}: max abs err vs reference {err:.2e}")
            assert err <= REF_TOL, (k, j, err)
            _check_bound(out, x, mel.tables.fb.numpy(), c, f"config {k} signal {j}")  # bitwise the reference's


def test_issue_example_matches_reference(dev, fixture):
    from beat_this_b200.preprocessing import LogMelSpect

    g, cfgs = fixture
    kw = dict(sample_rate=44100, n_fft=2048, hop_length=512, n_mels=80, mel_scale="htk", normalized=False, power=2.0)
    k = next(i for i, c in enumerate(cfgs) if all(c[a] == v for a, v in kw.items()) and c["f_max"] == 11000)
    mel = LogMelSpect(**kw, device=dev)
    assert mel.tables is not None  # the general kernel
    out = mel(torch.tensor(_x(g, k, 1), device=dev)).cpu().numpy()
    assert np.abs(out - g[f"y{k}_1"]).max() <= REF_TOL


@pytest.mark.parametrize("cfg", [
    dict(sample_rate=8000, n_fft=64, hop_length=1, f_min=0, f_max=None, n_mels=40, mel_scale="htk", normalized=False,
         power=2.0, log_multiplier=1e4),
    dict(sample_rate=16000, n_fft=512, hop_length=160, f_min=0, f_max=None, n_mels=80, mel_scale="slaney",
         normalized="window", power=0.5, log_multiplier=1000),
    dict(sample_rate=44100, n_fft=8192, hop_length=441, f_min=30, f_max=16000, n_mels=256, mel_scale="slaney",
         normalized="frame_length", power=1, log_multiplier=1000),
    # the defaults: the model path's logmel_kernel (bt_logmel), every Audio2Frames call and the benchmark run it
    dict(sample_rate=22050, n_fft=1024, hop_length=441, f_min=30, f_max=11000, n_mels=128, mel_scale="slaney",
         normalized="frame_length", power=1, log_multiplier=1000),
])
def test_ragged_batches_edges_and_repeatability(dev, cfg):
    """Batches of 1, 7 and 213 clips (enough frame groups for several grid-stride rounds at every n_fft), lengths of
    exactly n_fft // 2 + 1, = 0 and = hop - 1 (mod hop), and clips far longer than one CTA's span; outputs start as NaN
    and must match the float64 bound; a second run is bitwise the first."""
    from beat_this_b200.preprocessing import LogMelSpect, MelTables

    mel = LogMelSpect(**cfg, device=dev)
    assert (mel.tables is None) == (tuple(cfg.values()) == LogMelSpect.DEFAULTS)
    tables = mel.tables if mel.tables is not None else MelTables(*LogMelSpect.DEFAULTS)
    n, hop = cfg["n_fft"], cfg["hop_length"]
    rng = np.random.default_rng(n + hop)
    base = [n // 2 + 1, hop * (n // hop + 3), hop * (n // hop + 3) + hop - 1, 40 * n + 13]
    for n_clips in (1, 7, 213):
        lens = (base * (n_clips // len(base) + 1))[:n_clips]
        lens = [int(v + (rng.integers(0, 3 * n) if i >= len(base) else 0)) for i, v in enumerate(lens)]
        sigs = [(0.2 * rng.standard_normal(v)).astype(np.float32) for v in lens]
        outs = _run(mel, sigs)
        for s, o in zip(sigs, outs):
            assert o.shape == (1 + len(s) // hop, cfg["n_mels"])
        fb = tables.fb.numpy()
        for i in sorted(set(rng.integers(0, n_clips, 6).tolist()) | {0, n_clips - 1}):
            _check_bound(outs[i], sigs[i], fb, cfg, f"{n_clips} clips, clip {i}")
        again = _run(mel, sigs, fill=0.0)
        assert all(np.array_equal(a, b) for a, b in zip(outs, again))


def test_general_kernel_at_defaults_matches_the_model_path(dev):
    from beat_this_b200 import synthetic
    from beat_this_b200.preprocessing import LogMelSpect

    g = np.load(os.path.join(GOLDEN, "logmel.npz"))
    fused, general = LogMelSpect(device=dev), LogMelSpect(device=dev, _general=True)
    assert fused.tables is None and general.tables is not None
    for idx in (0, 1):
        x = torch.tensor(synthetic.synth_clip(idx, float(g[f"clip{idx}_secs"])), dtype=torch.float32, device=dev)
        a, b = fused(x).cpu().numpy(), general(x).cpu().numpy()
        assert a.shape == b.shape == g[f"clip{idx}_mel"].shape
        assert np.abs(a - b).max() <= REF_TOL and np.abs(b - g[f"clip{idx}_mel"]).max() <= REF_TOL


def test_which_kernel_runs(dev):
    """The ctx's launch profile names every kernel the library launches (BT_LAUNCHED): one launch of `logmel` for a
    default LogMelSpect, one of `logmel_config` otherwise."""
    from beat_this_b200.preprocessing import LogMelSpect

    x = torch.randn(30000, device=dev) * 0.1
    default, other = LogMelSpect(device=dev), LogMelSpect(n_fft=2048, hop_length=512, device=dev)
    for mel, name in ((default, "logmel"), (other, "logmel_config")):
        mel(x)
        torch.cuda.synchronize()
        mel.engine.profile_enable(True)
        mel.engine.profile_reset()
        before = mel.engine.launches
        mel(x)
        assert mel.engine.launches == before + 1
        prof = mel.engine.profile_results()
        mel.engine.profile_enable(False)
        assert set(prof) == {name} and prof[name][1] == 1, prof


def test_bad_offsets_are_refused_before_anything_is_enqueued(dev):
    from beat_this_b200._lib import BTError
    from beat_this_b200.preprocessing import LogMelSpect

    mel = LogMelSpect(n_fft=512, hop_length=160, sample_rate=16000, f_max=None, device=dev)
    eng, t, d = mel.engine, mel.tables, mel.device_tables
    audio = torch.zeros(5000, device=dev)
    spect = torch.zeros(100, t.n_mels, device=dev)

    def call(so, fo, cfg=t.config):
        return eng.lib.bt_logmel_config(
            eng.ctx, ctypes.byref(cfg), *(c_void_p(d[k].data_ptr()) for k in ("window", "twiddle", "fb_start", "fb_ptr", "fb_w")),
            c_void_p(audio.data_ptr()), (ctypes.c_int64 * len(so))(*so), len(so) - 1, c_void_p(spect.data_ptr()),
            (ctypes.c_int64 * len(fo))(*fo), eng._stream())

    before = eng.launches
    assert call([0, 256], [0, 2]) == -1  # n_fft // 2 samples: reflect padding needs more
    assert call([0, 1000, 900], [0, 7, 7]) == -1  # decreasing sample offsets
    assert call([0, 1000], [0, 6]) == -1  # 1 + 1000 // 160 = 7 frames
    assert call([0, 1000], [1, 8]) == -1  # frame offsets must start at 0
    bad = type(t.config)(500, 160, t.n_mels, 0, 1.0, 1000.0)
    assert call([0, 1000], [0, 7], bad) == -1  # n_fft not a power of two
    assert eng.launches == before
    with pytest.raises(BTError):
        mel([0.0] * 256)
    assert call([0, 1000], [0, 7]) == 0 and eng.launches == before + 1
