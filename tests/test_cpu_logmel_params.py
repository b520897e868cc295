"""CPU checks of the general log-mel front end (bt_logmel_config, include/beatthis.h): the float64 restatement of the
contract (tests/logmel_reference.py) against the reference's outputs (tests/golden/logmel_params.npz, written by
oracle/make_golden_logmel_params.py; inputs rebuilt from their seeds by logmel_reference.pcm_signal, filterbanks pinned
by their SHA-256), the host-built tables, and the arguments the contract rejects."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import logmel_reference as R
from conftest import GOLDEN

from beat_this_b200.preprocessing import LogMelSpect, MelTables, filterbank_csr, mel_filterbank

REF_TOL = 2e-3  # the log-mel contract (DESIGN section 2): the reference computes in fp32


def _fixture():
    g = np.load(os.path.join(GOLDEN, "logmel_params.npz"))
    return g, [json.loads(str(g[f"cfg{k}"])) for k in range(int(g["n"]))]


def _fmax(cfg):
    return cfg["f_max"] if cfg["f_max"] is not None else float(cfg["sample_rate"] // 2)


def _fb(cfg):
    """The filterbank of a configuration, built here; test_filterbank_is_bitwise_the_reference pins it to the
    reference's."""
    return mel_filterbank(cfg["n_fft"] // 2 + 1, cfg["f_min"], _fmax(cfg), cfg["n_mels"], cfg["sample_rate"],
                          cfg["mel_scale"]).numpy()


def _x(g, k, j):
    seed, n = (int(v) for v in g[f"sig{k}_{j}"])
    return R.pcm_signal(seed, n)


def test_fixture_covers_the_parameter_space():
    g, cfgs = _fixture()
    assert len(cfgs) >= 16
    assert {c["n_fft"] for c in cfgs} >= {64, 256, 512, 1024, 2048, 4096, 8192}
    assert {c["sample_rate"] for c in cfgs} >= {8000, 11025, 16000, 22050, 44100, 48000}
    assert {c["mel_scale"] for c in cfgs} == {"slaney", "htk"}
    assert {json.dumps(c["normalized"]) for c in cfgs} == {'"frame_length"', '"window"', "true", "false"}
    assert {float(c["power"]) for c in cfgs} == {0.5, 1.0, 2.0} and {float(c["log_multiplier"]) for c in cfgs} == {1, 1e3, 1e4}
    assert {c["n_mels"] for c in cfgs} >= {1, 40, 80, 128, 229, 256}
    assert any(c["hop_length"] == 1 for c in cfgs) and any(c["hop_length"] > c["n_fft"] for c in cfgs)
    assert any(c["f_max"] is None for c in cfgs) and any(c["f_max"] is not None for c in cfgs)
    assert tuple(cfgs[0].values()) == LogMelSpect.DEFAULTS
    assert any((g[f"fb_nnz{k}"] == 0).any() for k in range(len(cfgs)))  # a configuration with all-zero bands
    for k, c in enumerate(cfgs):
        assert int(g[f"sig{k}_0"][1]) == c["n_fft"] // 2 + 1 and int(g[f"sig{k}_1"][1]) > c["hop_length"]


def test_restatement_matches_reference_fixture():
    g, cfgs = _fixture()
    for k, c in enumerate(cfgs):
        fb = _fb(c)
        for j in (0, 1):
            x, y = _x(g, k, j), g[f"y{k}_{j}"]
            ref = R.logmel(x, fb, c["n_fft"], c["hop_length"], c["normalized"], c["power"], c["log_multiplier"])
            assert ref.shape == y.shape == (1 + len(x) // c["hop_length"], c["n_mels"])
            err = np.abs(ref - y).max()
            assert err <= REF_TOL, (k, j, err)
            # the reference's own fp32 result lies within the bound stated for the device kernel
            lo, hi = R.device_bound(x, fb, c["n_fft"], c["hop_length"], c["normalized"], c["power"], c["log_multiplier"])
            assert (y >= lo).all() and (y <= hi).all(), (k, j)


def test_filterbank_is_bitwise_the_reference():
    g, cfgs = _fixture()
    for k, c in enumerate(cfgs):
        fb = mel_filterbank(c["n_fft"] // 2 + 1, c["f_min"], _fmax(c), c["n_mels"], c["sample_rate"], c["mel_scale"])
        assert fb.dtype == torch.float32 and fb.is_contiguous() and list(fb.shape) == g[f"fb_shape{k}"].tolist(), k
        assert np.array_equal((fb != 0).sum(0).numpy(), g[f"fb_nnz{k}"]), k
        assert hashlib.sha256(fb.numpy().tobytes()).hexdigest() == str(g[f"fb_sha256{k}"]), k
        tables = MelTables(*(c[a] for a in ("sample_rate", "n_fft", "hop_length", "f_min", "f_max", "n_mels", "mel_scale",
                                             "normalized", "power", "log_multiplier")))
        assert torch.equal(tables.fb, fb)


def test_csr_packing_round_trips():
    g, cfgs = _fixture()
    for k, c in enumerate(cfgs):
        fb = _fb(c)
        start, ptr, w = filterbank_csr(fb)
        assert start.dtype == ptr.dtype == np.int32 and w.dtype == np.float32
        assert ptr[0] == 0 and (np.diff(ptr) >= 0).all() and ptr[-1] == len(w)
        back = np.zeros_like(fb)
        for m in range(fb.shape[1]):
            run = w[ptr[m]:ptr[m + 1]]
            assert start[m] + len(run) <= fb.shape[0]
            back[start[m]:start[m] + len(run), m] = run
        assert np.array_equal(back, fb), k


def test_twiddles_and_window():
    t = MelTables(16000, 64, 10, 0, None, 8, "slaney", False, 1, 1)
    tw = t.twiddle.reshape(-1, 2).astype(np.float64)
    j = np.arange(32)
    assert np.abs(tw[:, 0] + 1j * tw[:, 1] - np.exp(-2j * np.pi * j / 64)).max() < 2 ** -24
    assert torch.equal(t.window, torch.hann_window(64, periodic=True))
    assert (t.config.n_fft, t.config.hop_length, t.config.n_mels, t.config.norm_mode) == (64, 10, 8, 0)


@pytest.mark.parametrize("kwargs, error", [
    ({"normalized": "frame"}, ValueError),
    ({"normalized": "Window"}, ValueError),
    ({"normalized": 1}, TypeError),
    ({"mel_scale": "mel"}, ValueError),
    ({"f_min": 12000}, ValueError),
    ({"f_min": 9000, "f_max": None, "sample_rate": 16000}, ValueError),
    ({"power": None}, NotImplementedError),
    ({"power": 0}, NotImplementedError),
    ({"power": -1.0}, NotImplementedError),
    ({"power": float("inf")}, NotImplementedError),
    ({"log_multiplier": float("nan")}, NotImplementedError),
    ({"n_fft": 1000}, NotImplementedError),
    ({"n_fft": 32}, NotImplementedError),
    ({"n_fft": 16384}, NotImplementedError),
    ({"hop_length": 0}, NotImplementedError),
    ({"n_mels": 0}, NotImplementedError),
    ({"n_mels": 1025}, NotImplementedError),
])
def test_rejected_arguments_raise_the_contracts_error(kwargs, error):
    with pytest.raises(error):
        LogMelSpect(**kwargs, device="cuda")  # raises before any device is touched
