"""The resampler's reference and bound (tests/resample_reference.py) without a GPU: a float32 emulation of
resample_kernel's operation order stays within the bound at every rate the GPU test runs, and the indexing mistakes a
kernel could make (a tap off by one, the phase row off by one, the K mod 4 tail dropped, a neighbouring clip's samples
read instead of zeros) each exceed it."""
import math

import numpy as np
import pytest

import resample_reference as R
from beat_this_b200 import preprocessing as P

RATES = ([(sr, R.SR) for sr in R.INFERENCE_RATES] + R.pitch_rate_pairs(44100) + R.pitch_rate_pairs(22050)
         + [(R.OPT_IN_RATE, R.SR), (R.MAX_RATE, R.SR)])


def _case(sr_in, sr_out, n_out=600, seed=0, clicks=False):
    """A clip of about n_out outputs and the indices checked: all of them for short filters, a spread of them for long
    ones (the direct form costs K + 3 kernel evaluations per output).  clicks: isolated unit impulses K + 5 samples
    apart instead of noise, so that an output's sum holds one term."""
    coef, L, M, K = R.bank(sr_in, sr_out)
    rng = np.random.default_rng(seed + sr_in)
    x = rng.uniform(-1, 1, int(math.ceil(n_out * M / L)) + K // 2).astype(np.float32)
    if clicks:
        x = np.where(np.arange(len(x)) % (K + 5) == 3, np.sign(x), 0).astype(np.float32)
    n_all = P.resampled_length(len(x), L, M)
    n = np.arange(n_all)
    if K > 1000:
        n = np.unique(np.r_[n[:100], n[-100:], rng.choice(n_all, 100, replace=False)])
    return x, coef, L, M, K, n


def test_kernel_slope_constant():
    """H_SLOPE bounds |h'(t)| (the float64 phase term of the bound): central differences on a fine grid."""
    t = np.linspace(-P.RESAMPLE_ZERO_CROSSINGS, P.RESAMPLE_ZERO_CROSSINGS, 2_000_001)
    d = np.diff(P.resample_kernel(t)) / np.diff(t)
    assert np.abs(d).max() < 0.9 * R.H_SLOPE, np.abs(d).max()


def test_rate_families():
    """The GPU test's special ratios are what their names say."""
    for sr, more in ((R.OPT_IN_RATE, True), (R.MAX_RATE, True), (R.REFUSED_RATE, True), (44100, False)):
        coef, L, M, K = R.bank(sr)
        assert coef.shape == (L, K) and K == R.taps(sr)
        assert (R.staged_bytes(L, M, K) > R.SMEM_OPT_IN) == more, sr
    assert R.staged_bytes(1, 32, R.taps(R.OPT_IN_RATE)) < R.MAX_SMEM
    assert R.staged_bytes(*P.resample_ratio(R.MAX_RATE), R.taps(R.MAX_RATE)) <= R.MAX_SMEM
    assert R.staged_bytes(*P.resample_ratio(R.REFUSED_RATE), R.taps(R.REFUSED_RATE)) > R.MAX_SMEM
    L, M = P.resample_ratio(R.HUGE_BANK_RATE)
    assert L * R.taps(R.HUGE_BANK_RATE) > 1 << 26
    with pytest.raises(ValueError):
        P.resample_filter_bank(R.HUGE_BANK_RATE)
    pitch = R.pitch_rate_pairs(44100)
    assert len(pitch) == 11 and all(sr_out == 44100 for _, sr_out in pitch)
    assert any(max(P.resample_ratio(*p)) > 10000 for p in pitch)  # ratios that barely reduce: L, M in the tens of thousands


@pytest.mark.parametrize("sr_in,sr_out", RATES, ids=[f"{a}-{b}" for a, b in RATES])
def test_emulation_is_within_the_bound(sr_in, sr_out):
    x, coef, L, M, K, n = _case(sr_in, sr_out)
    ref, bound, trunc = R.direct(x.astype(np.float64), sr_in, sr_out, n)
    r = R.ratio(R.emulate(x, coef, L, M, K, n), ref, bound, trunc)
    print(f"resample {sr_in} -> {sr_out} (L {L}, M {M}, K {K}): emulation at {r:.3f} of its bound")
    assert r <= 1


def _perturbed():
    """(name, sr_in, sr_out, emulate keywords): each mistake at rates where it changes the arithmetic (the phase row
    needs L > 1, the tail K = 2 mod 4)."""
    out = []
    tail = [(a, b) for a, b in RATES if R.taps(a, b) % 4 == 2]
    assert tail, "no rate with K = 2 mod 4"
    for a, b in [(44100, R.SR), (48000, R.SR), R.pitch_rate_pairs(44100)[5], (R.OPT_IN_RATE, R.SR)]:
        out.append(("tap+1", a, b, {"tap_shift": 1}))
        out.append(("tap-1", a, b, {"tap_shift": -1}))
        out.append(("neighbour", a, b, {"outside": True}))
        if P.resample_ratio(a, b)[0] > 1:
            out.append(("row+1", a, b, {"row_shift": 1}))
    for a, b in tail[:3]:  # its two taps sit where the window is ~1e-7: noise hides them, an isolated click does not
        out.append(("no tail", a, b, {"drop_tail": True}))
    return out


@pytest.mark.parametrize("name,sr_in,sr_out,kw", _perturbed(), ids=[f"{c[0]}-{c[1]}" for c in _perturbed()])
def test_indexing_mistakes_exceed_the_bound(name, sr_in, sr_out, kw):
    x, coef, L, M, K, n = _case(sr_in, sr_out, n_out=300, seed=1, clicks=name == "no tail")
    if kw.get("outside"):
        rng = np.random.default_rng(2)
        kw = {"outside": (rng.uniform(-1, 1, K), rng.uniform(-1, 1, K))}
        n = np.unique(np.r_[n[: 2 * K], n[-2 * K :]])  # outputs whose taps reach past the clip
    ref, bound, trunc = R.direct(x.astype(np.float64), sr_in, sr_out, n)
    r = R.ratio(R.emulate(x, coef, L, M, K, n, **kw), ref, bound, trunc)
    print(f"resample {sr_in} -> {sr_out}, {name}: {r:.3g} x its bound")
    assert r > 1, f"{name} at {sr_in} -> {sr_out} stays within the bound ({r:.3g})"
