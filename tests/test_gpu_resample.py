"""resample_kernel through bt_resample / Engine.resample_cat against the float64 direct form, with the elementwise bound
of tests/resample_reference.py, at every rate it serves: the inference inputs to 22.05 kHz, the pitch-shift steps of
augment.py, a ratio whose staged span needs more than 48 KB of shared memory, the largest ratio bt_resample takes and
the next one (refused).  Ragged tables with empty, one-sample and filter-length clips, output counts around the
256-output CTA, offsets that do not start at 0 and NaN guards on both sides; ten-minute clips checked by sampling; and
more clips in one call than a grid holds in y -- for bt_resample, bt_logmel and bt_audio2frames.

`pytest -s` prints each family's worst error as a fraction of its bound."""
import ctypes
from ctypes import c_void_p

import numpy as np
import pytest
import torch

import resample_reference as R
from beat_this_b200 import preprocessing as P

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

BT_ERR_ARG = -1
GUARD_BITS = 0x7FC0DEAD  # a NaN no arithmetic produces: an output guard that still holds it was not written
MANY = 70_000  # clips in one call: more than the 65535 a grid holds in y


def p(t):
    return c_void_p(t.data_ptr())


def i64(v):
    return (ctypes.c_int64 * len(v))(*[int(x) for x in v])


@pytest.fixture(scope="module")
def eng(lib_built):
    from beat_this_b200.engine import Engine

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device")
    return Engine.mel_only("cuda:0")


WORST = {}


def _report(family, label, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    print(f"resample {family:10s} {label}: worst error {ratio:.3f} of its bound (family worst {WORST[family]:.3f})")


def _guarded(n, lead):
    """A float32 device buffer of lead + n + lead elements filled with the GUARD_BITS NaN."""
    return torch.full((2 * lead + n,), GUARD_BITS, dtype=torch.int32, device="cuda:0").view(torch.float32)


def _resample_table(eng, sr_in, sr_out, clips, n_outs):
    """One bt_resample call over `clips` (float32 arrays) with the output counts n_outs, laid out with NaN guards: the
    input starts after a guard and a guard clip of K NaN samples with no outputs sits between every two clips (a read
    past a clip's edge brings NaN in); the output buffer is GUARD_BITS-filled with guards before out_offsets[0] and
    after the last output.  Returns (outputs per clip, whole output buffer, launches)."""
    coef, L, M, K = R.bank(sr_in, sr_out)
    coef_d = torch.from_numpy(coef).cuda()
    g = K + 7
    parts, in_off, out_off = [np.full(g, np.nan, np.float32)], [g], [g]
    for x, n in zip(clips, n_outs):
        parts += [x, np.full(g, np.nan, np.float32)]
        in_off += [in_off[-1] + len(x), in_off[-1] + len(x) + g]
        out_off += [out_off[-1] + n, out_off[-1] + n]
    audio = torch.from_numpy(np.concatenate(parts)).cuda()
    out = _guarded(out_off[-1] - g, g)
    before = eng.launches
    code = eng.lib.bt_resample(eng.ctx, p(audio), i64(in_off), len(in_off) - 1, p(coef_d), L, M, K, p(out), i64(out_off),
                               None)
    assert code == 0, eng.lib.bt_last_error(eng.ctx)
    launches = eng.launches - before
    torch.cuda.synchronize()
    host = out.cpu().numpy()
    bits = host.view(np.int32)
    assert (bits[:g] == GUARD_BITS).all() and (bits[out_off[-1]:] == GUARD_BITS).all(), "a guard was written"
    got = [host[out_off[2 * i] : out_off[2 * i + 1]] for i in range(len(clips))]
    return got, host, launches, (audio, in_off, out_off, coef_d, L, M, K)


def _ragged(sr_in, sr_out, rng):
    """Input lengths 0, 1, K/2 - 1, K/2, K and a few thousand (their natural output counts), then output counts 255,
    256, 257, 511, 512 (around the 256-output CTA) from the inputs they need; noise, and one clip of isolated clicks."""
    _, L, M, K = R.bank(sr_in, sr_out)
    lens = [0, 1, K // 2 - 1, K // 2, K, 2000 + int(rng.integers(0, 3000))]
    n_outs = [P.resampled_length(n, L, M) for n in lens]
    for n in (255, 256, 257, 511, 512):
        lens.append(-(-n * M // L))
        n_outs.append(n)
    clips = [rng.uniform(-1, 1, n).astype(np.float32) for n in lens]
    clicks = np.zeros(lens[5], np.float32)
    clicks[3 :: K + 5] = 1.0  # one sample per output window: a term the noise would hide (the far taps) shows alone
    return clips + [clicks], n_outs + [n_outs[5]]


def _check_table(eng, family, sr_in, sr_out, seed):
    rng = np.random.default_rng(seed)
    clips, n_outs = _ragged(sr_in, sr_out, rng)
    got, host, launches, args = _resample_table(eng, sr_in, sr_out, clips, n_outs)
    assert launches == 1
    worst = 0.0
    for x, y in zip(clips, got):
        ref, bound, trunc = R.direct(x.astype(np.float64), sr_in, sr_out, np.arange(len(y)))
        worst = max(worst, R.ratio(y, ref, bound, trunc))
    _report(family, f"{sr_in} -> {sr_out}", worst)
    assert worst <= 1, f"{sr_in} -> {sr_out}: {worst:.3g} x its bound"
    # a second call writes the same bytes
    audio, in_off, out_off, coef_d, L, M, K = args
    out2 = _guarded(out_off[-1] - out_off[0], out_off[0])
    assert eng.lib.bt_resample(eng.ctx, p(audio), i64(in_off), len(in_off) - 1, p(coef_d), L, M, K, p(out2),
                               i64(out_off), None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(out2.cpu().numpy().view(np.int32), host.view(np.int32)), "a second call wrote other bytes"


@pytest.mark.parametrize("sr", R.INFERENCE_RATES)
def test_inference_rates(eng, sr):
    _check_table(eng, "inference", sr, R.SR, sr)


PITCH = R.pitch_rate_pairs(44100) + R.pitch_rate_pairs(22050)


@pytest.mark.parametrize("sr_in,sr_out", PITCH, ids=[f"{a}-{b}" for a, b in PITCH])
def test_pitch_shift_rates(eng, sr_in, sr_out):
    _check_table(eng, "pitch", sr_in, sr_out, sr_in + sr_out)


@pytest.mark.parametrize("sr", [R.OPT_IN_RATE, R.MAX_RATE], ids=["over-48KB", "largest"])
def test_large_shared_memory_ratios(eng, sr):
    _, L, M, K = R.bank(sr)
    assert R.staged_bytes(L, M, K) > R.SMEM_OPT_IN
    _check_table(eng, "large-smem", sr, R.SR, sr)


def test_ratio_above_the_shared_memory_limit_is_refused(eng):
    """The next integer ratio past the largest: BT_ERR_ARG before anything is enqueued (launch count and profile stay)."""
    coef, L, M, K = R.bank(R.REFUSED_RATE)
    assert R.staged_bytes(L, M, K) > R.MAX_SMEM
    coef_d = torch.from_numpy(coef).cuda()
    audio = torch.zeros(100_000, device="cuda:0")
    out = torch.zeros(1000, device="cuda:0")
    so, oo = [0, 100_000], [0, P.resampled_length(100_000, L, M)]
    eng.profile_enable(True)
    eng.profile_reset()
    before = eng.launches
    code = eng.lib.bt_resample(eng.ctx, p(audio), i64(so), 1, p(coef_d), L, M, K, p(out), i64(oo), None)
    assert code == BT_ERR_ARG and eng.lib.bt_last_error(eng.ctx).decode().startswith("bt_resample:")
    assert eng.launches == before
    prof = eng.profile_results()
    eng.profile_enable(False)
    assert not any(n for _, n in prof.values()), prof


def test_bank_too_large_raises_before_any_launch(eng):
    before = eng.launches
    with pytest.raises(ValueError):
        eng.resample_cat(torch.zeros(1000, device="cuda:0"), [0, 1000], R.HUGE_BANK_RATE)
    assert eng.launches == before


def test_negative_clip_count_is_refused(eng):
    coef, L, M, K = R.bank(44100)
    coef_d = torch.from_numpy(coef).cuda()
    buf = torch.zeros(16, device="cuda:0")
    before = eng.launches
    assert eng.lib.bt_resample(eng.ctx, p(buf), i64([0]), -1, p(coef_d), L, M, K, p(buf), i64([0]), None) == BT_ERR_ARG
    assert eng.lib.bt_last_error(eng.ctx).decode().startswith("bt_resample:")
    assert eng.lib.bt_logmel(eng.ctx, p(buf), i64([0]), -1, p(buf), i64([0]), None) == BT_ERR_ARG
    assert eng.lib.bt_last_error(eng.ctx).decode().startswith("bt_logmel:")
    assert eng.launches == before


LONG = [(48000, R.SR), (44100, R.SR), R.pitch_rate_pairs(44100)[0]]


@pytest.mark.parametrize("sr_in,sr_out", LONG, ids=[f"{a}-{b}" for a, b in LONG])
def test_ten_minute_clip(eng, sr_in, sr_out):
    """Ten minutes at sr_in between two short clips: the output count is resampled_length, and the direct form holds at
    the first and last 2K outputs, +-2 around 300 CTA boundaries and 20 000 random outputs."""
    _, L, M, K = R.bank(sr_in, sr_out)
    rng = np.random.default_rng(sr_in)
    x = rng.uniform(-1, 1, 600 * sr_in).astype(np.float32)
    short = [rng.uniform(-1, 1, n).astype(np.float32) for n in (300, 5000)]
    so = [0, len(short[0]), len(short[0]) + len(x), len(short[0]) + len(x) + len(short[1])]
    audio = torch.from_numpy(np.concatenate([short[0], x, short[1]])).cuda()
    before = eng.launches
    out, oo = eng.resample_cat(audio, so, sr_in, sr_out)
    assert eng.launches - before == 1
    n_out = P.resampled_length(len(x), L, M)
    assert oo[2] - oo[1] == n_out
    host = out.cpu().numpy()
    idx = R.sample_indices(n_out, K, rng)
    ref, bound, trunc = R.direct(x.astype(np.float64), sr_in, sr_out, idx)
    worst = R.ratio(host[oo[1] + idx], ref, bound, trunc)
    for c, i in ((short[0], 0), (short[1], 2)):
        ref_c, bound_c, trunc_c = R.direct(c.astype(np.float64), sr_in, sr_out, np.arange(oo[i + 1] - oo[i]))
        worst = max(worst, R.ratio(host[oo[i] : oo[i + 1]], ref_c, bound_c, trunc_c))
    _report("long", f"{sr_in} -> {sr_out}, {len(idx)} outputs", worst)
    assert worst <= 1


def _short_clips(rng, lo, hi, n=MANY):
    lens = rng.integers(lo, hi + 1, n)
    so = np.concatenate([[0], np.cumsum(lens)])
    return torch.from_numpy(rng.uniform(-1, 1, int(so[-1])).astype(np.float32)).cuda(), [int(v) for v in so]


def _per_1000(fn, so):
    """fn(audio-relative offsets of clips [a, b)) for the clips in runs of at most 1000."""
    return [fn(so[a : min(a + 1000, len(so) - 1) + 1]) for a in range(0, len(so) - 1, 1000)]


def test_many_clips_resample(eng):
    """70 000 clips of 0 to 700 samples at 48 kHz in one call: one launch, bitwise what calls of at most 1000 clips
    give, and the direct form's bound on 600 clips (every clip past the 65535th CTA row among them)."""
    rng = np.random.default_rng(70_000)
    audio, so = _short_clips(rng, 0, 700)
    before = eng.launches
    out, oo = eng.resample_cat(audio, so, 48000)
    assert eng.launches - before == 1
    host = out.cpu().numpy()
    parts = _per_1000(lambda s: eng.resample_cat(audio[s[0] : s[-1]], [v - s[0] for v in s], 48000)[0].cpu().numpy(), so)
    assert np.array_equal(np.concatenate(parts).view(np.int32), host.view(np.int32))
    check = np.unique(np.r_[rng.choice(MANY, 300, replace=False), [0, 65534, 65535, 65536, MANY - 1],
                            rng.choice(np.arange(65535, MANY), 300, replace=False)])
    a_host = audio.cpu().numpy().astype(np.float64)
    worst = 0.0
    for i in check:
        ref, bound, trunc = R.direct(a_host[so[i] : so[i + 1]], 48000, R.SR, np.arange(oo[i + 1] - oo[i]))
        worst = max(worst, R.ratio(host[oo[i] : oo[i + 1]], ref, bound, trunc))
    _report("many", f"{MANY} clips, {len(check)} checked", worst)
    assert worst <= 1


def test_many_clips_logmel(eng):
    """bt_logmel over 70 000 clips of 513 to 1400 samples in one launch: each clip's spectrogram bitwise what calls of
    at most 1000 clips give, and 300 of them within REF_TOL of the general kernel at the same parameters."""
    from beat_this_b200.preprocessing import LogMelSpect

    rng = np.random.default_rng(513)
    audio, so = _short_clips(rng, 513, 1400)
    before = eng.launches
    spect, fo = eng.logmel_cat(audio, so)
    assert eng.launches - before == 1
    host = spect.cpu().numpy()
    parts = _per_1000(lambda s: eng.logmel_cat(audio[s[0] : s[-1]], [v - s[0] for v in s])[0].cpu().numpy(), so)
    assert np.array_equal(np.concatenate(parts).view(np.int32), host.view(np.int32))
    general = LogMelSpect(device="cuda:0", _general=True)
    check = np.unique(np.r_[rng.choice(MANY, 150, replace=False), rng.choice(np.arange(65535, MANY), 150, replace=False)])
    want = general.batch([audio[so[i] : so[i + 1]] for i in check])
    err = max(float(np.abs(host[fo[i] : fo[i + 1]] - w.cpu().numpy()).max()) for i, w in zip(check, want))
    print(f"logmel {MANY} clips: {len(check)} within {err:.3e} of the general kernel")
    assert err <= 2e-3  # REF_TOL of test_gpu_logmel_params


def test_many_clips_audio2frames(lib_built, small0_ckpt):
    """bt_audio2frames over 70 000 short clips in one call: bitwise what calls of at most 1000 clips give."""
    from beat_this_b200.inference import Spect2Frames

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device")
    eng = Spect2Frames(small0_ckpt, "cuda:0", False).model.engine
    rng = np.random.default_rng(1400)
    audio, so = _short_clips(rng, 513, 1400)

    def run(a, s):
        fo = eng.frame_offsets(s)
        beat = torch.empty(fo[-1], device="cuda:0")
        down = torch.empty(fo[-1], device="cuda:0")
        code = eng.lib.bt_audio2frames(eng.ctx, p(a), i64(s), len(s) - 1, p(beat), p(down), i64(fo), None)
        assert code == 0, eng.lib.bt_last_error(eng.ctx)
        torch.cuda.synchronize()
        return np.concatenate([beat.cpu().numpy(), down.cpu().numpy()]).reshape(2, -1)

    whole = run(audio, so)
    parts = np.concatenate(_per_1000(lambda s: run(audio[s[0] : s[-1]], [v - s[0] for v in s]), so), axis=1)
    assert whole.shape == parts.shape and np.array_equal(whole.view(np.int32), parts.view(np.int32))
