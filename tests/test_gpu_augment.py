"""GPU tests of the augmentation kernels through the C ABI (Engine.stft_cat / phase_vocoder_cat / istft_cat) and the
Python layer (augment, prepare) against the float64 restatement of tests/augment_reference.py."""
import ctypes
import os
import subprocess
import sys
import wave
from ctypes import c_void_p

import numpy as np
import pytest
import torch

import augment_reference as R
from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from beat_this_b200.engine import Engine

    return Engine.mel_only("cuda:0")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "augment.npz"))


def tables(eng, n_fft, hop):
    from beat_this_b200.augment import StftTables

    return StftTables(n_fft, hop, eng.device)


def ragged(n_clips, n_fft, seed, longest=6000):
    rng = np.random.default_rng(seed)
    lens = [n_fft // 2 + 1] + [int(v) for v in rng.integers(n_fft // 2 + 1, longest, n_clips - 1)]
    return [R.hash_signal(seed * 1000 + i, n) for i, n in enumerate(lens)]


def run_stft(eng, clips, t):
    so = np.concatenate([[0], np.cumsum([len(c) for c in clips])]).tolist()
    spec, fo = eng.stft_cat(torch.from_numpy(np.concatenate(clips)).cuda(), so, t)
    torch.cuda.synchronize()
    return spec, fo


@pytest.mark.parametrize("n_clips,n_fft,hop", [(1, 64, 16), (7, 512, 128), (7, 2048, 512), (3, 8192, 2048), (213, 512, 441),
                                               (2, 64, 1), (7, 1024, 512)])
def test_stft_within_bound_repeatable_and_batch_independent(eng, n_clips, n_fft, hop):
    clips = ragged(n_clips, n_fft, n_fft + hop, longest=max(6000, 3 * n_fft))
    t = tables(eng, n_fft, hop)
    spec, fo = run_stft(eng, clips, t)
    spec2, _ = run_stft(eng, clips, t)
    assert torch.equal(spec.view(torch.float32), spec2.view(torch.float32))
    worst = 0.0
    for i in range(0, n_clips, max(1, n_clips // 9)):
        got = spec[fo[i] : fo[i + 1]].cpu().numpy().astype(np.complex128)
        ref, bound = R.stft(clips[i], n_fft, hop), R.stft_bound(clips[i], n_fft, hop)
        assert got.shape == ref.shape
        frac = (np.abs(got - ref) / bound).max()
        worst = max(worst, frac)
        assert frac <= 1.0, (i, frac)
        alone, _ = run_stft(eng, [clips[i]], t)
        assert torch.equal(alone.view(torch.float32), spec[fo[i] : fo[i + 1]].view(torch.float32))
    print(f"stft n_fft {n_fft} hop {hop}: worst {worst:.3f} of the bound")


def random_spec(rng, frames, bins):
    return (rng.standard_normal((frames, bins)) + 1j * rng.standard_normal((frames, bins))).astype(np.complex64)


@pytest.mark.parametrize("n_clips,n_fft", [(1, 64), (7, 512), (213, 128), (3, 2048)])
def test_phase_vocoder_within_bound_repeatable_and_batch_independent(eng, n_clips, n_fft):
    rng = np.random.default_rng(n_clips + n_fft)
    bins = n_fft // 2 + 1
    Ts = [int(v) for v in rng.integers(1, 90, n_clips)]
    specs = [random_spec(rng, T, bins) for T in Ts]
    specs[0][0, :3] = 0  # angle 0 = 0
    fo = np.concatenate([[0], np.cumsum(Ts)]).tolist()
    rates = [0.25, 0.8, 0.84, 1.0, 1.2, 2 ** (5 / 12), 2 ** (-6 / 12), 4.0]
    v_clip = [c for c in range(n_clips) for _ in range(2)]
    v_rate = [rates[(2 * c + k) % len(rates)] for c in range(n_clips) for k in range(2)]
    spec = torch.from_numpy(np.concatenate(specs)).cuda()
    out, oo = eng.phase_vocoder_cat(spec, fo, v_clip, v_rate)
    out2, _ = eng.phase_vocoder_cat(spec, fo, v_clip, v_rate)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.float32), out2.view(torch.float32))
    worst = 0.0
    for v in range(0, len(v_clip), max(1, len(v_clip) // 12)):
        X = specs[v_clip[v]]
        ref, bound = R.phase_vocoder(X, v_rate[v], n_fft // 4), R.vocoder_bound(X, v_rate[v])
        got = out[oo[v] : oo[v + 1]].cpu().numpy().astype(np.complex128)
        assert got.shape == ref.shape
        frac = (np.abs(got - ref) / bound).max()
        worst = max(worst, frac)
        assert frac <= 1.0, (v, frac)
        alone, _ = eng.phase_vocoder_cat(torch.from_numpy(X).cuda(), [0, len(X)], [0], [v_rate[v]])
        assert torch.equal(alone.view(torch.float32), out[oo[v] : oo[v + 1]].view(torch.float32))
    print(f"phase_vocoder n_fft {n_fft}: worst {worst:.3f} of the bound")


def test_one_analysis_with_22_variants_equals_22_single_calls(eng):
    from beat_this_b200.augment import Augmenter

    aug = Augmenter(44100, _engine=eng)
    rates = [r for _, r, _ in aug.variants]
    assert len(rates) == 21
    rng = np.random.default_rng(5)
    spec = torch.from_numpy(random_spec(rng, 40, 1025)).cuda()
    out, oo = eng.phase_vocoder_cat(spec, [0, 40], [0] * 21, rates)
    for v, r in enumerate(rates):
        one, _ = eng.phase_vocoder_cat(spec, [0, 40], [0], [r])
        assert torch.equal(one.view(torch.float32), out[oo[v] : oo[v + 1]].view(torch.float32))


@pytest.mark.parametrize("n_seqs,n_fft,hop", [(1, 64, 16), (7, 512, 128), (7, 2048, 512), (213, 256, 100), (2, 64, 1),
                                              (3, 8192, 2048), (5, 512, 256)])
def test_istft_within_bound_repeatable_and_batch_independent(eng, n_seqs, n_fft, hop):
    rng = np.random.default_rng(n_seqs * n_fft + hop)
    bins = n_fft // 2 + 1
    Fs = [int(v) for v in rng.integers(2, 40, n_seqs)]
    specs = [random_spec(rng, F, bins) for F in Fs]
    # lengths: short, exactly the frames' span, and (where the envelope allows) past it into the zero extension
    lens = [max(1, hop * (F - 1) + (0 if k % 3 == 0 else (-hop // 2 if k % 3 == 1 else min(hop, n_fft // 4))))
            for k, F in enumerate(Fs)]
    fo = np.concatenate([[0], np.cumsum(Fs)]).tolist()
    t = tables(eng, n_fft, hop)
    spec = torch.from_numpy(np.concatenate(specs)).cuda()
    out, so = eng.istft_cat(spec, fo, lens, t)
    out2, _ = eng.istft_cat(spec, fo, lens, t)
    torch.cuda.synchronize()
    assert torch.equal(out, out2) and not torch.isnan(out).any()
    worst = 0.0
    for s in range(0, n_seqs, max(1, n_seqs // 9)):
        ref, bound = R.istft(specs[s], n_fft, hop, lens[s]), R.istft_bound(specs[s], n_fft, hop, lens[s])
        got = out[so[s] : so[s + 1]].cpu().numpy().astype(np.float64)
        frac = (np.abs(got - ref) / bound).max()
        worst = max(worst, frac)
        assert frac <= 1.0, (s, frac)
        alone, _ = eng.istft_cat(torch.from_numpy(specs[s]).cuda(), [0, Fs[s]], [lens[s]], t)
        assert torch.equal(alone, out[so[s] : so[s + 1]])
    print(f"istft n_fft {n_fft} hop {hop}: worst {worst:.3f} of the bound")


def test_istft_zero_extends_past_the_last_frame(eng):
    rng = np.random.default_rng(2)
    t = tables(eng, 64, 16)
    spec = torch.from_numpy(random_spec(rng, 5, 33)).cuda()
    out, _ = eng.istft_cat(spec, [0, 5], [16 * 4 + 32 + 50], t)
    assert torch.all(out[16 * 4 + 32 :] == 0) and torch.any(out[: 16 * 4 + 32] != 0)


def test_composed_stretch_and_shift_against_the_fixture(eng, golden):
    """The device's fp32 analysis perturbs the phases the vocoder accumulates by err / |X| per bin, which no elementwise
    bound of the output covers; the stated tolerance is 2e-3 of the clip's peak."""
    from beat_this_b200 import augment as A

    ps = int(golden["probe"][0])
    worst = 0.0
    for k, ((n_fft, hop, n), rate) in enumerate(zip(golden["configs"], golden["rates"])):
        n_fft, hop, n, rate = int(n_fft), int(hop), int(n), float(rate)
        x = R.hash_signal(int(golden["seeds"][k]), n)
        aug = A.Augmenter(44100, None, None, n_fft, hop, _engine=eng)
        y = aug.apply([x], [("v", rate, None)])[0]["v"].cpu().numpy()
        assert len(y) == int(golden["shapes"][k][1]) == R.stretched_length(n, rate)
        ref = golden[f"y{k}"]
        err = np.abs(y[::ps] - ref).max() / np.abs(ref).max()
        worst = max(worst, err / 2e-3)
        assert err <= 2e-3, (k, n_fft, hop, rate, err)
    print(f"composed stretch vs torchaudio float64: worst {worst:.3f} of the 2e-3 tolerance")


def test_ten_minute_clip_keeps_its_phase(eng):
    """50 000 frames: the accumulated phase of the last frame inside (2 j + 1) 2^-21 rad plus the sincosf term."""
    rng = np.random.default_rng(9)
    T, bins, rate = 50000, 33, 1.04
    X = random_spec(rng, T, bins)
    out, oo = eng.phase_vocoder_cat(torch.from_numpy(X).cuda(), [0, T], [0], [rate])
    got = out.cpu().numpy().astype(np.complex128)
    ref, bound = R.phase_vocoder(X, rate, 16), R.vocoder_bound(X, rate)
    frac = np.abs(got - ref) / bound
    last = np.abs(np.angle(got[-1] * np.conj(ref[-1])))
    print(f"10-minute clip: worst {frac.max():.3f} of the bound; phase error of the last frame {last.max():.2e} rad "
          f"(bound {(2 * len(ref)) * R.ATAN2F_ERR:.2e})")
    assert frac.max() <= 1.0
    assert last.max() <= 2 * len(ref) * R.ATAN2F_ERR


def test_click_train_lands_on_stretched_annotations(eng):
    from beat_this_b200 import augment as A

    sr = 44100
    beats = np.arange(1, 16) * 0.5  # 120 BPM
    x = np.zeros(8 * sr, np.float32)
    for b in beats:
        i = int(round(b * sr))
        x[i : i + 64] = np.hanning(64)
    y = A.time_stretch([x], sr, 20, device=eng.device)[0].cpu().numpy()
    assert len(y) == round(len(x) / 1.2)
    want = A.stretch_annotations({"beat_time": beats}, 20)["beat_time"]
    # A phase vocoder spreads a click over the analysis frames that hold it, so its energy lands within half a frame
    # (n_fft / 2 = 1024 samples, 23 ms) of the stretched time, not within a hop: the float64 contract itself is up to
    # 750 samples off on this signal.
    energy = y.astype(np.float64) ** 2
    for tb in want:
        c = int(round(tb * sr))
        seg = energy[c - 2048 : c + 2048]
        centroid = (seg * np.arange(len(seg))).sum() / seg.sum() + c - 2048
        assert abs(centroid - c) <= 1024, tb
    quiet = energy[int(want[3] * sr) + 4096 : int(want[4] * sr) - 4096]
    assert quiet.max() <= 1e-3 * energy.max()  # nothing between the clicks


def test_sine_shifted_an_octave_peaks_in_its_mel_band(eng):
    from beat_this_b200 import augment as A
    from beat_this_b200.preprocessing import LogMelSpect, mel_filterbank

    sr = 22050
    x = (0.5 * np.sin(2 * np.pi * 440 * np.arange(3 * sr) / sr)).astype(np.float32)
    y = A.pitch_shift([x], sr, 12, device=eng.device)[0]
    assert y.numel() == len(x)
    spect = LogMelSpect(_engine=eng).batch([y])[0].cpu().numpy()
    fb = mel_filterbank().numpy()
    band_880 = int(fb[int(round(880 * 1024 / sr))].argmax())
    mid = spect[20:-20].mean(0)
    assert abs(int(mid.argmax()) - band_880) <= 1


def test_bad_arguments_launch_nothing(eng):
    from beat_this_b200._lib import BTError, bt_stft_config, i64_array

    lib, ctx = eng.lib, eng.ctx
    t = tables(eng, 64, 16)
    audio = torch.zeros(1000, device="cuda")
    spec = torch.zeros((200, 33), dtype=torch.complex64, device="cuda")
    out = torch.zeros(4000, device="cuda")
    p = lambda x: c_void_p(x.data_ptr())  # noqa: E731
    eng.profile_enable(True)
    eng.profile_reset()
    before = eng.launches

    def stft(cfg, so, fo, a=audio, w=t.window):
        return lib.bt_stft(ctx, ctypes.byref(cfg) if cfg else None, p(w) if w is not None else None, p(t.twiddle),
                           p(a) if a is not None else None, i64_array(so), len(so) - 1, p(spec), i64_array(fo), None)

    ok = bt_stft_config(64, 16)
    assert stft(bt_stft_config(100, 16), [0, 1000], [0, 63]) == -1
    assert stft(bt_stft_config(32, 16), [0, 1000], [0, 63]) == -1
    assert stft(bt_stft_config(64, 0), [0, 1000], [0, 63]) == -1
    assert stft(ok, [0, 1000], [0, 62]) == -1
    assert stft(ok, [0, 1000], [1, 64]) == -1
    assert stft(ok, [0, 32], [0, 3]) == -1  # n_fft / 2 samples: reflect padding undefined
    assert stft(ok, [0, 1000], [0, 63], a=None) == -1
    assert stft(ok, [0, 1000], [0, 63], w=None) == -1
    assert stft(None, [0, 1000], [0, 63]) == -1

    def voc(clips, rates, oo, fo=(0, 10), n_fft=64):
        return lib.bt_phase_vocoder(ctx, n_fft, p(spec), i64_array(fo), len(fo) - 1,
                                    (ctypes.c_int32 * len(clips))(*clips), (ctypes.c_double * len(rates))(*rates),
                                    len(clips), p(out), i64_array(oo), None)

    assert voc([0], [0.2], [0, 50]) == -1
    assert voc([0], [4.5], [0, 3]) == -1
    assert voc([0], [float("nan")], [0, 10]) == -1
    assert voc([0], [float("inf")], [0, 0]) == -1
    assert voc([1], [1.0], [0, 10]) == -1
    assert voc([-1], [1.0], [0, 10]) == -1
    assert voc([0], [1.2], [0, 8]) == -1  # ceil(10 / 1.2) = 9
    assert voc([0], [1.0], [0, 10], n_fft=100) == -1
    assert voc([0], [1.0], [1, 11]) == -1

    def istft(cfg, fo, so):
        return lib.bt_istft(ctx, ctypes.byref(cfg), p(t.window), p(t.twiddle), p(spec), i64_array(fo), len(fo) - 1, p(out),
                            i64_array(so), None)

    assert istft(bt_stft_config(64, 64), [0, 10], [0, 100]) == -1  # envelope zero at every frame start
    assert istft(bt_stft_config(64, 100), [0, 10], [0, 100]) == -1
    assert istft(bt_stft_config(8192, 4096), [0, 10], [0, 4096 * 9 + 4096]) == -1  # reaches the window's last samples
    assert istft(bt_stft_config(100, 16), [0, 10], [0, 100]) == -1
    assert istft(ok, [0, 0], [0, 100]) == -1
    assert istft(ok, [1, 10], [0, 100]) == -1
    assert istft(ok, [0, 10], [100, 0]) == -1
    torch.cuda.synchronize()
    assert eng.launches == before
    assert not any(k in eng.profile_results() and eng.profile_results()[k][1] for k in ("stft", "phase_vocoder", "istft"))
    eng.profile_enable(False)
    # the Python layer raises for the same
    from beat_this_b200 import augment as A

    with pytest.raises(ValueError):
        A.time_stretch([np.zeros(5000, np.float32)], 44100, 400)
    with pytest.raises(ValueError):
        A.time_stretch([np.zeros(100, np.float32)], 44100, 20)
    with pytest.raises(NotImplementedError):
        A.time_stretch([np.zeros(5000, np.float32)], 44100, 20, n_fft=1000)
    with pytest.raises(BTError):
        eng.istft_cat(spec[:10], [0, 10], [100], tables(eng, 64, 64))


def test_launch_profile_names(eng):
    eng.profile_enable(True)
    eng.profile_reset()
    t = tables(eng, 64, 16)
    x = torch.from_numpy(R.hash_signal(1, 500)).cuda()
    spec, fo = eng.stft_cat(x, [0, 500], t)
    v, vo = eng.phase_vocoder_cat(spec, fo, [0], [1.2])
    eng.istft_cat(v, vo, [R.stretched_length(500, 1.2)], t)
    res = eng.profile_results()
    eng.profile_enable(False)
    assert {k: res[k][1] for k in ("stft", "phase_vocoder", "istft", "istft_overlap_add")} == {
        "stft": 1, "phase_vocoder": 1, "istft": 1, "istft_overlap_add": 1}


def write_wav(path, x, sr):
    pcm = np.clip(np.round(np.asarray(x) * 32767), -32768, 32767).astype("<i2")
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1 if pcm.ndim == 1 else pcm.shape[1])
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes(pcm.tobytes())


def test_prepare_end_to_end(eng, tmp_path, small0_ckpt):
    from beat_this_b200 import augment as A
    from beat_this_b200 import synthetic
    from beat_this_b200.prepare import prepare
    from beat_this_b200.preprocessing import load_audio, resample_ratio, resampled_length

    audio, ann = tmp_path / "audio", tmp_path / "ann"
    audio.mkdir()
    ann.mkdir()
    mono = synthetic.synth_clip(1, 4.0)
    stereo = np.stack([synthetic.synth_clip(2, 3.0), synthetic.synth_clip(3, 3.0)], axis=1)
    hi = np.interp(np.arange(int(3.5 * 48000)) / 48000 * 22050, np.arange(len(synthetic.synth_clip(4, 4.0))),
                   synthetic.synth_clip(4, 4.0))
    write_wav(audio / "a_mono.wav", mono, 22050)
    write_wav(audio / "b_stereo.wav", stereo, 22050)
    write_wav(audio / "c_48k.wav", hi, 48000)
    write_wav(audio / "d_unannotated.wav", mono, 22050)
    for stem in ("a_mono", "b_stereo", "c_48k"):
        (ann / f"{stem}.beats").write_text("".join(f"{0.5 * (i + 1):.3f}\t{i % 4 + 1}\n" for i in range(5)))
    out = tmp_path / "data"
    res = prepare([audio], ann, out, "toy", pitch_shift=(-1, 1), time_stretch=(4, 4), batch=2, device="cuda:0")
    assert res["written"] == ["a_mono", "b_stereo", "c_48k"] and list(res["skipped"]) == ["d_unannotated"]
    names = [f[:-4] for f in A.precomputed_augmentation_filenames(A.augmentation_dict((-1, 1), (4, 4)))]
    bundle = np.load(res["bundle"])
    assert bundle.files == [f"{s}/{n}" for s in res["written"] for n in names]
    for stem, n_in, sr in (("a_mono", len(mono), 22050), ("b_stereo", len(stereo), 22050), ("c_48k", len(hi), 48000)):
        n44 = resampled_length(n_in, *resample_ratio(sr, 44100))
        for name in names:
            spect = bundle[f"{stem}/{name}"]
            assert spect.dtype == np.float16 and spect.shape[1] == 128
            if name == "track":
                n_out = resampled_length(n_in, *resample_ratio(sr, 22050))
            else:
                n_aug = R.stretched_length(n44, 1 + int(name[8:]) / 100) if name[6:8] == "ts" else n44
                n_out = resampled_length(n_aug, *resample_ratio(44100, 22050))
            assert spect.shape[0] == 1 + n_out // 441, (stem, name)
        # track: the float16 cast of the inference front end for that file (mono mix, resample, log-mel)
        w, _ = load_audio(audio / f"{stem}.wav", dtype="float32")
        x = torch.from_numpy(np.asarray(w if w.ndim == 1 else w.mean(1), np.float32)).cuda()
        if sr != 22050:
            x, _ = eng.resample_cat(x, [0, x.numel()], sr)
        front = eng.logmel([x])[0].to(torch.float16).cpu().numpy()
        if w.ndim == 1:
            assert np.array_equal(front, bundle[f"{stem}/track"]), stem
        else:  # the native reader mixes the channels in its own order of operations
            assert np.abs(front.astype(np.float32) - bundle[f"{stem}/track"].astype(np.float32)).max() <= 1e-2, stem
    assert sorted(p.name for p in (out / "annotations" / "toy" / "annotations" / "beats").iterdir()) == [
        "a_mono.beats", "b_stereo.beats", "c_48k.beats"]
    r = subprocess.run([sys.executable, "-m", "beat_this_b200.evaluate", "--data", str(out), "--models", small0_ckpt],
                       cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
