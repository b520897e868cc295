"""CPU tests of the augmentation contract: the float64 restatement against the torchaudio fixture, known answers, the
reference's filename / annotation helpers, argument checks and the bundle writer."""
import json
import os
import zipfile
from pathlib import Path

import numpy as np
import pytest

import augment_reference as R
from conftest import GOLDEN

from beat_this_b200 import augment as A


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "augment.npz"))


def test_restatement_matches_torchaudio_fixture(golden):
    ps, pf, pb = (int(v) for v in golden["probe"])
    worst = 0.0
    for k, ((n_fft, hop, n), rate, seed) in enumerate(zip(golden["configs"], golden["rates"], golden["seeds"])):
        n_fft, hop, n, rate = int(n_fft), int(hop), int(n), float(rate)
        x = R.hash_signal(int(seed), n)
        Y = R.phase_vocoder(R.stft(x, n_fft, hop), rate, hop)
        y = R.istft(Y, n_fft, hop, R.stretched_length(n, rate))
        assert (len(Y), len(y)) == tuple(golden["shapes"][k])
        peak = np.abs(golden[f"y{k}"]).max()
        err = np.abs(y[::ps] - golden[f"y{k}"]).max() / peak
        # the accumulated phase is compared modulo 2 pi, through the complex value
        errY = np.abs(Y[::pf, ::pb] - golden[f"Y{k}"]).max() / np.abs(golden[f"Y{k}"]).max()
        worst = max(worst, err, errY)
        assert err <= 1e-9 and errY <= 1e-9, (k, n_fft, hop, rate, err, errY)
    print(f"restatement vs torchaudio float64: worst {worst:.2e} of the peak")


def test_rate_one_returns_the_input():
    for n_fft in (64, 512):
        hop = n_fft // 4
        x = R.hash_signal(3, 20 * n_fft + 5).astype(np.float64)
        y = R.stretch(x, 1.0, n_fft, hop)
        assert len(y) == len(x)
        inner = slice(n_fft // 2, len(x) - n_fft // 2)
        assert np.abs(y[inner] - x[inner]).max() <= 1e-12


@pytest.mark.parametrize("rate", [0.25, 0.8, 0.84, 1.2, 2 ** (5 / 12), 2 ** (-6 / 12), 4.0])
def test_stationary_tone_keeps_frequency_and_amplitude(rate):
    # A cosine at a bin centre is periodic in every frame and even about sample 0, so the reflect-padded first frames,
    # whose phases the scan starts from, are stationary too (a sine's are not: its bins start out of step and a rate
    # below 1, which reads the first pair of frames twice, keeps them so).
    n_fft, hop, k0 = 512, 128, 40
    n = 128 * 400
    x = 0.5 * np.cos(2 * np.pi * k0 * np.arange(n) / n_fft)
    y = R.stretch(x, rate, n_fft, hop)
    inner = y[2 * n_fft : len(y) - 2 * n_fft]
    m = len(inner) // n_fft * n_fft
    spec = np.abs(np.fft.rfft(inner[:m] * np.hanning(m))) / (np.hanning(m).sum() / 2)
    assert spec.argmax() == k0 * m // n_fft
    assert abs(spec.max() - 0.5) <= 1e-6
    assert abs(np.abs(inner[: m // 2]).max() - 0.5) <= 1e-6  # away from the far end, which is not a mirror point


def test_plain_fp32_running_sum_loses_the_phase_and_the_reduced_sum_does_not():
    """Emulation of the two accumulations over 50 000 frames with increments as large as pi * hop."""
    rng = np.random.default_rng(0)
    hop, n = 512, 50000
    d = (rng.uniform(-np.pi, np.pi, n) + np.pi * hop * 0.73).astype(np.float32)  # wrap(.) + omega_k of a high bin
    exact = np.cumsum(d.astype(np.float64))
    plain = np.cumsum(d, dtype=np.float32).astype(np.float64)
    reduced = np.empty(n)
    phi = 0.0
    for j in range(n):
        phi += float(d[j])
        phi -= 2 * np.pi * np.rint(phi / (2 * np.pi))
        reduced[j] = phi
    wrap = lambda e: np.abs(e - 2 * np.pi * np.rint(e / (2 * np.pi)))  # noqa: E731
    assert wrap(plain - exact).max() > 1.0  # the phase is gone
    assert wrap(reduced - exact).max() < 1e-6


def test_helpers_match_the_reference(golden):
    h = json.loads(bytes(golden["helpers"]).decode())
    for d, (npy, wav) in zip(h["dicts"], h["names"]):
        assert A.precomputed_augmentation_filenames(d) == npy
        assert A.precomputed_augmentation_filenames(d, "wav") == wav
    beats = np.array(h["beats"])
    for it in h["items"]:
        item = {"spect_path": Path("data/audio/spectrograms/ballroom/Albums-Cafe_Paradiso-05/track.npy"), "beat_time": beats}
        assert str(A.stretch_filename(item, it["amount"])["spect_path"]) == it["stretch_path"]
        assert str(A.shift_filename(item, it["amount"])["spect_path"]) == it["shift_path"]
        assert np.array_equal(A.stretch_annotations(item, it["amount"])["beat_time"], np.array(it["beat_time"]))
    assert A.augmentation_dict((-5, 6), (20, 4)) == h["dicts"][3]
    assert len(A.precomputed_augmentation_filenames(A.augmentation_dict((-5, 6), (20, 4)))) == 22


def test_rejected_arguments():
    for rate in (0.2, 4.5, float("nan"), float("inf"), -1.0):
        with pytest.raises(ValueError):
            A.check_rate(rate)
    for n_fft, hop in ((1000, 256), (32, 8), (16384, 512), (2048, 0), (2048.0, 512)):
        with pytest.raises(NotImplementedError):
            A.StftTables(n_fft, hop, "cpu")
    with pytest.raises(ValueError):  # +25 semitones: rate below 0.25
        A.check_rate(A.shift_rate(25))
    assert A.stretched_length(5, 2.0) == 2 and A.stretched_length(7, 2.0) == 4  # half to even, as Python's round
    with pytest.raises(ValueError):
        R.istft(np.ones((4, 33), np.complex128), 64, 64, 100)  # hop = n_fft: the Hann window leaves zeros


def test_bundle_writer_layout_is_read_by_discover_data(tmp_path):
    from beat_this_b200.evaluate import discover_data
    from beat_this_b200.prepare import BundleWriter, audio_files

    names = [f[:-4] for f in A.precomputed_augmentation_filenames(A.augmentation_dict((-1, 1), (4, 4)))]
    rng = np.random.default_rng(1)
    spects = {stem: {n: rng.random((10 + i, 128), dtype=np.float32) for i, n in enumerate(names)} for stem in ("b", "a")}
    bundle = tmp_path / "audio" / "spectrograms" / "toy.npz"
    with BundleWriter(bundle) as w:
        for stem in sorted(spects):
            w.add(stem, spects[stem])
    with zipfile.ZipFile(bundle) as z:
        assert [i.filename for i in z.infolist()] == [f"{s}/{n}.npy" for s in ("a", "b") for n in names]
        assert all(i.compress_type == zipfile.ZIP_STORED for i in z.infolist())
    loaded = np.load(bundle)
    for stem in spects:
        for n in names:
            assert loaded[f"{stem}/{n}"].dtype == np.float16
            assert np.array_equal(loaded[f"{stem}/{n}"], spects[stem][n].astype(np.float16))
    beats = tmp_path / "annotations" / "toy" / "annotations" / "beats"
    beats.mkdir(parents=True)
    for stem in spects:
        (beats / f"{stem}.beats").write_text("0.5\t1\n1.0\t2\n")
    pieces = discover_data(tmp_path)
    assert [p.name for p in pieces] == ["toy/a/track.npy", "toy/b/track.npy"]
    assert np.array_equal(pieces[0].spect, spects["a"]["track"].astype(np.float16).astype(np.float32))
    with pytest.raises(RuntimeError):  # a failed write leaves no bundle behind
        with BundleWriter(tmp_path / "x.npz"):
            raise RuntimeError("stop")
    assert not (tmp_path / "x.npz").exists() and not list(tmp_path.glob("x.npz.tmp*"))
    (tmp_path / "in").mkdir()
    for f in ("b.wav", "a.wav", "a.beats"):
        (tmp_path / "in" / f).write_bytes(b"")
    assert [f.name for f in audio_files([tmp_path / "in"])] == ["a.wav", "b.wav"]
