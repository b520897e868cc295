"""CPU checks of post-processing and scoring at frame rates other than 50: the numpy restatement of the minimal
post-processor (tests/postp_reference.py) against the reference's outputs at 10 to 200 fps (tests/golden/postp_fps.npz,
oracle/make_golden_postp_fps.py), the framewise truth and horizon of beat_this_b200.evaluate against the reference's
prepare_annotations at those rates, and the argument checks of Postprocessor and evaluate."""
import math
import os
import types

import numpy as np
import pytest

import postp_reference as PR
from conftest import GOLDEN

G = np.load(os.path.join(GOLDEN, "postp_fps.npz"))
RATES = [int(f) if float(f).is_integer() else float(f) for f in G["fps"]]
ENGINE = object()  # stands in for the device context: nothing below reaches it


def test_fixture_rates():
    assert RATES == [10, 25, 22050 / 512, 86, 100, 200]


@pytest.mark.parametrize("r", range(len(RATES)))
def test_restatement_equals_reference(r):
    fps = RATES[r]
    for k in range(int(G["n"])):
        bt, dt = PR.postp_minimal(G[f"beat{k}"], G[f"down{k}"], fps)
        want_b, want_d = G[f"beat_times{r}_{k}"], G[f"down_times{r}_{k}"]
        assert bt.dtype == dt.dtype == np.float64
        assert np.array_equal(bt, want_b) and np.array_equal(dt, want_d), (fps, k)
    lens = G["pad_mask"].sum(1)
    for i, n in enumerate(lens):
        bt, dt = PR.postp_minimal(G["pad_beat"][i, :n], G["pad_down"][i, :n], fps)
        assert np.array_equal(bt, G[f"pad_beat_times{r}_{i}"]) and np.array_equal(dt, G[f"pad_down_times{r}_{i}"]), (fps, i)


def test_fixture_exercises_the_rate():
    """Every rate gives other times than 50 fps would, snapping meets argmin ties, and some clips have no peaks."""
    ties = 0
    for r, fps in enumerate(RATES):
        for k in range(int(G["n"])):
            b50, d50 = PR.postp_minimal(G[f"beat{k}"], G[f"down{k}"], 50)
            if np.any(b50 > 0):  # frame 0 is time 0 at every rate
                assert not np.array_equal(G[f"beat_times{r}_{k}"], b50)
            bt = G[f"beat_times{r}_{k}"]
            frames = PR.merge_adjacent(PR.peak_frames(G[f"down{k}"])) / fps
            for d in frames:
                dist = np.abs(bt - d)
                ties += int(len(bt) > 1 and np.sum(dist == dist.min()) > 1)
    assert ties > 0
    assert any(len(G[f"beat_times0_{k}"]) == 0 for k in range(int(G["n"])))


def test_restatement_at_50_equals_the_50_fps_fixture():
    g = np.load(os.path.join(GOLDEN, "postp_minimal.npz"))
    for i in range(int(g["n"])):
        bt, dt = PR.postp_minimal(g[f"beat_{i}"], g[f"down_{i}"], 50)
        assert np.array_equal(bt, g[f"beat_times_{i}"]) and np.array_equal(dt, g[f"down_times_{i}"]), i


@pytest.mark.parametrize("r", range(len(RATES)))
def test_truth_and_horizon_equal_prepare_annotations(r):
    import loss_reference as LR
    from beat_this_b200 import evaluate as E

    fps = RATES[r]
    for j in range(int(G["n_truth"])):
        T, times, values = int(G[f"truth_T{j}"]), G[f"truth_times{j}"], G[f"truth_values{j}"]
        for sel, key in ((np.ones(len(times), bool), "beat"), (values == 1, "down")):
            want = G[f"truth_{key}{r}_{j}"]
            assert np.array_equal(E.framewise_truth(times[sel], T, fps) == 1, want), (fps, j, key)
            assert np.array_equal(LR.framewise_truth(times[sel], T, fps) == 1, want), (fps, j, key)
            assert np.array_equal(E.horizon(times[sel], T, fps), G[f"truth_orig_{key}{r}_{j}"]), (fps, j, key)
    # the default keeps 50 fps
    times = G["truth_times0"]
    assert np.array_equal(E.framewise_truth(times, 9), E.framewise_truth(times, 9, 50))
    assert np.array_equal(E.horizon(times, 9), E.horizon(times, 9, 50))


@pytest.mark.parametrize("fps", [0, -1, -0.5, math.nan, math.inf, -math.inf, True, "50", None])
@pytest.mark.parametrize("type", ["minimal", "dbn"])
def test_postprocessor_rejects_bad_fps(type, fps):
    from beat_this_b200.postprocessor import Postprocessor

    with pytest.raises(ValueError, match="fps"):  # before any device context is made (engine=None)
        Postprocessor(type, fps=fps, dbn_impl="native")


@pytest.mark.parametrize("fps", RATES + [50, 50.0, np.float64(100.0), np.int64(25)])
def test_postprocessor_builds_at_every_rate(fps):
    from beat_this_b200.postprocessor import Postprocessor

    assert Postprocessor("minimal", fps, engine=ENGINE).fps == fps
    for impl in ("auto", "native", "device"):
        try:
            post = Postprocessor("dbn", fps, engine=ENGINE, dbn_impl=impl)
        except ImportError:  # "auto" found madmom but it failed to import
            continue
        if impl == "device":
            assert post.on_device and post.dbn_params["fps"] == float(fps)
        dbn = post.dbn
        if hasattr(dbn, "track_params"):  # the native tracker: its state space follows the rate
            lo, hi = 60.0 * fps / 215.0, 60.0 * fps / 55.0
            for m in dbn.models:
                assert m.intervals.min() == np.round(lo) and m.intervals.max() == np.round(hi)


def test_host_dbn_at_100_fps(lib_built):
    """A beat every 0.5 s, downbeat every fourth, given at 100 fps: the host tracker of Postprocessor("dbn", 100) puts
    the beats at those times (at 50 fps it would report twice the times)."""
    from beat_this_b200.postprocessor import Postprocessor

    fps, T = 100, 3000
    t = np.arange(T)
    beat = np.full(T, -6.0, np.float32)
    down = np.full(T, -6.0, np.float32)
    beat[t % 50 == 0] = 6.0
    down[t % 200 == 0] = 6.0
    post = Postprocessor("dbn", fps, engine=ENGINE, dbn_impl="native")
    (bt, dt), = post.batch_host(beat, down, [0, T])
    assert len(bt) >= 55
    assert np.abs(np.diff(bt) - 0.5).max() < 1e-9
    assert np.all(np.abs(dt / 2.0 - np.round(dt / 2.0)) < 1e-9)


def _fake_runner(hparams):
    from beat_this_b200.postprocessor import Postprocessor

    post = Postprocessor("minimal", engine=ENGINE)
    return types.SimpleNamespace(frames2beats=post, model=types.SimpleNamespace(checkpoint_hparams=hparams, engine=ENGINE))


def test_evaluate_rate_arguments():
    from beat_this_b200 import evaluate as E

    ap = E.build_parser()
    assert ap.parse_args(["--models", "m", "--data", "d"]).fps is None
    assert ap.parse_args(["--models", "m", "--data", "d", "--fps", "43.06640625"]).fps == 22050 / 512
    audio = [E.Piece("a.wav", np.zeros(0), np.zeros(0), audio="a.wav")]
    # audio files are analysed by the 50 fps front end: another rate, from the checkpoint or given, is refused
    with pytest.raises(ValueError, match="100"):
        E.evaluate(_fake_runner({"fps": 100}), audio)
    with pytest.raises(ValueError, match="25"):
        E.evaluate(_fake_runner({}), audio, fps=25)
    for bad in (0, -50, math.nan, math.inf):
        with pytest.raises(ValueError, match="fps"):
            E.evaluate(_fake_runner({}), audio, fps=bad)
        with pytest.raises(ValueError, match="fps"):
            E.evaluate(_fake_runner({"fps": bad}), audio)
