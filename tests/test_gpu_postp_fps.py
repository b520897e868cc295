"""GPU tests of post-processing and scoring at frame rates other than 50 (H100): the device peak picker
(bt_peakpick_fps) against the reference's outputs at 10 to 200 fps, bitwise; fps = 50 against bt_peakpick; refused
rates; the device DBN at 100 and 25 fps against the host tracker; evaluate on a checkpoint whose fps is 100."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import beat_metrics_reference as BM
import loss_reference as LR
import postp_reference as PR
from conftest import GOLDEN

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

G = np.load(os.path.join(GOLDEN, "postp_fps.npz"))
RATES = [int(f) if float(f).is_integer() else float(f) for f in G["fps"]]
DEV = "cuda:0"


@pytest.fixture(scope="module")
def eng(lib_built):
    from beat_this_b200.engine import Engine

    return Engine.mel_only(DEV)


def _cat(arrays):
    fo = np.cumsum([0] + [len(a) for a in arrays]).tolist()
    return torch.tensor(np.concatenate(arrays), device=DEV), fo


@pytest.mark.parametrize("r", range(len(RATES)))
def test_peakpick_equals_reference_at_every_rate(eng, r):
    from beat_this_b200.postprocessor import Postprocessor

    fps = RATES[r]
    post = Postprocessor("minimal", fps, engine=eng)
    n = int(G["n"])
    for k in range(n):  # one clip per call (unbatched API)
        bt, dt = post(torch.tensor(G[f"beat{k}"]), torch.tensor(G[f"down{k}"]))
        assert bt.dtype == dt.dtype == np.float64
        assert np.array_equal(bt, G[f"beat_times{r}_{k}"]) and np.array_equal(dt, G[f"down_times{r}_{k}"]), (fps, k)
    b, fo = _cat([G[f"beat{k}"] for k in range(n)])  # every clip in one launch
    d, _ = _cat([G[f"down{k}"] for k in range(n)])
    before = eng.launches
    res = post.batch_cat(b, d, fo)
    assert eng.launches == before + 1
    for k in range(n):
        assert np.array_equal(res[k][0], G[f"beat_times{r}_{k}"]) and np.array_equal(res[k][1], G[f"down_times{r}_{k}"])
    # a padded batch with its mask (large positive logits under the padding)
    bts, dts = post(torch.tensor(G["pad_beat"]), torch.tensor(G["pad_down"]), torch.tensor(G["pad_mask"]))
    assert len(bts) == len(dts) == len(G["pad_mask"])
    for i, (bt, dt) in enumerate(zip(bts, dts)):
        assert np.array_equal(bt, G[f"pad_beat_times{r}_{i}"]) and np.array_equal(dt, G[f"pad_down_times{r}_{i}"]), (fps, i)
    # the asynchronous entry point carries the rate as well
    h = eng.peakpick_async(b, d, fo, None, fps)
    out = h.result()
    assert all(np.array_equal(o[0], x[0]) and np.array_equal(o[1], x[1]) for o, x in zip(out, res))


def _raw_peakpick(eng, fn, beat, down, fo, fps=None):
    n = len(fo) - 1
    width = max([1] + [b - a for a, b in zip(fo[:-1], fo[1:])])
    times = torch.full((2, n, width), -1.0, dtype=torch.float64, device=DEV)
    cnt = torch.full((2, n), -1, dtype=torch.int32, device=DEV)
    from beat_this_b200._lib import i64_array

    head = (eng.ctx, ctypes.c_void_p(beat.data_ptr()), ctypes.c_void_p(down.data_ptr()), i64_array(fo), n)
    tail = (ctypes.c_void_p(times[0].data_ptr()), ctypes.c_void_p(cnt[0].data_ptr()), ctypes.c_void_p(times[1].data_ptr()),
            ctypes.c_void_p(cnt[1].data_ptr()), width, None)
    code = fn(*head, *tail) if fps is None else fn(*head, fps, *tail)
    torch.cuda.synchronize()
    return code, times.cpu().numpy(), cnt.cpu().numpy()


def test_fps_50_is_bt_peakpick(eng):
    """On the 50 fps fixture: bitwise the same buffers, whole buffers compared, and the same one "peakpick" launch."""
    g = np.load(os.path.join(GOLDEN, "postp_minimal.npz"))
    n = int(g["n"])
    b, fo = _cat([g[f"beat_{i}"] for i in range(n)])
    d, _ = _cat([g[f"down_{i}"] for i in range(n)])
    eng.profile_enable(True)
    eng.profile_reset()
    try:
        c0, t0, n0 = _raw_peakpick(eng, eng.lib.bt_peakpick, b, d, fo)
        c1, t1, n1 = _raw_peakpick(eng, eng.lib.bt_peakpick_fps, b, d, fo, 50.0)
        prof = eng.profile_results()
    finally:
        eng.profile_enable(False)
    assert c0 == c1 == 0
    assert np.array_equal(n0, n1) and t0.tobytes() == t1.tobytes()
    assert set(prof) == {"peakpick"} and prof["peakpick"][1] == 2
    for i in range(n):
        assert np.array_equal(t1[0, i, : n1[0, i]], g[f"beat_times_{i}"]) and np.array_equal(t1[1, i, : n1[1, i]], g[f"down_times_{i}"])
    res = eng.peakpick_cat(b, d, fo)  # the engine's default rate
    assert all(np.array_equal(res[i][0], g[f"beat_times_{i}"]) and np.array_equal(res[i][1], g[f"down_times_{i}"])
               for i in range(n))


def test_bad_fps_refused_before_any_launch(eng):
    from beat_this_b200._lib import BTError

    b, fo = _cat([G["beat4"], G["beat5"]])
    before = eng.launches
    for fps in (0.0, -0.0, -50.0, math.nan, math.inf, -math.inf):
        code, _, cnt = _raw_peakpick(eng, eng.lib.bt_peakpick_fps, b, b, fo, fps)
        assert code == -1 and (cnt == -1).all(), fps  # BT_ERR_ARG, outputs untouched
        code, _, _ = _raw_peakpick(eng, eng.lib.bt_peakpick_fps, b, b, [0], fps)  # even with no clips
        assert code == -1, fps
        with pytest.raises(BTError, match="fps"):
            eng.peakpick_cat(b, b, fo, fps)
    assert eng.launches == before


@pytest.mark.parametrize("fps", [100, 25])
def test_device_dbn_equals_host_tracker(eng, fps):
    from beat_this_b200.dbn import DBNDownBeatTracker
    from beat_this_b200.postprocessor import Postprocessor

    rng = np.random.default_rng(fps)
    # activations of beat trains at several tempi, with noise, as bt_dbn_track takes them
    acts = []
    for secs, bpm in ((30, 120), (12, 71), (45, 178), (3, 95), (20, 140)):
        T = int(secs * fps)
        t = np.arange(T) / fps
        ph = (t * bpm / 60.0) % 1.0
        beat = np.exp(-((np.minimum(ph, 1 - ph) * 60 / bpm) ** 2) / 2e-4) * 0.9
        down = beat * ((np.floor(t * bpm / 60.0) % 4) == 0)
        a = np.stack([np.clip(beat - down, 0, 1), down], 1) * rng.uniform(0.6, 1.0, (T, 1)) + rng.uniform(0, 0.05, (T, 2))
        acts.append(np.clip(a, 1e-5, 0.99) / 1.02)
    fo = np.cumsum([0] + [len(a) for a in acts]).tolist()
    cat = np.concatenate(acts)
    host = DBNDownBeatTracker(fps=fps)
    want = host.batch_cat(cat, fo)
    got = eng.dbn_cat(None, None, fo, host.track_params, activations=torch.tensor(cat, device=DEV))
    assert sum(len(w) for w in want) > 100
    for w, (bt, dt) in zip(want, got):
        assert np.array_equal(bt, w[:, 0]) and np.array_equal(dt, w[w[:, 1] == 1][:, 0])
    # padded logits through the Postprocessor: device and host decoders agree
    lens = [len(a) for a in acts]
    T = max(lens)
    logit = lambda p: np.log(p) - np.log1p(-p)  # noqa: E731
    bl = np.full((len(acts), T), 30.0, np.float32)
    dl = np.full((len(acts), T), 30.0, np.float32)
    for i, a in enumerate(acts):
        bl[i, : len(a)] = logit(np.clip(a.sum(1), 1e-4, 0.999))
        dl[i, : len(a)] = logit(a[:, 1])
    mask = torch.tensor(np.arange(T)[None, :] < np.asarray(lens)[:, None])
    dev = Postprocessor("dbn", fps, engine=eng, dbn_impl="device")(torch.tensor(bl), torch.tensor(dl), mask)
    nat = Postprocessor("dbn", fps, engine=eng, dbn_impl="native")(torch.tensor(bl), torch.tensor(dl), mask)
    assert sum(len(x) for x in nat[0]) > 100
    for i in range(len(acts)):
        assert np.array_equal(dev[0][i], nat[0][i]) and np.array_equal(dev[1][i], nat[1][i]), i


def test_device_dbn_too_large_at_200_fps(eng):
    """At 200 fps the four-beat model's state space needs more shared memory than a block has: refused, no launch."""
    from beat_this_b200._lib import BTError
    from beat_this_b200.postprocessor import Postprocessor

    post = Postprocessor("dbn", 200, engine=eng, dbn_impl="device")
    x = torch.zeros(400, device=DEV)
    before = eng.launches
    with pytest.raises(BTError, match="shared memory"):
        post.batch_cat(x, x, [0, 400])
    assert eng.launches == before


# ---- evaluate on a checkpoint at 100 fps ------------------------------------------------------------------------
SECS = (30.0, 14.0, 22.0)


def _ckpt(tmp_path, fps):
    from beat_this_b200 import synthetic

    ck = synthetic.make_checkpoint("small0", 0)
    ck["hyper_parameters"]["fps"] = fps
    path = tmp_path / f"small0_fps{fps}.ckpt"
    torch.save(ck, path)
    return str(path)


def test_evaluate_at_checkpoint_fps(tmp_path, capsys):
    from beat_this_b200 import evaluate as E
    from beat_this_b200 import synthetic
    from beat_this_b200.loss import loss_from_hparams, loss_spec
    from beat_this_b200.utils import save_beat_tsv

    fps = 100
    path = _ckpt(tmp_path, fps)
    runner = E.make_runner(path, DEV, False)
    assert runner.frames2beats.fps == 50  # the inference classes stay at 50
    clips = [synthetic.synth_clip(700 + i, s) for i, s in enumerate(SECS)]
    spects = [runner.signal2spect(x, 22050).cpu().numpy().astype(np.float16) for x in clips]
    root = tmp_path / "data"
    for i, s in enumerate(spects):
        (root / "audio" / "spectrograms" / "ds" / f"c{i}").mkdir(parents=True)
        np.save(root / "audio" / "spectrograms" / "ds" / f"c{i}" / "track.npy", s)
    ann = root / "annotations" / "ds" / "annotations" / "beats"
    ann.mkdir(parents=True)
    rng = np.random.default_rng(5)
    for i, s in enumerate(spects):
        # a beat grid running past the piece's end at 100 fps (len / 100 s) and past it at 50 fps
        beats = np.round(np.arange(0.31, len(s) / 50 + 2, rng.uniform(0.35, 0.6)), 2)
        save_beat_tsv(beats, beats[::4], ann / f"c{i}.beats")
    pieces = E.discover_data(root)
    res = E.evaluate(runner, pieces, min_beat_time=5.0, losses=True)

    logits = runner.spects2frames([p.spect for p in pieces])
    hp = runner.model.checkpoint_hparams
    est, ref = [], []
    for t in (0, 1):
        for p, (b, d), pred in zip(pieces, logits, res.predictions):
            want = PR.postp_minimal(b.cpu().numpy(), d.cpu().numpy(), fps)
            assert np.array_equal(pred[t], want[t])
            truth = p.beats if t == 0 else p.downbeats
            T = len(b)
            ref.append(truth[(truth >= 0) & (truth < T / fps)])
            est.append(want[t])
    assert any(len(r) < len(p.beats) for r, p in zip(ref, pieces))  # the 100 fps horizon cut some truth
    want = BM.beat_metrics(est, ref, min_beat_time=5.0)
    n = len(pieces)
    got = np.stack([np.concatenate([res.metrics[f"{f}_{tg}"] for tg in ("beat", "downbeat")]) for f in BM.FIELDS], 1)
    cemgil = [BM.FIELDS.index("cemgil"), BM.FIELDS.index("cemgil_max")]
    exact = [j for j in range(len(BM.FIELDS)) if j not in cemgil]
    assert np.array_equal(got[:, exact], want[:, exact])
    assert np.max(np.abs(got[:, cemgil] - want[:, cemgil])) <= 1e-12
    for t, target in enumerate(("beat", "downbeat")):
        kind, tol, pw = loss_spec(loss_from_hparams(hp)[t])
        x = [lg[t].cpu().numpy() for lg in logits]
        y = [LR.framewise_truth(p.beats if t == 0 else p.downbeats, len(xx), fps) for p, xx in zip(pieces, x)]
        off = np.cumsum([0] + [len(xx) for xx in x])
        want, _, _ = LR.loss_rows(np.concatenate(x), np.concatenate(y), None, off, kind, tol, pw)
        got = res.metrics[f"test_loss_{target}"]
        assert np.all(np.abs(got - want) <= 1e-6 * np.abs(want)), (target, got, want)
    assert len(res.metrics["test_loss"]) == n
    # the checkpoint's rate is the default; an explicit rate overrides it
    res50 = E.evaluate(runner, pieces, min_beat_time=5.0, fps=50)
    assert all(np.array_equal(a[0], b[0] * 2) for a, b in zip(res50.predictions, res.predictions))
    # the command line reads the checkpoint's rate, and --fps overrides it
    capsys.readouterr()
    E._print_single(res)
    api = capsys.readouterr().out
    assert E.main(["--models", path, "--data", str(root), "--eval-trim-beats", "5", "--no-float16", "--losses"]) == 0
    assert "\n".join(capsys.readouterr().out.splitlines()[1:]) + "\n" == api
    E._print_single(res50)
    api50 = capsys.readouterr().out
    assert E.main(["--models", path, "--data", str(root), "--eval-trim-beats", "5", "--no-float16", "--fps", "50"]) == 0
    assert "\n".join(capsys.readouterr().out.splitlines()[1:]) + "\n" == api50
