"""bt_beat_metrics (csrc/kernels_eval.cu) against the numpy restatement of its contract (tests/beat_metrics_reference.py),
and beat_this_b200.evaluate end to end: the model's own predictions, written as annotations, score 1, and shifted
annotations score what the restatement says, for audio files and for the stored-spectrogram layout."""
import numpy as np
import pytest
import torch

import beat_metrics_reference as BM

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

CEMGIL = [BM.FIELDS.index("cemgil"), BM.FIELDS.index("cemgil_max")]
EXACT = [i for i in range(len(BM.FIELDS)) if i not in CEMGIL]


def _assert_rows(got, want):
    assert got.shape == want.shape
    bad = np.flatnonzero(np.any(got[:, EXACT] != want[:, EXACT], axis=1))
    assert bad.size == 0, f"sets {bad[:5]}: {got[bad[:1]]} vs {want[bad[:1]]}"
    assert np.max(np.abs(got[:, CEMGIL] - want[:, CEMGIL]), initial=0.0) <= 1e-12


def _edge_sets(rng, n):
    """Sets built to hit the edges of the contract."""
    est, ref = [], []
    w = 0.07
    for i in range(n):
        kind = i % 6
        if kind == 0:  # hits exactly at est - w and est + w (and one ulp outside)
            e = np.sort(rng.uniform(4, 30, rng.integers(1, 40)))
            r = np.sort(np.concatenate([e[::2] + w, e[1::2] - w, np.nextafter(e[:3] + w, np.inf)]))
        elif kind == 1:  # grid times: exact midpoints (argmin ties), duplicate refs
            step = rng.choice([0.125, 0.25, 0.5])
            r = np.sort(4 + rng.integers(0, 64, rng.integers(1, 30)) * step)
            e = np.sort(4 + rng.integers(0, 128, rng.integers(1, 30)) * step / 2 + rng.choice([0.0, 0.01]))
        elif kind == 2:  # n_ref, n_est in {0, 1, 2, 3}
            r = np.sort(rng.uniform(3, 9, rng.integers(0, 4)))
            e = np.sort(rng.uniform(3, 9, rng.integers(0, 4)))
        elif kind == 3:  # many estimates per window
            r = np.sort(rng.uniform(5, 8, rng.integers(1, 50)))
            e = np.sort(rng.uniform(5, 8, rng.integers(1, 50)))
        else:  # tracked pieces with metrical errors
            e, r = BM.tracked_piece(rng, rng.uniform(5, 60))
        est.append(e)
        ref.append(r)
    for _ in range(4):  # sets of 10 000 beats
        e, r = BM.tracked_piece(rng, 10000 * 0.4)
        est.append(e[:10000])
        ref.append(r[:10000])
    return est, ref


@pytest.mark.parametrize("min_beat_time", [5.0, 0.0])
def test_kernel_equals_restatement(lib_built, min_beat_time):
    from beat_this_b200.evaluate import beat_metrics

    est, ref = _edge_sets(np.random.default_rng(7), 2400)
    got = beat_metrics(est, ref, min_beat_time=min_beat_time, device="cuda:0")
    _assert_rows(got, BM.beat_metrics(est, ref, min_beat_time=min_beat_time))
    again = beat_metrics(est, ref, min_beat_time=min_beat_time, device="cuda:0")
    assert np.array_equal(got, again)


def test_kernel_on_pieces_and_parameters(lib_built):
    from beat_this_b200.evaluate import beat_metrics

    est, ref = BM.pieces(11, 300)
    kw = dict(min_beat_time=2.0, f_window=0.05, cemgil_sigma=0.03, phase_threshold=0.2, period_threshold=0.15)
    _assert_rows(beat_metrics(est, ref, device="cuda:0", **kw), BM.beat_metrics(est, ref, **kw))


def test_errors_before_any_launch(lib_built):
    import ctypes

    from beat_this_b200 import _lib
    from beat_this_b200.evaluate import _engine

    eng = _engine("cuda:0")
    buf = torch.zeros(16, dtype=torch.float64, device=eng.device)
    out = torch.zeros((2, 12), dtype=torch.float64, device=eng.device)
    p = _lib.bt_beat_metric_params(5.0, 0.07, 0.04, 0.175, 0.175)
    ptr = ctypes.c_void_p(buf.data_ptr())
    before = eng.launches
    for eo, ro, n in (([0, 2, 1], [0, 1, 2], 2), ([-1, 0, 1], [0, 1, 2], 2), ([0, 1, 2], [0, 1, 2], -1)):
        code = eng.lib.bt_beat_metrics(eng.ctx, ptr, _lib.i64_array(eo), ptr, _lib.i64_array(ro), n, ctypes.byref(p),
                                       ctypes.c_void_p(out.data_ptr()), None)
        assert code == -1
    p.cemgil_sigma = float("nan")
    code = eng.lib.bt_beat_metrics(eng.ctx, ptr, _lib.i64_array([0, 1, 2]), ptr, _lib.i64_array([0, 1, 2]), 2,
                                   ctypes.byref(p), ctypes.c_void_p(out.data_ptr()), None)
    assert code == -1 and eng.launches == before


# ---- end to end ----------------------------------------------------------------------------------------------------
SECS = (30.0, 14.0, 9.0, 22.0)


@pytest.fixture(scope="module")
def clips():
    from beat_this_b200 import synthetic

    return [synthetic.synth_clip(500 + i, s) for i, s in enumerate(SECS)]


def _wav_tree(root, clips):
    from scipy.io import wavfile

    (root / "wav" / "set1").mkdir(parents=True)
    paths = []
    for i, x in enumerate(clips):
        p = root / "wav" / "set1" / f"c{i}.wav"
        wavfile.write(p, 22050, np.round(x * 32767).astype(np.int16))
        paths.append(p)
    return paths


def _data_tree(root, runner, clips):
    """The prepared layout with float16 spectrograms of the clips: two as track.npy, two in an .npz bundle."""
    spects = [runner.signal2spect(x, 22050).cpu().numpy().astype(np.float16) for x in clips]
    sdir = root / "data" / "audio" / "spectrograms"
    for i in (0, 1):
        (sdir / "ds" / f"c{i}").mkdir(parents=True)
        np.save(sdir / "ds" / f"c{i}" / "track.npy", spects[i])
    np.savez(sdir / "ds.npz", **{f"c{i}/track": spects[i] for i in (2, 3)})
    (root / "data" / "annotations" / "ds" / "annotations" / "beats").mkdir(parents=True)
    return spects


def _annotate(dirpath, names, preds, shift=0.0):
    from beat_this_b200.utils import save_beat_tsv

    for name, (b, d) in zip(names, preds):
        save_beat_tsv(b + shift, d + shift, dirpath / f"{name}.beats")


def _check_self_and_shifts(E, runner, make_pieces, ann_dir, names, preds):
    for shift in (0.0, 0.03, 0.08):
        _annotate(ann_dir, names, preds, shift)
        pieces = make_pieces()
        res = E.evaluate(runner, pieces, min_beat_time=5.0)
        for p, (b, d) in zip(res.predictions, preds):
            assert np.array_equal(p[0], b) and np.array_equal(p[1], d)  # evaluate reran the same path
        if shift == 0.0:
            for t, target in enumerate(("beat", "downbeat")):
                for i, pr in enumerate(preds):
                    if np.sum(pr[t] >= 5.0) >= 2:
                        vals = [res.metrics[f"{k}_{target}"][i] for k in ("P", "R", "F", "cemgil", "CMLc", "CMLt",
                                                                          "AMLc", "AMLt", "F-measure")]
                        assert vals == [1.0] * len(vals), (target, i, vals)
                        # a variation with extra beats near the estimates can score above 1 (as in mir_eval)
                        assert res.metrics[f"cemgil_max_{target}"][i] >= 1.0
        T = [len(p.spect) if p.spect is not None else E._frames_of_audio(runner, p.audio) for p in pieces]
        est = [b for b, _ in preds] + [d for _, d in preds]
        ref = [E.horizon(p.beats, t) for p, t in zip(pieces, T)] + [E.horizon(p.downbeats, t) for p, t in zip(pieces, T)]
        want = BM.beat_metrics(est, ref, min_beat_time=5.0)
        got = np.stack([np.concatenate([res.metrics[f"{f}_{tg}"] for tg in ("beat", "downbeat")]) for f in BM.FIELDS], 1)
        _assert_rows(got, want)
    return res


@pytest.mark.parametrize("float16", [False, True])
@pytest.mark.parametrize("dbn", [False, True])
def test_evaluate_end_to_end(small0_ckpt, clips, tmp_path, capsys, float16, dbn):
    from beat_this_b200 import evaluate as E

    runner = E.make_runner(small0_ckpt, "cuda:0", float16, dbn, "device")
    # audio files
    paths = _wav_tree(tmp_path, clips)
    preds = runner.batch(paths)
    ann = tmp_path / "ann"
    ann.mkdir()
    names = [p.stem for p in paths]
    res = _check_self_and_shifts(E, runner, lambda: E.discover_audio([tmp_path / "wav"], ann), ann, names, preds)
    assert [p.dataset for p in res.pieces] == ["set1"] * len(clips)
    # stored spectrograms
    spects = _data_tree(tmp_path, runner, clips)
    out = runner.spects2frames([s.astype(np.float32) for s in spects])
    sp_preds = [runner.frames2beats(b, d) for b, d in out]
    sp_ann = tmp_path / "data" / "annotations" / "ds" / "annotations" / "beats"
    res = _check_self_and_shifts(E, runner, lambda: E.discover_data(tmp_path / "data"), sp_ann, names, sp_preds)
    # the command line prints what the API computes
    capsys.readouterr()
    E._print_single(res)
    api = capsys.readouterr().out
    flags = ["--float16" if float16 else "--no-float16", "--dbn" if dbn else "--no-dbn", "--dbn-impl", "device"]
    assert E.main(["--models", small0_ckpt, "--data", str(tmp_path / "data"), "--eval-trim-beats", "5", *flags]) == 0
    cli = capsys.readouterr().out.splitlines()
    assert cli[0] == f"Single model prediction for {small0_ckpt}" and "\n".join(cli[1:]) + "\n" == api
