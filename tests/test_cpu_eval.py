"""Beat-metric contract (tests/beat_metrics_reference.py) on hand-derived answers, against literal per-beat loops and
scipy's maximum matching, and against mir_eval where it is installed; the .beats reader, the data discovery and the
output formats of beat_this_b200.evaluate.  No GPU needed."""
import json
import math

import numpy as np
import pytest

import beat_metrics_reference as BM
from beat_this_b200 import evaluate as E
from beat_this_b200.utils import save_beat_tsv

COL = {f: i for i, f in enumerate(BM.FIELDS)}


def _grid(bpm=120.0, t0=0.0, t1=60.0):
    return np.arange(t0, t1, 60.0 / bpm)


def test_fields_match_the_module():
    assert E.FIELDS == BM.FIELDS


def test_identical_sets_score_one():
    r = _grid()
    row = BM.set_metrics(r, r)
    for f in ("P", "R", "F", "cemgil", "cemgil_max", "CMLc", "CMLt", "AMLc", "AMLt"):
        assert row[COL[f]] == 1.0, f


def test_30ms_shift():
    r = _grid()
    row = BM.set_metrics(r + 0.03, r)
    assert row[COL["F"]] == 1.0 and row[COL["CMLt"]] == 1.0
    assert row[COL["cemgil"]] == pytest.approx(math.exp(-0.03**2 / (2 * 0.04**2)), abs=1e-12)


def test_80ms_shift_misses_every_window():
    r = _grid()
    assert BM.set_metrics(r + 0.08, r)[COL["F"]] == 0.0


@pytest.mark.parametrize("kind", ["double", "half", "offbeat"])
def test_metrical_levels(kind):
    r = _grid()
    est = {"double": _grid(240.0, 0.0, r[-1] + 0.1), "half": r[::2], "offbeat": r[:-1] + 0.25}[kind]
    row = BM.set_metrics(est, r)
    assert row[COL["CMLt"]] == 0.0 and row[COL["AMLt"]] == 1.0


def test_empty_sets_score_zero():
    r = _grid()
    for e, ref in ((np.zeros(0), r), (r, np.zeros(0)), (np.zeros(0), np.zeros(0)), (r[r < 5], r)):
        assert not BM.set_metrics(e, ref)[2:].any()


def test_beats_before_min_beat_time_are_ignored():
    r = _grid()
    e = r.copy()
    e[r < 5.0] += 0.3  # wrong, but only before 5 s
    row = BM.set_metrics(e, r)
    assert row[COL["F"]] == 1.0 and row[COL["CMLt"]] == 1.0
    assert row[COL["n_ref"]] == np.sum(r >= 5.0)
    assert BM.set_metrics(e, r, min_beat_time=0.0)[COL["F"]] < 1.0


def test_greedy_match_is_maximum():
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import maximum_bipartite_matching

    rng = np.random.default_rng(0)
    for _ in range(300):
        ref = np.sort(rng.uniform(0, 2, rng.integers(0, 40)))
        est = np.sort(rng.uniform(0, 2, rng.integers(0, 40)))  # several estimates per 0.14 s window
        hit = (ref[None, :] >= (est - 0.07)[:, None]) & (ref[None, :] <= (est + 0.07)[:, None])
        m = maximum_bipartite_matching(csr_matrix(hit.astype(np.int8)), perm_type="column") if hit.size else np.zeros(0)
        assert BM.match_count(ref, est, 0.07) == int(np.sum(m >= 0))


def _continuity_loop(v, e, pt=0.175, qt=0.175):
    """The continuity rule written as a per-estimate loop with np.argmin (the form mir_eval uses)."""
    L = max(len(v), len(e))
    used = np.zeros(len(v), bool)
    succ = np.zeros(L)
    for m in range(len(e)):
        diff = np.abs(e[m] - v)
        k = int(np.argmin(diff))
        if used[k]:
            continue
        if m == 0 or k == 0:
            ri = v[k + 1] - v[k] if k + 1 < len(v) else v[k] - v[k - 1]
            ei = e[m + 1] - e[m] if m + 1 < len(e) else e[m] - e[m - 1]
        else:
            ri, ei = v[k] - v[k - 1], e[m] - e[m - 1]
        if ri != 0 and abs(diff[k] / ri) < pt and abs(1 - ei / ri) < qt:
            used[k] = True
            succ[m] = 1
    runs = np.diff(np.flatnonzero(np.concatenate(([0], succ, [0])) == 0)) - 1
    return runs.max() / L, succ.sum() / L


def _tie_heavy(rng):
    """Grid-quantised times: duplicates, exact midpoints (argmin ties) and one- to three-element sets."""
    n_r, n_e = rng.integers(1, 12), rng.integers(1, 12)
    step = rng.choice([0.125, 0.25, 0.5])
    r = np.sort(rng.integers(0, 16, n_r) * step)
    e = np.sort(rng.integers(0, 32, n_e) * step / 2 + rng.choice([0.0, 0.01]))
    return r, e


def test_nearest_and_continuity_equal_the_loop():
    rng = np.random.default_rng(1)
    for _ in range(2000):
        r, e = _tie_heavy(rng)
        for v in BM.variations(r):
            if len(v) == 0:
                continue
            k, d = BM.nearest(v, e)
            assert np.array_equal(k, [np.argmin(np.abs(x - v)) for x in e])
            assert np.array_equal(d, [np.min(np.abs(x - v)) for x in e])
            assert BM.continuity(v, e, 0.175, 0.175) == _continuity_loop(v, e)


def test_double_variation_is_interp():
    r = np.sort(np.random.default_rng(2).uniform(0, 100, 57))
    v = BM.variations(r)
    assert np.array_equal(v[2], np.interp(np.arange(0, len(r) - 0.5, 0.5), np.arange(len(r)), r))
    assert np.array_equal(v[1], v[2][1::2])


def test_parity_with_mir_eval():
    mir_eval = pytest.importorskip("mir_eval")
    rng = np.random.default_rng(3)
    for _ in range(200):
        r = np.cumsum(rng.uniform(0.3, 0.7, rng.integers(2, 60)))
        e = np.sort(np.abs(np.concatenate([r + rng.normal(0, 0.03, len(r)), rng.uniform(0, r[-1], rng.integers(0, 4))])))
        rt, et = mir_eval.beat.trim_beats(r, 5.0), mir_eval.beat.trim_beats(e, 5.0)
        row = BM.set_metrics(e, r)
        if len(rt) < 2 or len(et) < 2:
            continue
        assert row[COL["F"]] == mir_eval.beat.f_measure(rt, et)
        c, cmax = mir_eval.beat.cemgil(rt, et)
        assert abs(row[COL["cemgil"]] - c) < 1e-12 and abs(row[COL["cemgil_max"]] - cmax) < 1e-12
        assert tuple(row[[COL["CMLc"], COL["CMLt"], COL["AMLc"], COL["AMLt"]]]) == tuple(mir_eval.beat.continuity(rt, et))


# ---- .beats reader, horizon, discovery, formats ----------------------------------------------------------------------
def test_load_beat_annotations(tmp_path):
    beats = np.array([0.5, 1.0, 1.5, 2.0, 2.5])
    down = beats[[0, 4]]
    save_beat_tsv(beats, down, tmp_path / "two.beats")
    b, d, has = E.load_beat_annotations(tmp_path / "two.beats")
    assert has and np.array_equal(b, beats) and np.array_equal(d, down)
    (tmp_path / "one.beats").write_text("0.5\n1.0\n1.5\n")
    b, d, has = E.load_beat_annotations(tmp_path / "one.beats")
    assert not has and np.array_equal(b, [0.5, 1.0, 1.5]) and d.size == 0
    (tmp_path / "single.beats").write_text("0.5\t1\n")  # one line of two columns is one beat, not two
    b, d, has = E.load_beat_annotations(tmp_path / "single.beats")
    assert has and np.array_equal(b, [0.5]) and np.array_equal(d, [0.5])
    for bad in ("1.0\n0.5\n", "-0.5\n1.0\n", "nan\n", "0.5\t1\n1.0\n"):
        (tmp_path / "bad.beats").write_text(bad)
        with pytest.raises(ValueError):
            E.load_beat_annotations(tmp_path / "bad.beats")


def test_horizon():
    t = np.array([0.0, 1.0, 1.98, 2.0, 3.0])
    assert np.array_equal(E.horizon(t, 100), [0.0, 1.0, 1.98])  # 100 frames at 50 fps: [0, 2 s)


def test_beat_metrics_checks_input():
    with pytest.raises(ValueError):
        E.beat_metrics([np.array([1.0, 0.5])], [np.array([1.0])])
    with pytest.raises(ValueError):
        E.beat_metrics([np.array([1.0])], [])


def _write_tree(root):
    ann = root / "annotations"
    spects = root / "audio" / "spectrograms"
    rng = np.random.default_rng(0)
    # dataset "a": track.npy files, info.json with downbeats
    (ann / "a" / "annotations" / "beats").mkdir(parents=True)
    (ann / "a" / "info.json").write_text(json.dumps({"has_downbeats": True}))
    for stem in ("x", "y"):
        save_beat_tsv(np.array([1.0, 1.5, 2.0]), np.array([1.0]), ann / "a" / "annotations" / "beats" / f"{stem}.beats")
        (spects / "a" / stem).mkdir(parents=True)
        np.save(spects / "a" / stem / "track.npy", rng.normal(size=(120, 128)).astype(np.float16))
    (ann / "a" / "annotations" / "beats" / "z.beats").write_text("1.0\n2.0\n")  # one column, downbeats declared: skipped
    (spects / "a" / "z").mkdir(parents=True)
    np.save(spects / "a" / "z" / "track.npy", np.zeros((10, 128), np.float16))
    # dataset "rwc": an .npz bundle, no info.json, one-column annotations
    (ann / "rwc" / "annotations" / "beats").mkdir(parents=True)
    (ann / "rwc" / "annotations" / "beats" / "rwc_pop_001.beats").write_text("0.5\n1.0\n")
    np.savez(spects / "rwc.npz", **{"rwc_pop_001/track": np.ones((80, 128), np.float16)})


def test_discover_data(tmp_path, capsys):
    _write_tree(tmp_path)
    pieces = E.discover_data(tmp_path)
    assert [p.name for p in pieces] == ["a/x/track.npy", "a/y/track.npy", "rwc/rwc_pop_001/track.npy"]
    assert "Skipping a/z" in capsys.readouterr().out
    assert [p.dataset for p in pieces] == ["a", "a", "rwc_pop"]
    assert [p.spect.shape for p in pieces] == [(120, 128), (120, 128), (80, 128)]
    assert all(p.spect.dtype == np.float32 for p in pieces)
    assert pieces[0].has_downbeats and np.array_equal(pieces[0].downbeats, [1.0])
    assert not pieces[2].has_downbeats and pieces[2].downbeats.size == 0
    (tmp_path / "items.txt").write_text("rwc/rwc_pop_001\na/y\n")
    assert [p.name for p in E.discover_data(tmp_path, tmp_path / "items.txt")] == ["rwc/rwc_pop_001/track.npy", "a/y/track.npy"]
    (tmp_path / "annotations" / "a" / "info.json").write_text(json.dumps({"has_downbeats": False}))
    assert all(p.downbeats.size == 0 for p in E.discover_data(tmp_path, tmp_path / "items.txt"))


def _fake_result():
    pieces = [E.Piece("a/x/track.npy", np.zeros(0), np.zeros(0), dataset="a"),
              E.Piece("b/y/track.npy", np.zeros(0), np.zeros(0), dataset="b"),
              E.Piece("b/z/track.npy", np.zeros(0), np.zeros(0), dataset="b")]
    metrics = {k: np.array([0.5, 1.0, 0.0]) + i for i, k in enumerate(E.SUMMARY_KEYS)}
    preds = [(np.array([1.0, 1.5, 2.0, 2.5]), np.array([1.0, 2.5]))] * 3
    return E.EvalResult(pieces, metrics, preds, {k: float(np.mean(v)) for k, v in metrics.items()})


def test_summary_format(capsys):
    E._print_single(_fake_result())
    lines = capsys.readouterr().out.splitlines()
    assert lines[0] == "Metrics" and lines[1] == "F-measure_beat: 0.5" and lines[9] == "Dataset metrics"
    assert lines[1 : 9] == [f"{k}: {0.5 + i}" for i, k in enumerate(E.SUMMARY_KEYS)]
    assert lines[10:14] == ["F-measure_beat", "a: 0.5", "b: 0.5", "------"]
    E._print_mean_std([{"F-measure_beat": 0.8}, {"F-measure_beat": 0.9}])
    assert capsys.readouterr().out.splitlines() == ["Metrics", "F-measure_beat: 0.85 +- 0.05"]


def test_dump_predictions_format(tmp_path):
    E.write_predictions(tmp_path / "p.npz", _fake_result())
    with np.load(tmp_path / "p.npz") as z:
        assert sorted(z.files) == ["a/x/track.npy", "b/y/track.npy", "b/z/track.npy"]
        assert np.array_equal(z["a/x/track.npy"], [[1.0, 1], [1.5, 2], [2.0, 3], [2.5, 1]])


def test_cli_options():
    a = E.build_parser().parse_args(["--models", "m.ckpt", "--data", "d"])
    assert a.float16 is True and a.dbn is None and a.eval_trim_beats is None and a.dbn_impl == "auto"
    a = E.build_parser().parse_args(["--models", "m1", "m2", "--audio", "x.wav", "--annotations", "ann", "--no-float16",
                                     "--dbn", "--dbn-impl", "device", "--eval-trim-beats", "0"])
    assert a.models == ["m1", "m2"] and not a.float16 and a.dbn and a.dbn_impl == "device" and a.eval_trim_beats == 0.0
    with pytest.raises(SystemExit):
        E.build_parser().parse_args(["--models", "m", "--data", "d", "--audio", "x"])
