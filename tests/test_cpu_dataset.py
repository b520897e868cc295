"""beat_this_b200.dataset on the host: the split reader, item loading, oversampling and positive weights against the
unmodified reference (tests/golden/train_batches.npz, oracle/make_golden_train_batches.py), the random draws with the
numpy restatement of bt_train_batch (tests/dataset_reference.py) against every fixture item bitwise, the mask row map
against the reference's in-place operations, the refusals, and evaluate's --datasplit / k-fold selection."""
import contextlib
import io
import os

import numpy as np
import pytest

import dataset_reference as R
from conftest import GOLDEN
from dataset_reference import SEED, _dataset, _items, _tests


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "train_batches.npz"))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return R.write_tree(tmp_path_factory.mktemp("train_tree") / "data")


@pytest.mark.parametrize("name", list(R.SPLITS))
def test_split_lists_skips_and_positive_weights(tree, gold, name):
    from beat_this_b200.dataset import BeatTrackingDataset, split_items, test_items, train_val_items

    kw = R.SPLITS[name]
    train, val = train_val_items(tree, **kw)
    g = f"split/{name}/"
    assert train == gold[g + "train"].tolist()
    assert val == gold[g + "val"].tolist()
    assert test_items(tree) == gold[g + "test"].tolist()
    assert split_items(tree, "val", kw) == val and split_items(tree, "train", kw) == train
    log = io.StringIO()
    with contextlib.redirect_stdout(log):
        BeatTrackingDataset(val, tree, deterministic=True, train_length=R.TRAIN_LENGTH)
        ds = BeatTrackingDataset(train, tree, train_length=R.TRAIN_LENGTH, augmentations=R.AUGMENTATIONS)
    want = [ln for ln in str(gold[g + "log"]).splitlines() if ln.startswith("Skipping")]
    assert log.getvalue().splitlines() == want
    assert len(ds) == int(gold[g + "train_len"])
    pw = ds.positive_weights()
    assert [pw["beat"], pw["downbeat"]] == gold[g + "pos_weights"].tolist()


def test_split_ignores_other_hyper_parameters_and_the_test_set(tree):
    from beat_this_b200.dataset import split_items

    hp = {"batch_size": 8, "num_workers": 20, "augmentations": {}, "test_dataset": "gtzan", "fold": None}
    assert split_items(tree, "val", hp) == split_items(tree, "val")
    assert not any(i.startswith("gtzan/") for i in split_items(tree, "train", {"fold": 1}))
    assert split_items(tree, "test", {"test_dataset": "rwc"}) == sorted(f"rwc/{p[0]}" for p in R.DATASETS["rwc"][2])
    with pytest.raises(ValueError):
        split_items(tree, "predict")


@pytest.mark.parametrize("cfg", list(R.CONFIGS))
def test_items_and_draws_equal_the_reference(tree, gold, cfg):
    ds, log = _dataset(tree, cfg)
    assert [str(it["spect_path"]) for it in ds.items] == gold[f"{cfg}/items"].tolist()
    assert log == str(gold[f"{cfg}/log"])
    k = list(R.CONFIGS).index(cfg)
    np.random.seed(SEED + k)
    for j, i in enumerate(gold[f"{cfg}/seq"]):
        e = ds.draw(int(i))
        g = f"{cfg}/{j}/"
        L = ds.train_length if ds.train_length is not None else e.n
        spect = R.gather(e.spect[e.start : e.start + e.n], e.row_map, L)
        assert np.array_equal(spect, gold[g + "spect"]), (cfg, j)
        beat, pad = R.targets(e.beat_frames, e.n, L)
        down, _ = R.targets(e.downbeat_frames, e.n, L)
        assert np.array_equal(beat, gold[g + "truth_beat"]) and np.array_equal(down, gold[g + "truth_downbeat"])
        assert np.array_equal(pad, gold[g + "padding_mask"])
        assert e.start == int(gold[g + "start_frame"]) and e.downbeat_mask == bool(gold[g + "downbeat_mask"])
        assert e.spect_path == str(gold[g + "spect_path"]) and e.dataset == str(gold[g + "dataset"])
        assert e.truth_orig_beat == gold[g + "truth_orig_beat"].tobytes()
        assert e.truth_orig_downbeat == gold[g + "truth_orig_downbeat"].tobytes()


def test_frame_counts_and_bundle_views(tree):
    from beat_this_b200.dataset import Bundle

    ds, _ = _dataset(tree, "pt")
    for i in range(len(ds)):
        assert ds.get_frame_count(i) == len(ds._spect(ds.items[i]["spect_path"]))
        assert ds.get_beat_count(i) == len(ds.items[i]["beat_time"])
        assert ds.get_downbeat_count(i) == int((ds.items[i]["beat_value"] == 1).sum())
    b = Bundle(tree / "audio" / "spectrograms" / "rwc.npz")
    ref = np.load(tree / "audio" / "spectrograms" / "rwc.npz")
    assert sorted(b.files) == sorted(ref.files)
    for name in ref.files:
        v = b[name]
        assert b.frames(name) == len(ref[name]) and np.array_equal(v, ref[name])
        assert np.shares_memory(v, b.mmap)  # a view of the map, not a copy


def test_bundle_lists_stored_members_only(tmp_path):
    import zipfile

    from beat_this_b200.dataset import Bundle

    with zipfile.ZipFile(tmp_path / "x.npz", "w") as z:
        for name, comp in (("a/track", zipfile.ZIP_STORED), ("b/track", zipfile.ZIP_DEFLATED)):
            buf = io.BytesIO()
            np.save(buf, np.ones((3, 128), np.float16))
            z.writestr(zipfile.ZipInfo(name + ".npy"), buf.getvalue(), compress_type=comp)
    b = Bundle(tmp_path / "x.npz")
    assert b.files == ["a/track"] and "a/track" in b and "b/track" not in b
    assert b.frames("a/track") == 3


def test_row_map_equals_the_reference_mask_operations():
    from beat_this_b200.dataset import mask_row_map

    meta = np.random.RandomState(77)
    raised = 0
    for s in range(3000):
        kind = ("zero", "permute")[s % 2]
        n = int(meta.randint(1, 400))
        lo = int(meta.randint(0, 30))
        mask = {"kind": kind, "min_count": int(meta.randint(0, 3)), "max_count": int(meta.randint(3, 7)),
                "min_len": lo / 50, "max_len": (lo + int(meta.randint(0, 120))) / 50, "min_parts": int(meta.randint(1, 4)),
                "max_parts": int(meta.randint(4, 80))}
        data = meta.randint(1, 1 << 30, size=(n, 3))
        r1, r2 = np.random.RandomState(s), np.random.RandomState(s)
        try:
            want = R.apply_mask_reference(data.copy(), mask, 50, r1)
        except ValueError:
            with pytest.raises(ValueError):
                mask_row_map(n, mask, 50, r2)
            raised += 1
            continue
        m = mask_row_map(n, mask, 50, r2)
        assert m.dtype == np.int32 and m.min(initial=0) >= -1 and m.max(initial=0) < n
        got = np.where(m[:, None] >= 0, data[np.maximum(m, 0)], 0)
        assert np.array_equal(got, want), s
        assert r1.randint(1 << 30) == r2.randint(1 << 30)  # the same number of draws
    assert 0 < raised < 1500  # both outcomes were exercised


def test_errors(tree, tmp_path):
    from beat_this_b200.dataset import BeatTrackingDataset, Bundle, TrainingBatches

    with pytest.raises(ValueError, match="Unsupported augmentations"):
        BeatTrackingDataset(_items(), tree, augmentations={"noise": {}})
    with pytest.raises(ValueError, match="Unsupported mask operation"):
        BeatTrackingDataset(_items(), tree, augmentations={"mask": {**R.ZERO_MASK, "kind": "shuffle"}})
    np.savez(tmp_path / "f32.npz", **{"p/track": np.ones((5, 128), np.float32)})
    with pytest.raises(ValueError, match="float16"):
        Bundle(tmp_path / "f32.npz")["p/track"]
    # a loose float32 member
    ann = tmp_path / "d" / "annotations" / "x"
    (ann / "annotations" / "beats").mkdir(parents=True)
    (ann / "info.json").write_text('{"has_downbeats": false}')
    (ann / "annotations" / "beats" / "p.beats").write_text("0.5\n1.0\n")
    (tmp_path / "d" / "audio" / "spectrograms" / "x" / "p").mkdir(parents=True)
    np.save(tmp_path / "d" / "audio" / "spectrograms" / "x" / "p" / "track.npy", np.ones((300, 128), np.float32))
    ds = BeatTrackingDataset(["x/p"], tmp_path / "d")
    with pytest.raises(ValueError, match="float16"):
        ds.draw(0)
    full = BeatTrackingDataset(_tests(), tree, train_length=None, deterministic=True)
    with pytest.raises(ValueError, match="batch_size=1"):
        TrainingBatches(full, batch_size=2)
    # a mask as long as the excerpt: numpy's randint(0, 0) raises, as in the reference
    long_mask = {**R.ZERO_MASK, "min_count": 1, "min_len": 4.0, "max_len": 4.0}
    ds = BeatTrackingDataset(["rwc/rwc_classical_001"], tree, train_length=R.TRAIN_LENGTH,
                             augmentations={"mask": long_mask})
    with pytest.raises(ValueError):
        ds.draw(0, np.random.RandomState(0))


def test_evaluate_datasplit_arguments_and_selection(tree, capsys):
    from beat_this_b200 import evaluate as E
    from beat_this_b200.dataset import split_items

    ap = E.build_parser()
    a = ap.parse_args(["--models", "m.ckpt", "--data", "d", "--datasplit", "val", "--aggregation-type", "k-fold"])
    assert a.datasplit == "val" and a.aggregation_type == "k-fold"
    assert ap.parse_args(["--models", "m.ckpt", "--data", "d"]).datasplit is None
    with pytest.raises(SystemExit):
        ap.parse_args(["--models", "m", "--data", "d", "--datasplit", "val", "--items", "x.txt"])
    with pytest.raises(SystemExit):
        ap.parse_args(["--models", "m", "--data", "d", "--datasplit", "predict"])
    with pytest.raises(SystemExit):
        E.run(["m"], audio=["x"], annotations="y", datasplit="val")
    for hp in ({}, {"fold": 0}, {"fold": 3, "no_val": True}):
        for split in ("train", "val", "test"):
            names = split_items(tree, split, hp)
            pieces = E.split_pieces(tree, split, hp)
            skipped = [n for n in names if n == R.ONE_COLUMN]  # the only piece discover_data skips here
            assert [p.name for p in pieces] == [f"{n}/track.npy" for n in names if n not in skipped]
            assert all(p.spect.dtype == np.float32 for p in pieces)
    capsys.readouterr()
    with pytest.raises(ValueError, match="datasplit"):
        E.evaluate(None, [], data=None, datasplit="val")


def test_k_fold_concatenation_refuses_repeated_pieces():
    from beat_this_b200 import evaluate as E

    def res(names, v):
        pieces = [E.Piece(n, np.zeros(0), np.zeros(0), dataset=n.split("/")[0]) for n in names]
        m = {k: np.full(len(names), v) for k in E.SUMMARY_KEYS}
        return E.EvalResult(pieces, m, [(np.zeros(0), np.zeros(0))] * len(names), {k: v for k in E.SUMMARY_KEYS})

    r = E.concat_results([res(["a/x", "b/y"], 1.0), res(["a/z"], 0.0)])
    assert [p.name for p in r.pieces] == ["a/x", "b/y", "a/z"]
    assert r.dataset_summary()["F-measure_beat"] == {"a": 0.5, "b": 1.0}
    with pytest.raises(ValueError, match="repeated pieces"):
        E.concat_results([res(["a/x"], 1.0), res(["a/x"], 0.0)])
