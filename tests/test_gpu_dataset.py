"""bt_train_batch (csrc/kernels_data.cu) and beat_this_b200.dataset.TrainingBatches on the GPU: batches bitwise equal to
the unmodified reference's items (tests/golden/train_batches.npz), the kernel against the numpy restatement
(tests/dataset_reference.py) on seeded tables with sentinel-filled outputs, repeatability, the refused tables, one batch
through the training losses, and evaluate's --datasplit and k-fold aggregation."""
import ctypes

import numpy as np
import pytest
import torch

import dataset_reference as R
import loss_reference as LR
from dataset_reference import SEED, _dataset, _items

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = "cuda:0"
BT_ERR_ARG = -1


@pytest.fixture(scope="module")
def gold():
    import os

    from conftest import GOLDEN

    return np.load(os.path.join(GOLDEN, "train_batches.npz"))


@pytest.fixture(scope="module")
def tree(tmp_path_factory, lib_built):
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device")
    return R.write_tree(tmp_path_factory.mktemp("train_tree_gpu") / "data")


@pytest.fixture(scope="module")
def engine(tree):
    from beat_this_b200.evaluate import _engine

    return _engine(DEV)


def _bits(t):
    return t.cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("cfg", list(R.CONFIGS))
def test_batches_equal_the_reference(tree, gold, cfg):
    from beat_this_b200.dataset import TrainingBatches

    ds, _ = _dataset(tree, cfg)
    seq = gold[f"{cfg}/seq"].tolist()
    np.random.seed(SEED + list(R.CONFIGS).index(cfg))
    if cfg == "full":  # full pieces: one item per batch, as the reference's test and predict loaders
        tb = TrainingBatches(ds, batch_size=1, device=DEV)
        batches = [tb.batch([i]) for i in seq]
    else:
        tb = TrainingBatches(ds, batch_size=len(seq), device=DEV)
        batches = [tb.batch(seq)]
    j = 0
    for b in batches:
        B = len(b["spect_path"])
        assert b["spect"].dtype == torch.float16 and b["spect"].device.type == "cuda"
        assert b["start_frame"].dtype == torch.int64 and b["downbeat_mask"].dtype == torch.bool
        for k in range(B):
            g = f"{cfg}/{j}/"
            assert np.array_equal(_bits(b["spect"][k]), gold[g + "spect"]), (cfg, j)
            for key in ("truth_beat", "truth_downbeat", "padding_mask"):
                assert b[key].dtype == torch.bool
                assert np.array_equal(b[key][k].cpu().numpy(), gold[g + key]), (cfg, j, key)
            assert int(b["start_frame"][k]) == int(gold[g + "start_frame"])
            assert bool(b["downbeat_mask"][k]) == bool(gold[g + "downbeat_mask"])
            assert b["spect_path"][k] == str(gold[g + "spect_path"]) and b["dataset"][k] == str(gold[g + "dataset"])
            assert b["truth_orig_beat"][k] == gold[g + "truth_orig_beat"].tobytes()
            assert b["truth_orig_downbeat"][k] == gold[g + "truth_orig_downbeat"].tobytes()
            j += 1
    assert j == len(seq)


def test_iteration_order(tree):
    """Iterating gives the batches of torch.randperm(seed) in order (drop_last), the same as batch() on those indices
    with the same draws, although each batch's successor is staged before it is handed out."""
    from beat_this_b200.dataset import TrainingBatches

    ds, _ = _dataset(tree, "all")
    tb = TrainingBatches(ds, batch_size=3, seed=11, device=DEV)
    assert len(tb) == len(ds) // 3
    order = torch.randperm(len(ds), generator=torch.Generator().manual_seed(11)).tolist()
    np.random.seed(5)
    got = [{k: (v.cpu().clone() if torch.is_tensor(v) else v) for k, v in b.items()} for b in tb]
    np.random.seed(5)
    ref = TrainingBatches(ds, batch_size=3, shuffle=False, device=DEV)
    want = [ref.batch(order[i : i + 3]) for i in range(0, 3 * len(tb), 3)]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for k in g:
            if torch.is_tensor(g[k]):
                assert torch.equal(g[k], w[k].cpu()), k
            else:
                assert g[k] == w[k], k


def _tables(rng, B, L):
    """Seeded windows and tables: window lengths from 0 to L, identity, all-zero, repeating and random maps, beats at 0
    and n - 1 and duplicates."""
    n = rng.integers(0, L + 1, B)
    n[0] = L
    if B > 2:
        n[1], n[2] = 1, 0
    rows = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    maps, beats, downs = [], [], []
    for i, ni in enumerate(n):
        kind = i % 4
        if kind == 0:
            m = np.arange(ni)
        elif kind == 1:
            m = np.full(ni, -1)
        elif kind == 2:
            m = rng.integers(0, max(ni, 1), ni) if ni else np.zeros(0)
        else:
            m = np.where(rng.random(ni) < 0.2, -1, rng.permutation(ni))
        maps.append(m.astype(np.int32))
        if ni:
            f = np.sort(np.concatenate([[0, ni - 1, ni - 1], rng.integers(0, ni, rng.integers(0, 40))]))
            d = np.sort(np.concatenate([[0], f[rng.random(len(f)) < 0.3]]))
        else:
            f = d = np.zeros(0)
        beats.append(f.astype(np.int32))
        downs.append(d.astype(np.int32))
    off = lambda a: np.concatenate([[0], np.cumsum([len(x) for x in a])]).astype(np.int64)  # noqa: E731
    return rows, np.concatenate(maps), np.concatenate(beats), off(beats), np.concatenate(downs), off(downs), n


def _launch(engine, src, rows, L, maps, beats, boff, downs, doff, sentinel=True):
    from beat_this_b200.dataset import train_batch

    B = len(rows) - 1
    spect = torch.empty((B, L, 128), dtype=torch.int16, device=DEV)
    outs = [torch.empty((B, L), dtype=torch.uint8, device=DEV) for _ in range(3)]
    if sentinel:  # any element the kernel does not write shows
        spect.fill_(0x5A5A)
        for o in outs:
            o.fill_(0xA5)
    train_batch(engine, src, rows, L, maps, beats, boff, downs, doff, spect, *outs)
    torch.cuda.synchronize()
    return spect.cpu().numpy().view(np.uint16), [o.cpu().numpy() for o in outs]


@pytest.mark.parametrize("B", [1, 7, 64, 256])
@pytest.mark.parametrize("L", [17, 1500, 3000])
def test_kernel_equals_restatement(engine, B, L):
    rng = np.random.default_rng(B * 10000 + L)
    rows, maps, beats, boff, downs, doff, n = _tables(rng, B, L)
    host = rng.integers(0, 1 << 16, (int(rows[-1]), 128), dtype=np.uint16)
    src = torch.from_numpy(host.view(np.int16).reshape(-1)).to(DEV)
    for use_map in (True, False):
        m = maps if use_map else None
        spect, (tb, td, pm) = _launch(engine, src, rows, L, m, beats, boff, downs, doff)
        for i in range(B):
            a, b = rows[i], rows[i + 1]
            want = R.gather(host[a:b], m[a:b] if use_map else None, L)
            assert np.array_equal(spect[i], want), (i, use_map)
            y, pad = R.targets(beats[boff[i] : boff[i + 1]], n[i], L)
            yd, _ = R.targets(downs[doff[i] : doff[i + 1]], n[i], L)
            assert np.array_equal(tb[i], y.astype(np.uint8)) and np.array_equal(td[i], yd.astype(np.uint8))
            assert np.array_equal(pm[i], pad.astype(np.uint8))
        again = _launch(engine, src, rows, L, m, beats, boff, downs, doff, sentinel=False)
        assert np.array_equal(again[0], spect) and all(np.array_equal(x, y) for x, y in zip(again[1], (tb, td, pm)))


def _profiled(lib, ctx):
    """Launches in the ctx's profile, over every kernel class."""
    total = 0
    for i in range(lib.bt_profile_count(ctx)):
        n = ctypes.c_int64()
        lib.bt_profile_get(ctx, i, None, 0, None, ctypes.byref(n))
        total += n.value
    return total


def test_bad_train_batch_tables_are_refused_before_any_launch(engine):
    lib, ctx = engine.lib, engine.ctx
    rng = np.random.default_rng(3)
    L = 40
    rows, maps, beats, boff, downs, doff, n = _tables(rng, 5, L)
    src = torch.zeros(int(rows[-1]) * 128 + 128, dtype=torch.int16, device=DEV)
    outs = [torch.zeros((5, L, 128), dtype=torch.int16, device=DEV)] + [torch.zeros((5, L), dtype=torch.uint8,
                                                                                    device=DEV) for _ in range(3)]
    i0 = 0  # item 0 has n = L rows

    def call(rows=rows, L=L, maps=maps, beats=beats, boff=boff, downs=downs, doff=doff):
        from beat_this_b200._lib import i32_array, i64_array

        ptr = lambda t: engine._dev_ptr(t, dtype=t.dtype)  # noqa: E731
        return lib.bt_train_batch(ctx, ptr(src), i64_array(rows), len(rows) - 1, L, i32_array(maps), i32_array(beats),
                                  i64_array(boff), i32_array(downs), i64_array(doff), *[ptr(o) for o in outs],
                                  engine._stream())

    bad_map = maps.copy()
    bad_map[rows[i0] + 3] = n[i0]  # a source row past the window
    neg_map = maps.copy()
    neg_map[rows[i0]] = -2
    bad_beat = beats.copy()
    bad_beat[boff[i0 + 1] - 1] = n[i0]  # a frame past the window
    unsorted = beats.copy()
    unsorted[boff[i0]], unsorted[boff[i0] + 1] = 5, 1
    dec = rows.copy()
    dec[2] = dec[1] - 1
    cases = {"map index >= n_i": dict(maps=bad_map), "map index < -1": dict(maps=neg_map),
             "frame out of range": dict(beats=bad_beat), "unsorted frames": dict(beats=unsorted),
             "decreasing offsets": dict(rows=dec), "n_i > length": dict(L=L - 1),
             "beat offsets not from 0": dict(boff=boff + 1), "negative downbeat frame": dict(downs=downs - 1)}
    lib.bt_profile_enable(ctx, 1)
    try:
        for name, kw in cases.items():
            torch.cuda.synchronize()
            lib.bt_profile_reset(ctx)
            before = lib.bt_launch_count(ctx)
            assert call(**kw) == BT_ERR_ARG, name
            assert b"bt_train_batch" in lib.bt_last_error(ctx), name
            assert lib.bt_launch_count(ctx) == before, name
            assert lib.bt_profile_collect(ctx) == 0 and _profiled(lib, ctx) == 0, name
        assert call() == 0  # the valid tables pass, and are profiled under the kernel's name
        assert lib.bt_profile_collect(ctx) == 0 and _profiled(lib, ctx) == 1
    finally:
        lib.bt_profile_enable(ctx, 0)


def test_batch_through_the_training_losses(tree):
    from beat_this_b200.dataset import TrainingBatches
    from beat_this_b200.loss import loss_from_hparams, loss_spec

    ds, _ = _dataset(tree, "all")
    np.random.seed(1)
    b = TrainingBatches(ds, batch_size=6, seed=0, device=DEV).batch(list(range(6)))
    assert not all(b["downbeat_mask"].tolist())  # beatles items have no downbeats
    g = torch.Generator(device=DEV).manual_seed(9)
    preds = {k: torch.randn(b["spect"].shape[:2], generator=g, device=DEV) * 3 for k in ("beat", "downbeat")}
    for hp in ({}, {"loss_type": "weighted_bce", "pos_weights": {"beat": 4, "downbeat": 9}},
               {"loss_type": "splitted_shift_tolerant_weighted_bce", "pos_weights": {"beat": 2, "downbeat": 3}}):
        beat_loss, down_loss = loss_from_hparams(hp)
        beat_mask = b["padding_mask"]  # pl_module._compute_loss (pl_module.py:99-114)
        down_mask = beat_mask * b["downbeat_mask"].to(DEV)[:, None]
        got = [float(beat_loss(preds["beat"], b["truth_beat"].float(), beat_mask)),
               float(down_loss(preds["downbeat"], b["truth_downbeat"].float(), down_mask))]
        B, L = beat_mask.shape
        off = (np.arange(B + 1) * L).tolist()
        for v, key, mask, mod in zip(got, ("beat", "downbeat"), (beat_mask, down_mask), (beat_loss, down_loss)):
            x = preds[key].cpu().numpy().reshape(-1)
            y = b[f"truth_{key}"].cpu().numpy().reshape(-1).astype(np.float32)
            m = mask.cpu().numpy().reshape(-1).astype(np.float32)
            _, want, _ = LR.loss_rows(x, y, m, off, *loss_spec(mod))
            assert abs(v - want) <= 1e-5 * abs(want) + 1e-7, (hp, key, v, want)


def _fold_ckpts(tmp_path, small0_ckpt, folds):
    paths = []
    for i, f in enumerate(folds):
        ck = torch.load(small0_ckpt, weights_only=True)
        ck["datamodule_hyper_parameters"] = {"fold": f, "batch_size": 8}
        paths.append(str(tmp_path / f"fold{i}_{f}.ckpt"))
        torch.save(ck, paths[-1])
    return paths


def test_evaluate_datasplit_and_k_fold(tree, small0_ckpt, tmp_path, capsys):
    from beat_this_b200 import evaluate as E
    from beat_this_b200.dataset import split_items

    c0, c1 = _fold_ckpts(tmp_path, small0_ckpt, (0, 1))
    # --datasplit val scores exactly the val pieces of the checkpoint's split
    dump = tmp_path / "val.npz"
    assert E.main(["--models", c0, "--data", str(tree), "--datasplit", "val", "--dump-predictions", str(dump)]) == 0
    val0 = [n for n in split_items(tree, "val", {"fold": 0}) if n != R.ONE_COLUMN]
    assert sorted(np.load(dump).files) == sorted(f"{n}/track.npy" for n in val0)
    # k-fold: each checkpoint on its own fold, per-piece metrics concatenated
    singles = [E.evaluate(c, data=tree, datasplit="val", device=DEV) for c in (c0, c1)]
    want = E.concat_results(singles)
    assert [p.name for p in want.pieces] == [p.name for r in singles for p in r.pieces]
    capsys.readouterr()
    E._print_k_fold(want)
    table = capsys.readouterr().out
    dump = tmp_path / "kfold.npz"
    assert E.run([c0, c1], data=str(tree), datasplit="val", aggregation_type="k-fold", dump_predictions=str(dump)) == 0
    out = capsys.readouterr().out.splitlines()
    assert out[0] == "Model 1/2" and "Model 2/2" in out
    start = out.index("Dataset metrics")
    assert "\n".join(out[start : start + table.count("\n")]) + "\n" == table
    assert sorted(np.load(dump).files) == sorted(p.name for p in want.pieces)
    for k in E.SUMMARY_KEYS:
        assert np.array_equal(want.metrics[k], np.concatenate([r.metrics[k] for r in singles]))
    # overlapping folds score a piece twice: refused
    a, b = _fold_ckpts(tmp_path, small0_ckpt, (0, 0))
    with pytest.raises(ValueError, match="repeated pieces"):
        E.run([a, b], data=str(tree), datasplit="val", aggregation_type="k-fold")
    assert _items()  # the tree is the fixture's
