"""The loss restatement (tests/loss_reference.py) against the unmodified reference's outputs (tests/golden/loss.npz,
oracle/make_golden_loss.py), the framewise truth builder of beat_this_b200.evaluate, loss_from_hparams and --losses."""
import numpy as np
import pytest

import loss_reference as R
from loss_reference import CASES, GOLD, GRAD_TOL, fixture_case


@pytest.mark.parametrize("k", CASES)
def test_restatement_matches_reference(k):
    x, y, m, off, kind, t, pw, loss, grad = fixture_case(k)
    rows, mean, g = R.loss_rows(x, y, m, off, kind, t, pw)
    assert abs(mean - loss) <= 1e-6 * abs(loss)
    assert np.max(np.abs(g - grad)) <= GRAD_TOL * np.max(np.abs(grad), initial=1e-30)
    assert np.array_equal(g != 0, grad != 0)
    assert np.isclose(np.mean(rows), mean, rtol=1e-12)  # equal-length rows: the mean of the row losses


def test_restatement_edges():
    # split and shift-tolerant agree on binary targets, differ on soft ones
    rng = np.random.default_rng(3)
    x = rng.standard_normal(60)
    y = (rng.random(60) < 0.2).astype(float)
    off = [0, 25, 60]
    a = R.loss_rows(x, y, np.ones(60), off, R.SHIFT_TOLERANT, 2, 3.0)
    b = R.loss_rows(x, y, np.ones(60), off, R.SPLIT_SHIFT_TOLERANT, 2, 3.0)
    assert np.allclose(a[0], b[0]) and np.allclose(a[2], b[2])
    ys = y * 0.9 + 0.05
    a = R.loss_rows(x, ys, np.ones(60), off, R.SHIFT_TOLERANT, 2, 3.0)
    b = R.loss_rows(x, ys, np.ones(60), off, R.SPLIT_SHIFT_TOLERANT, 2, 3.0)
    assert not np.allclose(a[1], b[1])
    with pytest.raises(ValueError):
        R.row_terms(x[:8], y[:8], None, R.SHIFT_TOLERANT, 2, 1.0)


@pytest.mark.parametrize("i", range(int(GOLD["n_truth"])))
def test_framewise_truth_matches_prepare_annotations(i):
    from beat_this_b200.evaluate import framewise_truth

    T, times, values = int(GOLD[f"truth_T{i}"]), GOLD[f"truth_times{i}"], GOLD[f"truth_values{i}"]
    beat, down = framewise_truth(times, T), framewise_truth(times[values == 1], T)
    assert beat.dtype == np.float32
    assert np.array_equal(beat.astype(bool), GOLD[f"truth_beat{i}"])
    assert np.array_equal(down.astype(bool), GOLD[f"truth_down{i}"])
    assert np.array_equal(R.framewise_truth(times, T), beat)


@pytest.mark.parametrize("loss_type,cls,pws", [
    ("shift_tolerant_weighted_bce", "ShiftTolerantBCELoss", (7.0, 40.0)),
    ("weighted_bce", "MaskedBCELoss", (7.0, 40.0)),
    ("bce", "MaskedBCELoss", (1.0, 1.0)),
    ("splitted_shift_tolerant_weighted_bce", "SplittedShiftTolerantBCELoss", (7.0, 40.0)),
])
def test_loss_from_hparams(loss_type, cls, pws):
    import torch

    from beat_this_b200 import loss as L

    beat, down = L.loss_from_hparams({"loss_type": loss_type, "pos_weights": {"beat": 7, "downbeat": 40}})
    assert type(beat).__name__ == cls and type(down).__name__ == cls
    assert (float(beat.pos_weight), float(down.pos_weight)) == pws
    assert beat.pos_weight.dtype == torch.get_default_dtype()
    if cls != "MaskedBCELoss":
        assert beat.tolerance == 3
    kind, t, pw = L.loss_spec(beat)
    assert pw == pws[0] and t == (0 if cls == "MaskedBCELoss" else 3)


def test_loss_from_hparams_defaults_and_unknown():
    from beat_this_b200 import loss as L

    beat, down = L.loss_from_hparams({})
    assert isinstance(beat, L.ShiftTolerantBCELoss) and float(down.pos_weight) == 1.0
    with pytest.raises(ValueError):
        L.loss_from_hparams({"loss_type": "focal"})


def test_split_class_quirks():
    from beat_this_b200 import loss as L

    m = L.SplittedShiftTolerantBCELoss(pos_weight=2, tolerance=1)
    assert (m.tolerance, m.spread_preds, m.spread_targets) == (3, 1, 2)
    assert L.loss_spec(m) == (L.SPLIT_SHIFT_TOLERANT, 1, 2.0)


def test_modules_refuse_cpu_tensors():
    import torch

    from beat_this_b200 import loss as L

    x = torch.zeros(2, 20)
    for m in (L.MaskedBCELoss(), L.ShiftTolerantBCELoss(), L.SplittedShiftTolerantBCELoss()):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m(x, x, torch.ones(2, 20))


def test_losses_flag():
    from beat_this_b200.evaluate import build_parser

    ap = build_parser()
    assert ap.parse_args(["--models", "m", "--data", "d", "--losses"]).losses is True
    assert ap.parse_args(["--models", "m", "--data", "d"]).losses is False
