"""CPU tests of the parameterised chunk planner (bt_plan_chunking) against the UNMODIFIED reference's split_piece and
aggregate_prediction over a sweep of piece lengths, chunk sizes, borders and both overlap modes
(tests/golden/chunking_modes.npz, oracle/make_golden_chunking_modes.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN

MODES = ("keep_first", "keep_last")


def _gold():
    return np.load(os.path.join(GOLDEN, "chunking_modes.npz"))


def _plan(lib, T, c, b, mode):
    """bt_plan_chunking -> (return code or count, starts, lens, own_lo, own_hi) as lists."""
    from beat_this_b200._lib import bt_chunking

    ck = bt_chunking(c, b, mode)
    n = lib.bt_plan_chunking(T, ctypes.byref(ck), None, None, None, None, 0)
    if n <= 0:
        return n, [], [], [], []
    arrs = [(ctypes.c_int64 * n)() for _ in range(4)]
    assert lib.bt_plan_chunking(T, ctypes.byref(ck), *arrs, n) == n
    return (n, *[list(a) for a in arrs])


def test_plan_matches_reference_and_covers_every_frame(lib_built):
    g = _gold()
    assert int(g["n"]) > 150
    for k in range(int(g["n"])):
        T, c, b, m = (int(v) for v in g[f"case{k}"])
        n, starts, lens, lo, hi = _plan(lib_built, T, c, b, m)
        assert n == len(g[f"starts{k}"]), k
        assert starts == g[f"starts{k}"].tolist() and lens == g[f"lens{k}"].tolist(), k
        owner = np.full(T, -1000, np.int32)
        for i in range(n):
            assert 0 <= lo[i] < hi[i] <= T, (k, i)  # every chunk owns something inside the piece
            assert (owner[lo[i] : hi[i]] == -1000).all(), (k, i)  # ... that no other chunk owns
            owner[lo[i] : hi[i]] = i
        assert np.array_equal(owner, g[f"owner{k}"]), (k, T, c, b, MODES[m])
        assert (owner >= 0).all(), k  # no frame is left at -1000


def test_default_chunking_is_bt_plan_chunks(lib_built):
    from beat_this_b200._lib import BT_KEEP_FIRST

    for T in [1, 2, 13, 1487, 1488, 1489, 1500, 1501, 2976, 2977, 3000, 4465, 15001, 40000]:
        n, starts, lens, lo, hi = _plan(lib_built, T, 1500, 6, BT_KEEP_FIRST)
        st, ln = (ctypes.c_int64 * n)(), (ctypes.c_int64 * n)()
        assert lib_built.bt_plan_chunks(T, st, ln, n) == n
        assert starts == list(st) and lens == list(ln), T
    assert _plan(lib_built, 0, 1500, 6, BT_KEEP_FIRST)[0] == 0


def test_python_helpers_agree_with_the_planner(lib_built):
    """chunk_starts and aggregate_prediction of beat_this_b200.inference (the per-chunk route of
    split_predict_aggregate) give the same starts and the same owner of every frame."""
    from beat_this_b200.inference import aggregate_prediction, chunk_starts, split_piece

    g = _gold()
    for k in range(int(g["n"])):
        T, c, b, m = (int(v) for v in g[f"case{k}"])
        n, starts, lens, lo, hi = _plan(lib_built, T, c, b, m)
        assert chunk_starts(T, c, b).tolist() == starts, k
        chunks, _ = split_piece(torch.zeros(T, 1), c, b)
        assert [len(ch) for ch in chunks] == lens, k
        preds = [{"beat": torch.full((len(ch),), float(i)), "downbeat": torch.zeros(len(ch))} for i, ch in enumerate(chunks)]
        owner, _ = aggregate_prediction(preds, starts, T, c, b, MODES[m], "cpu")
        assert np.array_equal(owner.numpy().astype(np.int32), g[f"owner{k}"]), k


INVALID = [(0, 0, 0), (-3, 0, 0), (1501, 0, 0), (1501, 6, 0), (64, -1, 0), (64, 32, 0), (64, 32, 1), (65, 33, 1), (1, 1, 0),
           (1500, 750, 0), (1500, 6, 2), (1500, 6, -1)]


@pytest.mark.parametrize("c,b,mode", INVALID)
def test_invalid_chunking_is_refused(lib_built, c, b, mode):
    from beat_this_b200._lib import bt_chunking
    from beat_this_b200.engine import chunking_struct

    st = (ctypes.c_int64 * 8)()
    assert lib_built.bt_plan_chunking(100, ctypes.byref(bt_chunking(c, b, mode)), st, st, st, st, 8) == -1  # BT_ERR_ARG
    with pytest.raises(ValueError):
        chunking_struct(c, b, MODES[mode] if mode in (0, 1) else "keep_middle")


def test_null_chunking_is_refused(lib_built):
    assert lib_built.bt_plan_chunking(100, None, None, None, None, None, 0) == -1


def test_limits_of_the_valid_range_are_accepted(lib_built):
    from beat_this_b200.engine import chunking_struct

    for c, b in ((1, 0), (1500, 749), (1500, 0), (3, 1)):
        for m in (0, 1):
            n, starts, lens, lo, hi = _plan(lib_built, 4507, c, b, m)
            assert n > 0 and lo[0] == 0 and hi[-1] == 4507 and all(hi[i] == lo[i + 1] for i in range(n - 1)), (c, b, m)
            ck = chunking_struct(c, b, MODES[m])
            assert (ck.chunk_size, ck.border, ck.overlap_mode) == (c, b, m)
