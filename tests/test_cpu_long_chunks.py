"""CPU tests of chunks longer than 1500 frames: bt_plan_chunking_max against the UNMODIFIED reference's split_piece and
aggregate_prediction (tests/golden/long_chunks.npz, oracle/make_golden_long_chunks.py), bt_plan_chunking unchanged,
the longer RoPE tables of pack_parameters, and the arguments the Python layer refuses."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN

MODES = ("keep_first", "keep_last")


def _gold():
    return np.load(os.path.join(GOLDEN, "long_chunks.npz"))


def _plan(lib, T, c, b, mode, max_chunk):
    """bt_plan_chunking_max -> (return code or count, starts, lens, own_lo, own_hi) as lists."""
    from beat_this_b200._lib import bt_chunking

    ck = bt_chunking(c, b, mode)
    n = lib.bt_plan_chunking_max(T, ctypes.byref(ck), max_chunk, None, None, None, None, 0)
    if n <= 0:
        return n, [], [], [], []
    arrs = [(ctypes.c_int64 * n)() for _ in range(4)]
    assert lib.bt_plan_chunking_max(T, ctypes.byref(ck), max_chunk, *arrs, n) == n
    return (n, *[list(a) for a in arrs])


def test_plan_matches_reference_and_covers_every_frame(lib_built):
    g = _gold()
    assert int(g["n"]) > 100
    for k in range(int(g["n"])):
        T, c, b, m = (int(v) for v in g[f"case{k}"])
        for max_chunk in (c, 8000, 384000):
            n, starts, lens, lo, hi = _plan(lib_built, T, c, b, m, max_chunk)
            assert n == len(g[f"starts{k}"]), k
            assert starts == g[f"starts{k}"].tolist() and lens == g[f"lens{k}"].tolist(), k
        owner = np.full(T, -1000, np.int32)
        for i in range(n):
            assert 0 <= lo[i] < hi[i] <= T, (k, i)
            assert (owner[lo[i] : hi[i]] == -1000).all(), (k, i)
            owner[lo[i] : hi[i]] = i
        assert np.array_equal(owner, g[f"owner{k}"]), (k, T, c, b, MODES[m])
        # one short of the chunk size is refused
        assert _plan(lib_built, T, c, b, m, c - 1)[0] == -1, k


def test_plan_chunking_keeps_its_limit(lib_built):
    """bt_plan_chunking is bt_plan_chunking_max at 1500: the same plans up to 1500 (the chunking_modes fixture), and
    BT_ERR_ARG for every longer chunk size of the long-chunk fixture."""
    from beat_this_b200._lib import bt_chunking

    g = np.load(os.path.join(GOLDEN, "chunking_modes.npz"))
    for k in range(int(g["n"])):
        T, c, b, m = (int(v) for v in g[f"case{k}"])
        ck = bt_chunking(c, b, m)
        arrs = [(ctypes.c_int64 * 64)() for _ in range(8)]
        n0 = lib_built.bt_plan_chunking(T, ctypes.byref(ck), *arrs[:4], 64)
        n1 = lib_built.bt_plan_chunking_max(T, ctypes.byref(ck), 1500, *arrs[4:], 64)
        assert n0 == n1 and all(list(x)[: min(n0, 64)] == list(y)[: min(n0, 64)] for x, y in zip(arrs[:4], arrs[4:])), k
    g = _gold()
    for k in range(int(g["n"])):
        T, c, b, m = (int(v) for v in g[f"case{k}"])
        assert lib_built.bt_plan_chunking(T, ctypes.byref(bt_chunking(c, b, m)), None, None, None, None, 0) == -1, k
    assert lib_built.bt_plan_chunking(100, ctypes.byref(bt_chunking(1501, 6, 0)), None, None, None, None, 0) == -1
    assert lib_built.bt_plan_chunking_max(100, ctypes.byref(bt_chunking(1501, 6, 0)), 1501, None, None, None, None, 0) == 1
    assert lib_built.bt_plan_chunking_max(100, None, 8000, None, None, None, None, 0) == -1
    assert lib_built.bt_plan_chunking_max(100, ctypes.byref(bt_chunking(1, 0, 0)), 0, None, None, None, None, 0) == -1


def test_whole_piece_is_one_chunk(lib_built):
    """chunk_size >= T with border 0: the piece runs as one sequence of T frames, as in the reference."""
    for T in (1, 1501, 7501, 30001):
        n, starts, lens, lo, hi = _plan(lib_built, T, 30001, 0, 0, 30001)
        assert (n, starts, lens, lo, hi) == (1, [0], [T], [0], [T]), T


def test_rope_tables_extend_the_default_bitwise():
    """pack_parameters(rope_positions=P): the first 1500 rows are today's table bit for bit, the rest rope_tables'."""
    from conftest import ckpt_path
    from beat_this_b200.weights import filter_hparams, pack_parameters, rope_tables

    ckpt = torch.load(ckpt_path("small0"), weights_only=True)
    hp = filter_hparams(ckpt["hyper_parameters"])
    sd = {k.replace("model.", ""): v for k, v in ckpt["state_dict"].items()}
    base = pack_parameters(sd, hp)
    assert base["rope.cos"].size == 1500 * 16
    freqs = [v for k, v in sd.items() if k.endswith("rotary_embed.freqs")][0]  # the buffer pack_parameters reads
    for P in (1501, 8000, 30001):
        long = pack_parameters(sd, hp, rope_positions=P)
        assert set(long) == set(base)
        for name, arr in base.items():
            if not name.startswith("rope."):
                assert np.array_equal(long[name].view(np.int32), arr.view(np.int32)), name
        cos, sin = rope_tables(freqs, P)
        for name, full in (("rope.cos", cos), ("rope.sin", sin)):
            got = long[name].reshape(P, 16)
            assert np.array_equal(got[:1500].view(np.int32), base[name].reshape(1500, 16).view(np.int32)), (name, P)
            assert np.array_equal(got.view(np.int32), full.numpy().view(np.int32)), (name, P)


@pytest.mark.parametrize("chunk", [1501, 3000, 8000])
def test_chunks_above_the_limit_raise_and_limits_give_triples(lib_built, chunk):
    """chunking_struct / engine_chunking refuse a chunk_size above the model's limit and name max_chunk_size; at the
    limit they accept it."""
    from beat_this_b200.engine import chunking_struct
    from beat_this_b200.inference import engine_chunking

    for fn in (chunking_struct, engine_chunking):
        with pytest.raises(ValueError, match="max_chunk_size"):
            fn(chunk, 6, "keep_first")
        with pytest.raises(ValueError, match="max_chunk_size"):
            fn(chunk + 1, 0, "keep_last", chunk)
    ck = chunking_struct(chunk, 6, "keep_last", chunk)
    assert (ck.chunk_size, ck.border, ck.overlap_mode) == (chunk, 6, 1)
    assert engine_chunking(chunk, 0, "keep_first", chunk) == (chunk, 0, "keep_first")
    assert engine_chunking(1500, 6, "keep_first", chunk) == (1500, 6, "keep_first")


@pytest.mark.parametrize("bad", [1499, 0, -1, 384001, 3000.0, "3000", True, None])
def test_bad_max_chunk_size_raises(bad):
    from beat_this_b200.inference import check_max_chunk_size, load_model

    with pytest.raises(ValueError, match="max_chunk_size"):
        check_max_chunk_size(bad)
    with pytest.raises(ValueError, match="max_chunk_size"):  # before the checkpoint is touched
        load_model("/nonexistent.ckpt", "cuda:0", max_chunk_size=bad)
    assert check_max_chunk_size(1500) == 1500 and check_max_chunk_size(np.int64(384000)) == 384000


def test_padded_frames_counts_the_chunks_bt_plan_chunking_max_cuts(lib_built):
    """pipeline.padded_frames: the chunks bt_plan_chunking_max cuts times chunk_size, for clips at 22.05 and 44.1 kHz."""
    from beat_this_b200.pipeline import padded_frames

    for n in (441, 661500, 22050 * 61, 22050 * 150, 22050 * 600):
        for sr in (22050, 44100):
            T = 1 + (n * 22050 // sr) // 441
            for c, b in ((3000, 6), (8000, 0), (30001, 0), (1500, 6)):
                count = _plan(lib_built, T, c, b, 0, 384000)[0]
                assert padded_frames(n, sr, c, b) == count * c, (n, sr, c, b)
