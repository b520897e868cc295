"""GPU test (pytest -m gpu) of the fused frontend kernels' row prefetch: each warp of fused_qkv_kernel<C> and
fused_ff_kernel<C, OP> stages its next 16 rows of X by cp.async while it computes the current ones, zero-filling the
rows >= M of a partial last group.  The cases put the last group at a warp's first, second and third grid-stride step,
with 16, 15 or 1 rows, or one row past a whole grid step.  X holds NaN beyond row M (so does O; the hook hands the
kernel only O's M rows): the outputs must be bitwise those of the same call with zeros there, and no row >= M may
change."""
import zlib

import pytest
import torch

from fused_reference import FF_CTAS, FUSED_WARPS, QKV_CTAS, WARP_ROWS, random_weights
from gemm_reference import QSCALE_TIME
from support import bits, dev  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

NAN = float("nan")
TAIL = 2 * WARP_ROWS  # rows past M in every buffer


@pytest.fixture(scope="module")
def eng(lib_built, dev):
    from beat_this_b200.engine import Engine

    return Engine(None, None, dev, half=True)


def _ms(ctas, sms):
    """M at which the last 16-row group is a warp's 1st, 2nd or 3rd grid-stride step, full (0), one row short of
    full (-1), a single row (-15) or a single row of one more group (+1)."""
    wave = WARP_ROWS * FUSED_WARPS * ctas * sms  # rows of one step of the whole persistent grid
    return sorted({5, WARP_ROWS} | {k * wave + d for k in (1, 2, 3) for d in (-15, -1, 0, 1)})


def _padded(x, M, fill):
    """x [M + TAIL, n] with rows >= M set to fill."""
    y = x.clone()
    y[M:] = fill
    return y


def _cases(ctas_of, sms):
    return [(C, M) for C in (32, 64) for M in _ms(ctas_of[C], sms)]


@pytest.mark.parametrize("op", [False, True])
def test_fused_ff_prefetch_past_m(eng, dev, op):
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    for C, M in _cases(FF_CTAS, sms):
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(f"ff {C} {op} {M}".encode()))
        w = {k: v.float() for k, v in random_weights(C, g, dev).items()}
        x = torch.randn(M + TAIL, C, generator=g, device=dev)
        o = torch.randn(M + TAIL, C, generator=g, device=dev)
        runs = {}
        for fill in (NAN, 0.0):
            X, O = _padded(x, M, fill), _padded(o, M, fill)
            XB = torch.full((M + TAIL, C), 7.0, device=dev)
            X_in = X.clone()
            eng.debug_fused_ff(X, w["w1"], w["b1"], w["w2"], w["b2"], M, C, o=O if op else None,
                               wout=w["wout"] if op else None, xb_out=XB)
            assert torch.equal(bits(X[M:]), bits(X_in[M:])), f"C={C} M={M} fill={fill}: X changed past row M"
            assert (XB[M:] == 7.0).all(), f"C={C} M={M} fill={fill}: 16-bit copy written past row M"
            assert torch.isfinite(X[:M]).all(), f"C={C} M={M} fill={fill}: non-finite rows < M"
            runs[fill == 0.0] = (X[:M], XB[:M])
        assert torch.equal(bits(runs[False][0]), bits(runs[True][0])), f"C={C} M={M}: rows past M reached X"
        assert torch.equal(bits(runs[False][1]), bits(runs[True][1])), f"C={C} M={M}: rows past M reached the copy"


def test_fused_qkv_prefetch_past_m(eng, dev):
    from beat_this_b200.weights import rope_tables

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    rope = tuple(t.to(dev).contiguous() for t in rope_tables(1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))))
    for C, M in _cases(QKV_CTAS, sms):
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(f"qkv {C} {M}".encode()))
        w = {k: v.float() for k, v in random_weights(C, g, dev).items()}
        x = torch.randn(M + TAIL, C, generator=g, device=dev)
        heads = C // 32
        runs = {}
        for fill in (NAN, 0.0):
            X = _padded(x, M, fill)
            QKV = torch.full((M + TAIL, 3 * C), 7.0, device=dev)
            G = torch.full((M + TAIL, heads), 7.0, device=dev)
            eng.debug_fused_qkv(X, w["wqkv"], w["wg"], w["bg"], rope[0], rope[1], QKV, G, M, C, 1500, 1, 0, QSCALE_TIME)
            assert (QKV[M:] == 7.0).all() and (G[M:] == 7.0).all(), f"C={C} M={M} fill={fill}: store past row M"
            assert torch.isfinite(QKV[:M]).all() and torch.isfinite(G[:M]).all(), f"C={C} M={M}: non-finite rows < M"
            runs[fill == 0.0] = (QKV[:M], G[:M])
        for i, what in enumerate(("qkv", "gates")):
            assert torch.equal(bits(runs[False][i]), bits(runs[True][i])), f"C={C} M={M}: rows past M reached {what}"
