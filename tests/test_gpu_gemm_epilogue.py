"""GPU tests of the staged epilogue of the 16-bit GEMM (gemm_tc_kernel kinds 0 and 1, csrc/kernels_gemm.cu): results
go through shared-memory staging units and TMA stores, the fp32 residual arrives by TMA into the units the result then
overwrites.  Checked against the float64 references of tests/gemm_reference.py at the tolerances of
tests/numerics.py, twice each (bitwise equal), with NaN sentinel rows around the output."""
import math
import zlib

import pytest
import torch

from gemm_reference import GemmCase, _check_gemm_case, _kind1, _run_gemm, plain_shape
from support import bits, dev, small_h16  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def ring_stages(bn: int, bk: int) -> int:
    """Depth of the TMA ring (TgCfg::STAGES): what 232 448 bytes of shared memory leave beside the staging units."""
    slots = {256: 2, 192: 4}.get(bn, bn // 32 + bn // min(bn, 64))
    fit = (232448 - 1280 - slots * 128 * 128) // (128 * bk * 2 + bn * bk * 2)
    return min(6, fit)


def staged_cases():
    cs = []
    # residual aliased to the fp32 output, 16-bit copy as well (the FFN in front of a convolution), every residual tile
    for bn, N in ((128, 256), (64, 192), (32, 96)):
        for bk, K in ((64, 128), (32, 96)):
            cs.append(GemmCase(f"alias-act-{bn}x{bk}", plain_shape(3, 300, N, K), bias=True, resid=True, out_act=True,
                               resid_epilogue=True))
    # persistent CTAs over >= 3 x 132 tiles (64 planes x 3 row tiles x N / BN) whose k-block counts bracket the ring:
    # 1, STAGES - 1, STAGES + 1, 2 STAGES + 1.  The residual is requested after the first min(STAGES - 1, k-blocks).
    for bn, N, resid in ((256, 768, False), (192, 576, False), (128, 640, False), (128, 384, True), (64, 320, True),
                         (32, 160, True)):
        bks = (64, 32) if resid else (64,)
        for bk in bks:
            if bk == 32 and bn > 128:
                continue
            s = ring_stages(bn, bk)
            for nkb in sorted({1, s - 1, s + 1, 2 * s + 1}):
                cs.append(GemmCase(f"ring-{bn}x{bk}-kb{nkb}{'-resid' if resid else ''}", plain_shape(64, 300, N, bk * nkb),
                                   bias=True, gelu=not resid, resid=resid, out_act=True, resid_epilogue=resid))
    for bn, C in ((256, 512), (192, 128)):  # QKV: the 16-bit units cycle through 2 (BN = 256) or 4 (BN = 192)
        cs.append(_kind1(f"ring-qkv-{bn}", 70, 300, C))
    # ragged planes: rows >= L of every plane are clipped by the output maps (and arrive as zeros in the residual)
    for L in (1, 13, 127, 129, 1500):
        cs.append(GemmCase(f"ragged-resid-L{L}", plain_shape(5, L, 128, 64), bias=True, resid=True, out_act=True,
                           resid_epilogue=True))
        cs.append(GemmCase(f"ragged-f32-act-L{L}", plain_shape(5, L, 256, 64), bias=True, gelu=True, out_act=True))
        cs.append(_kind1(f"ragged-qkv-L{L}", 5, L, 64))
    return cs


STAGED_CASES = staged_cases()


def test_ring_depths_of_the_cases():
    """The depths this file brackets are the ones of the tile each case lands on."""
    assert {(c.tile[0], c.tile[1]) for c in STAGED_CASES} >= {(256, 64), (192, 64), (128, 64), (128, 32), (64, 64),
                                                             (64, 32), (32, 64), (32, 32)}
    assert ring_stages(256, 64) == 4 and ring_stages(128, 64) == 4 and ring_stages(128, 32) == 6


@pytest.mark.parametrize("case", STAGED_CASES, ids=lambda c: c.id)
def test_staged_epilogue(small_h16, case):
    """float64 reference, tile policy, a NaN sentinel row after the output, bitwise repeatable (two launches)."""
    _check_gemm_case(small_h16.engine, True, case)


@pytest.mark.parametrize("L", [13, 129, 1500])
def test_staged_epilogue_leaves_neighbouring_rows(small_h16, L):
    """The fp32 output (residual aliased) sits between NaN rows: a store outside the [planes * L, N] region, or a
    residual tile read across it, shows up as a changed sentinel or a NaN in the result.  The values equal those of a
    launch on an unguarded buffer bit for bit."""
    eng = small_h16.engine
    case = GemmCase(f"guard-L{L}", plain_shape(3, L, 128, 128), bias=True, resid=True, out_act=True, resid_epilogue=True)
    M, N, K = case.M, 128, 128
    g = torch.Generator(device=eng.device).manual_seed(zlib.crc32(case.id.encode()))
    a = torch.randn(M, K, generator=g, device=eng.device)
    w = torch.randn(N, K, generator=g, device=eng.device) / math.sqrt(K)
    bias = torch.randn(N, generator=g, device=eng.device)
    resid = torch.randn(M, N, generator=g, device=eng.device)
    _, want32, want_act = _run_gemm(eng, case, a, w, bias, resid, (None, None))
    guard = 3
    buf = torch.full(((M + 2 * guard) * N,), float("nan"), device=eng.device)
    o32 = buf[guard * N : (guard + M) * N]
    o32.copy_(resid.flatten())
    oa = torch.full(((M + 1) * N,), float("nan"), device=eng.device)
    eng.debug_gemm_full(case.shape, a, w, bias=bias, resid=o32, out_f32=o32, out_act=oa, resid_epilogue=True)
    assert torch.isnan(buf[: guard * N]).all() and torch.isnan(buf[(guard + M) * N :]).all(), "store outside the output"
    assert torch.equal(bits(o32), bits(want32[: M * N]))
    assert torch.equal(bits(oa), bits(want_act))
