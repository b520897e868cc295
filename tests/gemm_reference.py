"""Cases and float64 references for the unit tests of the 16-bit GEMM (gemm_tc_kernel<BN, BK, KIND>) and the fp32
GEMM (gemm_simt_kernel) through bt_debug_gemm, and the check of one case on the device.  Shared by
tests/test_gpu_kernels.py and tests/test_gpu_gemm_epilogue.py (run the cases) and tests/test_cpu_gemm_sass.py (ties
GEMM_TILES to the instantiations in the built library)."""
import math
import re
import zlib
from dataclasses import dataclass, field

import torch

from numerics import (GATES_TOL, GEMM_ACC_TOL_F32, GEMM_ACC_TOL_H16, TANH_APPROX_TOL, gelu_erf, gelu_tanh, rnd,
                      rope_positions, rope_ref, ulp16)
from support import act_dtype, bits

# gemm_tc_kernel<BN, BK, KIND> in the SASS; KIND 2 (the N = 32 attention gates) keeps the IEEE-division sigmoid
GEMM_TC_KERNEL = re.compile(r"_ZN2bt14gemm_tc_kernelILi(\d+)ELi(\d+)E(?:Li(\d+)E)?E")
# every (BN, BK, KIND) instantiation of gemm_tc_kernel in the library; the GPU matrix runs each at least once
GEMM_TILES = sorted(
    [(bn, 64, k) for k in (0, 1) for bn in (256, 192, 128, 64, 32)]
    + [(bn, 32, k) for k in (0, 1) for bn in (128, 64, 32)]
    + [(32, 64, 2), (32, 32, 2)]
)


def stages(bn: int) -> int:
    """Depth of the TMA ring of a BN-wide tile (TgCfg::STAGES, kernels_gemm.cu)."""
    return {256: 4, 192: 5}.get(bn, 6)


def expected_tile(N: int, Kslab: int, resid_epilogue: bool):
    """The tile policy of tc_gemm_plan_create: BK = 64 when it divides Kslab, else 32; then the widest BN that
    divides N, at most 128 for BK = 32 tiles and for GEMMs whose epilogue adds the fp32 residual."""
    bk = 64 if Kslab % 64 == 0 else 32
    cap = 128 if bk == 32 or resid_epilogue else 256
    return next(bn for bn in (256, 192, 128, 64, 32) if bn <= cap and N % bn == 0), bk


# ---- the GemmShape values bt_api.cu builds (plain_shape, conv_shape, lin_shape)
def plain_shape(planes, L, N, K):
    return dict(form="plain", planes_out=planes, planes_in=planes, L=L, N=N, Kslab=K, nslab=1, plane_mul=1, lda=K,
                plane_add=[0], t_shift=[0])


def conv_shape(nb, F, L, C):
    """Conv2d(C -> 2C, k(2, 3), stride (2, 1), padding (0, 1)) over [nb, F, L, C]: slab df * 3 + dt."""
    return dict(form="conv", planes_out=nb * F // 2, planes_in=nb * F, L=L, N=2 * C, Kslab=C, nslab=6, plane_mul=2,
                lda=C, plane_add=[df for df in range(2) for dt in range(3)],
                t_shift=[dt - 1 for df in range(2) for dt in range(3)], nb=nb)


def lin_shape(nb, L, D, Fo, Co):
    """frontend.linear over "b c f t -> b t (c f)": slab f reads plane Fo * b + f."""
    return dict(form="lin", planes_out=nb, planes_in=nb * Fo, L=L, N=D, Kslab=Co, nslab=Fo, plane_mul=Fo, lda=Co,
                plane_add=list(range(Fo)), t_shift=[0] * Fo, nb=nb)


QSCALE_TIME = math.log2(math.e) / math.sqrt(32)  # the time attentions' q scale (softmax in log2 units)


@dataclass
class GemmCase:
    id: str
    shape: dict
    kind: int = 0
    bias: bool = False
    gelu: bool = False
    resid: bool = False  # residual aliased to out_f32, as ff_block / attention_block run it
    out_f32: bool = True
    out_act: bool = False
    resid_epilogue: bool = False
    C: int = 0
    heads: int = 0
    posmode: int = 0
    F: int = 1
    qscale: float = 1.0
    extra: dict = field(default_factory=dict)

    @property
    def tile(self):
        return expected_tile(self.shape["N"], self.shape["Kslab"], self.resid_epilogue)

    @property
    def M(self):
        return self.shape["planes_out"] * self.shape["L"]


def _kind1(id, planes, L, C, Kslab=None, posmode=0, F=1, qscale=QSCALE_TIME, resid_epilogue=False):
    return GemmCase(id, plain_shape(planes, L, 3 * C, Kslab or C), kind=1, out_f32=False, out_act=True, C=C,
                    heads=C // 32, posmode=posmode, F=F, qscale=qscale, resid_epilogue=resid_epilogue)


def _gates(id, planes, L, K, heads):
    return GemmCase(id, plain_shape(planes, L, 32, K), kind=2, bias=True, heads=heads)


def gemm_cases():
    cs = []
    # one case per instantiation (the tile each lands on is asserted against expected_tile)
    cs += [
        GemmCase("inst-k0-256x64", plain_shape(2, 300, 512, 64), bias=True, gelu=True, out_f32=False, out_act=True),
        GemmCase("inst-k0-192x64", plain_shape(2, 200, 384, 128)),
        GemmCase("inst-k0-128x64", plain_shape(2, 300, 512, 128), bias=True, resid=True, out_act=True, resid_epilogue=True),
        GemmCase("inst-k0-64x64", plain_shape(3, 129, 64, 64), out_act=True),
        GemmCase("inst-k0-32x64", plain_shape(3, 129, 32, 128), bias=True),
        GemmCase("inst-k0-128x32", plain_shape(2, 257, 256, 96), out_act=True),
        GemmCase("inst-k0-64x32", plain_shape(2, 100, 64, 32), bias=True, gelu=True),
        GemmCase("inst-k0-32x32", plain_shape(2, 100, 96, 96), resid=True, resid_epilogue=True),
        _kind1("inst-k1-256x64", 2, 300, 512),
        _kind1("inst-k1-192x64", 3, 300, 128),
        _kind1("inst-k1-128x64", 2, 200, 128, resid_epilogue=True),
        _kind1("inst-k1-64x64", 2, 200, 64, resid_epilogue=True),
        _kind1("inst-k1-32x64", 2, 200, 32, Kslab=64),
        _kind1("inst-k1-128x32", 2, 200, 128, Kslab=96),
        _kind1("inst-k1-64x32", 2, 200, 64, Kslab=96),
        _kind1("inst-k1-32x32", 2, 200, 32),
        _gates("inst-k2-32x64", 3, 257, 128, 4),
        _gates("inst-k2-32x32", 3, 257, 32, 1),
    ]
    # persistent CTAs over >= 3 x 132 tiles (64 planes x 3 row tiles x N / BN), num_kb = 1, STAGES - 1, STAGES + 1 and
    # one that is not a multiple of STAGES, so the ring phase flips at different points inside and between tiles
    for bn, N in ((256, 1536), (192, 1344), (128, 640), (64, 320), (32, 160)):
        s = stages(bn)
        for nkb in sorted({1, s - 1, s + 1, 2 * s + 1}):
            cs.append(GemmCase(f"persist-{bn}x64-kb{nkb}", plain_shape(64, 300, N, 64 * nkb), bias=True,
                               gelu=bn == 256, out_act=nkb == 1))
    for bn, N in ((128, 640), (64, 320), (32, 160)):
        for nkb in (stages(bn) - 1, 2 * stages(bn) + 1):
            cs.append(GemmCase(f"persist-{bn}x32-kb{nkb}", plain_shape(64, 300, N, 32 * nkb), resid=True,
                               resid_epilogue=True, out_act=True))
    # ragged rows: every row guard and the plane boundaries inside a tile
    i = 0
    for L in (1, 13, 127, 128, 129, 1500):
        for planes in (1, 3, 40):
            N = (192, 64, 96)[i % 3]
            cs.append(GemmCase(f"rows-L{L}-p{planes}-N{N}", plain_shape(planes, L, N, 64), bias=True, gelu=True,
                               out_act=True))
            i += 1
    # the three frontend convolutions (slab GEMMs with time shifts -1 / +1 and plane_mul 2) and frontend.linear
    for C, F in ((32, 32), (64, 16), (128, 8)):
        for L in (13, 129, 1500):
            last = C == 128  # conv 2 feeds frontend.linear in the activation dtype
            cs.append(GemmCase(f"conv-C{C}-L{L}", conv_shape(2, F, L, C), bias=True, gelu=True, out_f32=not last,
                               out_act=last))
    for L in (129, 1500):
        cs.append(GemmCase(f"lin-L{L}", lin_shape(2, L, 512, 4, 256), bias=True))
    # the epilogues of the main layers (D = 512, ff_mult 4)
    cs += [
        GemmCase("ffn-up", plain_shape(4, 1500, 2048, 512), bias=True, gelu=True, out_f32=False, out_act=True),
        GemmCase("ffn-down", plain_shape(4, 1500, 512, 2048), bias=True, resid=True, out_act=True, resid_epilogue=True),
        GemmCase("attn-out", plain_shape(4, 1500, 512, 512), resid=True, resid_epilogue=True),
    ]
    # RoPE / q-scale epilogue: time positions over all 1500 table rows, frequency positions p_out % F
    cs += [_kind1(f"qkv-time-C{C}", planes, 1500, C) for C, planes in ((32, 2), (64, 2), (128, 2), (512, 8))]
    cs += [_kind1(f"qkv-freq-F{F}", 2 * F, 129, C, posmode=1, F=F, qscale=1.0) for F, C in ((32, 32), (16, 64), (8, 128))]
    # attention gates: heads of the padded 32-row weight, BK 32 and 64
    for heads in (1, 2, 4, 16):
        cs.append(_gates(f"gates-h{heads}-bk64", 3, 257, 128 if heads < 16 else 512, heads))
        cs.append(_gates(f"gates-h{heads}-bk32", 3, 257, 96, heads))
    return cs


GEMM_CASES = gemm_cases()


# ---- float64 references, from the definition of each operation (not from the kernel's layout)
def gemm_ref(shape, a, w):
    """acc [M, N] of the GEMM on operands a [planes_in * L, lda], w [N, nslab * Kslab] (any float dtype)."""
    L, N, C = shape["L"], shape["N"], shape["Kslab"]
    if shape["form"] == "plain":
        return a @ w.T
    nb = shape["nb"]
    if shape["form"] == "conv":  # [nb, F, L, C] planes -> conv2d over [nb, C, F, L]; weight slab order (df, dt, c)
        F = shape["planes_in"] // nb
        x = a.view(nb, F, L, C).permute(0, 3, 1, 2)
        wt = w.view(N, 2, 3, C).permute(0, 3, 1, 2)  # [2C, C, 2, 3]
        y = torch.nn.functional.conv2d(x, wt, stride=(2, 1), padding=(0, 1))  # [nb, 2C, F / 2, L]
        return y.permute(0, 2, 3, 1).reshape(-1, N)
    Fo = shape["nslab"]  # frontend.linear: b c f t -> b t (c f), weight columns (f, c) back to (c f)
    x = a.view(nb, Fo, L, C).permute(0, 3, 1, 2)  # b c f t
    x = x.permute(0, 3, 1, 2).reshape(nb, L, C * Fo)
    wref = w.view(N, Fo, C).permute(0, 2, 1).reshape(N, C * Fo)
    return (x @ wref.T).reshape(nb * L, N)


def epilogue_ref(case, acc, bias, resid, half, rope_cos=None, rope_sin=None):
    """(out [M, ldo], pre-GELU value or None) in float64 for the case's epilogue on acc [M, N]."""
    if case.kind == 2:
        return torch.sigmoid(acc[:, : case.heads] + bias[: case.heads]), None
    if case.kind == 1:
        L, C = case.shape["L"], case.C
        pos = rope_positions(acc.shape[0], L, case.F, case.posmode, acc.device)
        out = acc.clone()
        out[:, :C] = rope_ref(acc[:, :C], rope_cos[pos], rope_sin[pos]) * case.qscale
        out[:, C : 2 * C] = rope_ref(acc[:, C : 2 * C], rope_cos[pos], rope_sin[pos])
        return out, None
    y = acc + bias if case.bias else acc
    pre = None
    if case.gelu:
        pre = y
        y = gelu_tanh(y) if half else gelu_erf(y)
    if case.resid:
        y = y + resid
    return y, pre


# ---- one case on the device: bt_debug_gemm against the float64 references above, at the tolerances of numerics.py
def _run_gemm(eng, case, a, w, bias, resid, rope):
    """One bt_debug_gemm call on fresh output buffers of M + 1 rows: the last row is a NaN sentinel, and every other
    element starts as NaN too (or as the residual where out_f32 doubles as it), so a missing store shows up."""
    M, N = case.M, case.shape["N"]
    ldo = case.heads if case.kind == 2 else N
    nan = float("nan")
    o32 = torch.full(((M + 1) * ldo,), nan, device=a.device) if case.out_f32 else None
    if case.resid:
        o32[: M * N] = resid.flatten()
    oa = torch.full(((M + 1) * N,), nan, device=a.device) if case.out_act else None
    tile = eng.debug_gemm_full(case.shape, a, w, bias=bias if (case.bias or case.kind == 2) else None,
                               resid=o32 if case.resid else None, out_f32=o32, out_act=oa, rope_cos=rope[0],
                               rope_sin=rope[1], resid_epilogue=case.resid_epilogue, kind=case.kind, gelu=case.gelu,
                               C=case.C, heads=case.heads, posmode=case.posmode, F=case.F, qscale=case.qscale)
    return tile, o32, oa


def _check_gemm_case(eng, half, case):
    from beat_this_b200.weights import rope_tables

    dev = eng.device
    sh, M, N = case.shape, case.M, case.shape["N"]
    Ktot = sh["Kslab"] * sh["nslab"]
    g = torch.Generator(device=dev).manual_seed(zlib.crc32(case.id.encode()))
    a = torch.randn(sh["planes_in"] * sh["L"], sh["lda"], generator=g, device=dev)
    w = torch.randn(N, Ktot, generator=g, device=dev) / math.sqrt(Ktot)
    bias = torch.randn(N, generator=g, device=dev) * 0.5
    resid = torch.randn(M, N, generator=g, device=dev) if case.resid else None
    freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
    rope = tuple(t.contiguous().to(dev) for t in rope_tables(freqs)) if case.kind == 1 else (None, None)

    tile, o32, oa = _run_gemm(eng, case, a, w, bias, resid, rope)
    if half:
        assert tile == case.tile, f"plan tile {tile}, policy {case.tile}"
        again = _run_gemm(eng, case, a, w, bias, resid, rope)  # the same launch twice: bitwise equal
        for x, y in zip((o32, oa), again[1:]):
            assert x is None or torch.equal(bits(x), bits(y)), "16-bit GEMM is not deterministic"
    else:
        assert tile == (0, 0)

    adt = act_dtype(eng)
    dt = adt if half else None
    acc = gemm_ref(sh, rnd(a.double(), dt), rnd(w.double(), dt))
    ref, pre = epilogue_ref(case, acc, bias.double(), resid.double() if resid is not None else None, half,
                            *(t.double() if t is not None else None for t in rope))
    tol = (GEMM_ACC_TOL_H16 if half else GEMM_ACC_TOL_F32) * (1 + ref.abs())
    if case.kind == 2:
        tol = torch.full_like(ref, GATES_TOL)
    if pre is not None and half:
        tol = tol + 0.5 * pre.abs() * TANH_APPROX_TOL
    ldo = ref.shape[1]
    line = f"gemm {'h16' if half else 'f32'} {case.id}: tile {tile[0]}x{tile[1]} kind {case.kind} M={M} N={N} K={Ktot}"

    def check(name, got, ref, bound):
        err = (got - ref).abs().nan_to_num(float("inf"))  # an unwritten (NaN) element fails
        worst, ratio = err.max().item(), (err / bound).max().item()
        print(f"{line} | {name} max abs err {worst:.3e} = {ratio:.2f} of its bound")
        assert ratio <= 1, f"{name} off by up to {worst:.3e}, {ratio:.2f} x its bound"

    if o32 is not None:
        assert torch.isnan(o32[M * ldo :]).all(), "fp32 store past the last row"
        check("f32 out", o32[: M * ldo].view(M, ldo).double(), ref, tol)
    if oa is not None:
        assert torch.isnan(oa[M * N :]).all(), "activation store past the last row"
        got = oa[: M * N].view(M, N).double()
        if half:
            ref16 = ref.to(adt).double()
            check(f"{eng.act_dtype} out", got, ref16, ulp16(ref16, adt) + tol)
        else:
            check("act out (fp32)", got, ref, tol)
