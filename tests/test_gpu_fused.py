"""GPU unit tests (pytest -m gpu) of the frontend's row kernels against the float64 restatements and bounds of
tests/fused_reference.py: norm_kernel<TAct, C> (bt_debug_norm, both contexts), fused_qkv_kernel<C> and
fused_ff_kernel<C, OP> (bt_debug_fused_qkv / bt_debug_fused_ff, 16-bit context).

Every case fills its outputs with NaN, and has one more row after M: a finite input row the kernel must not read
and a NaN output row it must not write (the in-place X of the fused FFN keeps a finite sentinel row, so that a store
to it shows).  Every row < M must be finite and within its elementwise bound, and a second run must give the same
bits.  Each case prints its worst error as a fraction of its bound; all cases run, and the failures are listed
together at the end."""
import math
import zlib

import pytest
import torch

from fused_reference import (ff_cases, ff_ref, gates_ref, norm_cases, norm_ref, qkv_cases, qkv_ref, random_weights,
                             special_rows)
from gemm_reference import QSCALE_TIME
from numerics import normalize
from support import act_dtype, bits, dev  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

NAN = float("nan")


@pytest.fixture(scope="module")
def engines(lib_built, dev):
    """Weight-less contexts: {False: fp32, True: 16-bit}."""
    from beat_this_b200.engine import Engine

    return {half: Engine(None, None, dev, half=half) for half in (False, True)}


def _rope(dev):
    from beat_this_b200.weights import rope_tables

    return tuple(t.to(dev).contiguous() for t in rope_tables(1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))))


def _f32(t):
    return t.float().contiguous()


def _with_row(x, row):
    """x [M, n] fp32 with one more row appended."""
    return torch.cat([_f32(x), row.reshape(1, -1).to(x.device, torch.float32)]).contiguous()


class Family:
    """The worst error-to-bound ratio of a family of cases, and its failures."""

    def __init__(self, name):
        self.name, self.worst, self.failures, self.cases = name, 0.0, [], 0

    def run(self, case_id, fn, *args):
        self.cases += 1
        try:
            fn(self, case_id, *args)
        except AssertionError as e:
            self.failures.append(f"{case_id}: {str(e).splitlines()[0]}")

    def check(self, case_id, what, got, ref, bound):
        assert torch.isfinite(got).all(), f"{what}: non-finite values in rows < M"
        ratio = ((got - ref).abs() / bound).max().item()
        print(f"{self.name} {case_id} | {what}: max {(got - ref).abs().max().item():.3e} = {ratio:.3f} of its bound")
        self.worst = max(self.worst, ratio)
        assert ratio <= 1, f"{what} off by {ratio:.2f} x its bound"

    def finish(self):
        print(f"{self.name}: worst error {self.worst:.3f} of its bound over {self.cases} cases")
        assert not self.failures, f"{len(self.failures)} of {self.cases} {self.name} cases failed:\n" + "\n".join(self.failures)


# ------------------------------------------------------------------------------ fused FFN
def _ff_case(fam, case_id, eng, C, op, xb, M, x, w, o):
    """x [M, C], o [M + 1, C] (its last row NaN) float64 on the device; w: float64 weights."""
    dt = act_dtype(eng)
    sentinel = torch.full((C,), 7.0)
    X0 = _with_row(x, sentinel)
    runs = []
    for _ in range(2):
        X = X0.clone()
        XB = torch.full((M + 1, C), NAN, device=x.device) if xb else None
        eng.debug_fused_ff(X, _f32(w["w1"]), _f32(w["b1"]), _f32(w["w2"]), _f32(w["b2"]), M, C,
                           o=_f32(o) if op else None, wout=_f32(w["wout"]) if op else None, xb_out=XB)
        runs.append((X, XB))
    (X, XB), (X2, XB2) = runs
    assert torch.equal(bits(X), bits(X2)) and (not xb or torch.equal(bits(XB), bits(XB2))), "not deterministic"
    assert torch.equal(bits(X[M]), bits(X0[M])), "X changed past row M"
    ref, bound = ff_ref(x, w["w1"], w["b1"], w["w2"], w["b2"], o[:M] if op else None, w["wout"] if op else None, dt)
    fam.check(case_id, "x", X[:M].double(), ref, bound)
    if xb:
        assert torch.isnan(XB[M]).all(), "16-bit copy written past row M"
        assert torch.equal(bits(XB[:M]), bits(X[:M].to(dt).float())), "16-bit copy is not round16 of the fp32 result"


def test_fused_ff(engines, dev):
    eng = engines[True]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    fam = Family("fused_ff")
    for C, op, xb, M in ff_cases(sms):
        case_id = f"C={C} outproj={op} xb={xb} M={M}"
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(case_id.encode()))
        w = random_weights(C, g, dev)
        x = special_rows(M, C, g, dev)
        o = torch.cat([torch.randn(M, C, generator=g, dtype=torch.float64, device=dev), torch.full((1, C), NAN, device=dev)])
        fam.run(case_id, _ff_case, eng, C, op, xb, M, x, w, o)
    fam.finish()


# ------------------------------------------------------------------------------ fused QKV
def _qkv_case(fam, case_id, eng, C, posmode, L, F, qscale, M, x, w, rope):
    dt = act_dtype(eng)
    heads = C // 32
    X = _with_row(x, torch.randn(C) * 3)
    runs = []
    for _ in range(2):
        QKV = torch.full((M + 1, 3 * C), NAN, device=x.device)
        G = torch.full((M + 1, heads), NAN, device=x.device)
        eng.debug_fused_qkv(X, _f32(w["wqkv"]), _f32(w["wg"]), _f32(w["bg"]), rope[0], rope[1], QKV, G, M, C, L, F,
                            posmode, qscale)
        runs.append((QKV, G))
    (QKV, G), (QKV2, G2) = runs
    assert torch.equal(bits(QKV), bits(QKV2)) and torch.equal(bits(G), bits(G2)), "not deterministic"
    assert torch.isnan(QKV[M]).all() and torch.isnan(G[M]).all(), "store past row M"
    cos, sin = (t.double() for t in rope)
    ref, bound, gref, gbound = qkv_ref(x, w["wqkv"], w["wg"], w["bg"], cos, sin, L, F, posmode, qscale, dt)
    fam.check(case_id, "qkv", QKV[:M].double(), ref, bound)
    fam.check(case_id, "gates", G[:M].double(), gref, gbound)


def test_fused_qkv(engines, dev):
    eng = engines[True]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    rope = _rope(dev)
    fam = Family("fused_qkv")
    for C, posmode, L, F, qscale, M in qkv_cases(sms):
        case_id = f"C={C} posmode={posmode} L={L} F={F} M={M}"
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(case_id.encode()))
        w = random_weights(C, g, dev)
        x = special_rows(M, C, g, dev)
        fam.run(case_id, _qkv_case, eng, C, posmode, L, F, qscale, M, x, w, rope)
    fam.finish()


# ------------------------------------------------------------------------------ norm
def _norm_case(fam, case_id, eng, C, heads, M, x, wg, bg):
    dt = act_dtype(eng) if eng.half else None
    X = _with_row(x, torch.randn(C) * 3)
    runs = []
    for _ in range(2):
        XN = torch.full((M + 1, C), NAN, device=x.device)
        G = torch.full((M + 1, max(heads, 1)), NAN, device=x.device)
        eng.debug_norm(X, XN, M, C, _f32(wg) if heads else None, _f32(bg) if heads else None, G if heads else None, heads)
        runs.append((XN, G))
    (XN, G), (XN2, G2) = runs
    assert torch.equal(bits(XN), bits(XN2)) and torch.equal(bits(G), bits(G2)), "not deterministic"
    assert torch.isnan(XN[M]).all() and torch.isnan(G[M]).all(), "store past row M"
    ref, bound = norm_ref(x, dt)
    fam.check(case_id, "xn", XN[:M].double(), ref, bound)
    if heads:
        gref, gbound = gates_ref(normalize(x), wg, bg, heads)
        fam.check(case_id, "gates", G[:M].double(), gref, gbound)
    else:
        assert torch.isnan(G).all(), "gates written without heads"


@pytest.mark.parametrize("half", [False, True])
def test_norm(engines, dev, half):
    eng = engines[half]
    fam = Family(f"norm {'16-bit' if half else 'fp32'}")
    for C, heads, M in norm_cases():
        case_id = f"C={C} heads={heads} M={M}"
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(case_id.encode()))
        x = special_rows(M, C, g, dev)
        wg = torch.randn(4, C, generator=g, dtype=torch.float64, device=dev) * 2 / math.sqrt(C)
        bg = torch.randn(4, generator=g, dtype=torch.float64, device=dev)
        fam.run(case_id, _norm_case, eng, C, heads, M, x, wg, bg)
    fam.finish()


# ------------------------------------------------------------------------------ production weights
def _sdpa_out(qkv, gates, B, F, L, C, freq):
    """gates * SDPA of the unrounded q, k, v [M, 3C] over F (freq) or L: the attention output O [M, C]."""
    heads = C // 32
    q, k, v = (t.reshape(B, F, L, heads, 32) for t in qkv.split(C, dim=1))
    perm = (0, 2, 3, 1, 4) if freq else (0, 1, 3, 2, 4)  # sequence axis second to last
    inv = (0, 3, 1, 2, 4) if freq else (0, 1, 3, 2, 4)
    o = torch.nn.functional.scaled_dot_product_attention(*(t.permute(*perm) for t in (q, k, v))).permute(*inv)
    return (o * gates.reshape(B, F, L, heads, 1)).reshape(-1, C)


def test_fused_production_weights(engines, dev):
    """The packed b0 / b1 weights of final0 on the oracle's activations at the inputs of the same layers."""
    from beat_this_b200 import synthetic, weights
    from oracle import beat_this_oracle as O

    eng = engines[True]
    hp = synthetic.model_hparams("final0")
    sd = synthetic.make_state_dict(hp, 0)
    packed = {k: torch.from_numpy(v).to(dev, torch.float64) for k, v in weights.pack_parameters(sd, hp).items()}
    B, L = 1, 150
    taps = {}
    with torch.inference_mode():
        O.forward(sd, torch.rand(B, L, 128, generator=torch.Generator().manual_seed(9)) * 7, taps)
    rope = _rope(dev)
    cos, sin = (t.double() for t in rope)
    fam = Family("production weights")
    for i, C, F in ((0, 32, 32), (1, 64, 16)):
        P = lambda n, *shape: packed[f"b{i}.{n}"].view(*shape)
        inputs = {"attnF": "stem" if i == 0 else "b0.conv", "ffF": f"b{i}.attnF", "attnT": f"b{i}.ffF", "ffT": f"b{i}.attnT"}
        X = {k: taps[v].to(dev, torch.float64).reshape(-1, C) for k, v in inputs.items()}
        M = X["attnF"].shape[0]
        for part, posmode, qscale in (("attnF", 1, 1.0), ("attnT", 0, QSCALE_TIME)):
            w = dict(wqkv=P(f"{part}.wqkv", 3 * C, C), wg=P(f"{part}.wg", 32, C), bg=P(f"{part}.bg", 32))
            fam.run(f"b{i}.{part}", _qkv_case, eng, C, posmode, L, F, qscale, M, X[part], w, rope)
        for part, attn in (("ffF", "attnF"), ("ffT", "attnT")):
            w = dict(w1=P(f"{part}.w1", 4 * C, C), b1=P(f"{part}.b1", 4 * C), w2=P(f"{part}.w2", C, 4 * C),
                     b2=P(f"{part}.b2", C), wout=P(f"{attn}.wout", C, C))
            nan_row = torch.full((1, C), NAN, device=dev)
            fam.run(f"b{i}.{part}", _ff_case, eng, C, False, True, M, X[part], w, torch.cat([X[part], nan_row]))
            # with the out-projection in front: x is the attention's input, O its gated output (float64 SDPA)
            qkv, _, gates, _ = qkv_ref(X[attn], P(f"{attn}.wqkv", 3 * C, C), P(f"{attn}.wg", 32, C), P(f"{attn}.bg", 32),
                                       cos, sin, L, F, 1 if attn == "attnF" else 0, 1.0, None)
            o = _sdpa_out(qkv, gates, B, F, L, C, attn == "attnF")
            fam.run(f"b{i}.{attn}+{part}", _ff_case, eng, C, True, True, M, X[attn], w, torch.cat([o, nan_row]))
    fam.finish()


# ------------------------------------------------------------------------------ argument checks and launch counts
def test_hooks_reject_bad_arguments_and_count_launches(engines, dev):
    from beat_this_b200._lib import BTError

    e16, e32 = engines[True], engines[False]
    C, M = 32, 20
    x = torch.randn(M + 1, C, device=dev)
    w = {k: _f32(v) for k, v in random_weights(C, torch.Generator(device=dev).manual_seed(0), dev).items()}
    rope = _rope(dev)
    qkv, gates, xn = torch.zeros(M, 3 * C, device=dev), torch.zeros(M, 1, device=dev), torch.zeros(M, C, device=dev)
    big = torch.zeros(1 << 16, device=dev)  # large enough for every geometry below
    bad = [
        lambda: e32.debug_fused_ff(x, w["w1"], w["b1"], w["w2"], w["b2"], M, C),  # fp32 context
        lambda: e16.debug_fused_ff(big, big, big, big, big, M, 48),
        lambda: e16.debug_fused_ff(x, w["w1"], w["b1"], w["w2"], w["b2"], M, C, o=x),  # o without wout
        lambda: e16.debug_fused_ff(x, w["w1"], w["b1"], w["w2"], w["b2"], 0, C),
        lambda: e16.debug_fused_ff(x.view(-1)[1:], w["w1"], w["b1"], w["w2"], w["b2"], M, C),  # x not 16-byte aligned
        lambda: e32.debug_fused_qkv(x, w["wqkv"], w["wg"], w["bg"], *rope, qkv, gates, M, C, 13, 1, 0, 1.0),
        lambda: e16.debug_fused_qkv(big, big, big, big, *rope, big, big, M, 128, 13, 1, 0, 1.0),
        lambda: e16.debug_fused_qkv(x, w["wqkv"], w["wg"], w["bg"], *rope, qkv, gates, M, C, 1501, 1, 0, 1.0),
        lambda: e16.debug_fused_qkv(x, w["wqkv"], w["wg"], w["bg"], *rope, qkv, gates, M, C, 13, 1, 2, 1.0),
        lambda: e16.debug_norm(big, big, M, 48),
        lambda: e16.debug_norm(x, xn, M, C, heads=1),  # heads without gates
        lambda: e32.debug_norm(x, xn, M, C, big, big, big, 2),  # 32 heads > C
        lambda: e32.debug_norm(x, xn, M, C, None, w["bg"], gates, 1),
        lambda: e32.debug_norm(x, big.view(-1)[1:], M, C),  # the fp32 context stores xn with 16-byte stores
    ]
    before = {h: e.lib.bt_launch_count(e.ctx) for h, e in engines.items()}
    for i, call in enumerate(bad):
        with pytest.raises(BTError, match="error -1"):
            call()
    with pytest.raises(AssertionError, match="elements"):  # the wrapper checks the sizes the hook cannot see
        e16.debug_norm(x, xn[: M - 1], M, C)
    assert {h: e.lib.bt_launch_count(e.ctx) for h, e in engines.items()} == before, "a rejected call launched"
    e16.debug_fused_ff(x, w["w1"], w["b1"], w["w2"], w["b2"], M, C)
    e16.debug_fused_qkv(x, w["wqkv"], w["wg"], w["bg"], *rope, qkv, gates, M, C, 13, 1, 0, 1.0)
    e16.debug_norm(x, xn, M, C)
    e32.debug_norm(x, xn, M, C, w["wg"], w["bg"], gates, 1)
    assert e16.lib.bt_launch_count(e16.ctx) == before[True] + 3
    assert e32.lib.bt_launch_count(e32.ctx) == before[False] + 1
