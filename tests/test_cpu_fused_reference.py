"""CPU tests (no GPU) of tests/fused_reference.py, the float64 restatement and bounds of the frontend's row kernels:
- without rounding, the restatement is the reference's block (oracle.feedforward and the part of oracle.attention in
  front of the softmax) on the packed weights of the synthetic checkpoints;
- a CPU emulation of each kernel in fp32, with the kernel's 16-bit rounding points, stays within the bound, and the same
  emulation with one mistake leaves it (the bound is neither unsound nor vacuous);
- the instantiations of norm_kernel, fused_qkv_kernel and fused_ff_kernel in the built library are exactly the ones
  the GPU cases run."""
import math
import os
import re

import numpy as np
import pytest
import torch

from fused_reference import (FF_CTAS, NORM_CS, QKV_CTAS, ff_cases, ff_ref, gates_ref, norm_cases, norm_ref, qkv_cases,
                             qkv_ref, random_weights, special_rows)
from gemm_reference import QSCALE_TIME
from numerics import gelu_erf, gelu_tanh, normalize, rope_positions, worst
from support import sass

H16 = torch.float16


def _packed(name):
    from beat_this_b200 import synthetic, weights

    hp = synthetic.model_hparams(name)
    sd = synthetic.make_state_dict(hp, 0)
    packed = {k: torch.from_numpy(v).double() for k, v in weights.pack_parameters(sd, hp).items()}
    return sd, packed


def _layer(packed, prefix, C):
    P = lambda n, *shape: packed[prefix + n].view(*shape)
    if "attn" in prefix:
        return dict(wqkv=P(".wqkv", 3 * C, C), wg=P(".wg", 32, C), bg=P(".bg", 32), wout=P(".wout", C, C))
    return dict(w1=P(".w1", 4 * C, C), b1=P(".b1", 4 * C), w2=P(".w2", C, 4 * C), b2=P(".b2", C))


def _oracle_pre_attention(z, sd, p, heads):
    """oracle.pre_attention on z [S, n, C]: roped q and k, v [S, n, C] and the gates [S, n, heads] (after the
    sigmoid)."""
    from oracle import beat_this_oracle as O

    S, n, C = z.shape
    q, k, v, gates = O.pre_attention(z, sd, p, heads)
    back = lambda t: t.permute(0, 2, 1, 3).reshape(S, n, C)
    return back(q), back(k), back(v), torch.sigmoid(gates)


@pytest.mark.parametrize("name", ["small0", "final0"])
def test_restatement_is_the_reference_block(name):
    from oracle import beat_this_oracle as O

    sd, packed = _packed(name)
    cos, sin = packed["rope.cos"].view(1500, 16), packed["rope.sin"].view(1500, 16)
    g = torch.Generator().manual_seed(7)
    B, L = 2, 13
    for i, C, Fq in ((0, 32, 32), (1, 64, 16)):
        heads = C // 32
        x = torch.randn(B, Fq, L, C, generator=g) * 2  # [B, F, L, C]: row m = (b F + f) L + t
        xf = x.double().reshape(-1, C)
        for part in ("ffF", "ffT"):
            w = _layer(packed, f"b{i}.{part}", C)
            ref = (x + O.feedforward(x, sd, f"frontend.blocks.{i}.partial.{part}")).reshape(-1, C).double()
            got, _ = ff_ref(xf, w["w1"], w["b1"], w["w2"], w["b2"], gelu=gelu_erf)
            err = ((got - ref).abs() / (1 + ref.abs())).max().item()
            print(f"{name} b{i}.{part}: restatement vs oracle.feedforward {err:.2e}")
            assert err < 2e-5, (name, i, part, err)
        for part, posmode in (("attnF", 1), ("attnT", 0)):
            w = _layer(packed, f"b{i}.{part}", C)
            if posmode == 1:  # sequences over the F planes of each (chunk, frame)
                z = x.permute(0, 2, 1, 3).reshape(B * L, Fq, C)
                unz = lambda t: t.view(B, L, Fq, -1).permute(0, 2, 1, 3).reshape(B * Fq * L, -1)
            else:
                z = x.reshape(B * Fq, L, C)
                unz = lambda t: t.reshape(B * Fq * L, -1)
            q, k, v, gates = (unz(t).double() for t in _oracle_pre_attention(z, sd, f"frontend.blocks.{i}.partial.{part}", heads))
            got, _, got_g, _ = qkv_ref(xf, w["wqkv"], w["wg"], w["bg"], cos, sin, L, Fq, posmode, 1.0, None)
            for what, a, b in (("q", got[:, :C], q), ("k", got[:, C : 2 * C], k), ("v", got[:, 2 * C :], v),
                               ("gates", got_g, gates)):
                err = ((a - b).abs() / (1 + b.abs())).max().item()
                print(f"{name} b{i}.{part} {what}: restatement vs oracle.attention {err:.2e}")
                assert err < 2e-5, (name, i, part, what, err)


# ---- CPU emulation of the kernels: fp32 arithmetic, 16-bit rounding where the kernel rounds
def _r16(t):
    return t.to(H16).float()


def _emu_norm(x32):
    return x32 * (1.0 / (x32 * x32).sum(-1, keepdim=True).sqrt().clamp_min(1e-12))


def emulate_ff(x, w1, b1, w2, b2, o=None, wout=None, drop_b2_block=False, b2_shift=0.0, hidden=H16):
    x32 = x.float()
    if o is not None:
        x32 = x32 + _r16(o) @ _r16(wout).T
    u16 = _r16(_emu_norm(x32))
    h16 = gelu_tanh(u16 @ _r16(w1).T + b1.float()).to(hidden).float()  # hidden: the type the hidden units round to
    b2e = b2.float().clone()
    if drop_b2_block:  # the mistake: b2 missing from one 8-column block
        b2e[-8:] = 0
    b2e[3] += b2_shift  # the mistake: one output column off by b2_shift
    return (x32 + b2e + h16 @ _r16(w2).T).double()


def emulate_qkv(x, wqkv, wg, bg, cos, sin, L, F, posmode, qscale, pos_mod_f=False):
    M, C = x.shape
    u = _emu_norm(x.float())
    gates = torch.sigmoid(u @ wg[: C // 32].float().T + bg[: C // 32].float())
    acc = _r16(u) @ _r16(wqkv).T
    m = torch.arange(M)
    pos = m % F if pos_mod_f else rope_positions(M, L, F, posmode)  # the mistake: posmode-1 position m % F
    c, s = cos[pos].float(), sin[pos].float()
    out = acc.clone()
    for which, sc in ((0, qscale), (1, 1.0)):
        p = acc[:, which * C : (which + 1) * C].reshape(M, -1, 16, 2)
        x0, x1 = p[..., 0], p[..., 1]
        rot = torch.stack(((x0 * c[:, None] - x1 * s[:, None]) * sc, (x1 * c[:, None] + x0 * s[:, None]) * sc), -1)
        out[:, which * C : (which + 1) * C] = rot.reshape(M, C)
    return _r16(out).double(), gates.double()


@pytest.mark.parametrize("C", [32, 64])
def test_bounds_hold_the_emulation_and_catch_a_mistake(C):
    from beat_this_b200.weights import rope_tables

    g = torch.Generator().manual_seed(C)
    w = random_weights(C, g)
    M = 2 * 16 * 150 + 7
    x = special_rows(M, C, g)
    o = torch.randn(M, C, generator=g, dtype=torch.float64)
    for op in (False, True):
        oo, wo = (o, w["wout"]) if op else (None, None)
        ref, bound = ff_ref(x, w["w1"], w["b1"], w["w2"], w["b2"], oo, wo, H16)
        good = worst(emulate_ff(x, w["w1"], w["b1"], w["w2"], w["b2"], oo, wo), ref, bound)
        bad = worst(emulate_ff(x, w["w1"], w["b1"], w["w2"], w["b2"], oo, wo, drop_b2_block=True), ref, bound)
        # an error of 1e-2 in one column: the size the stage taps (0.03 absolute) cannot see
        shift = worst(emulate_ff(x, w["w1"], w["b1"], w["w2"], w["b2"], oo, wo, b2_shift=1e-2), ref, bound)
        bf16 = worst(emulate_ff(x, w["w1"], w["b1"], w["w2"], w["b2"], oo, wo, hidden=torch.bfloat16), ref, bound)
        print(f"ff C={C} outproj={op}: emulation at {good:.3f} of the bound; with b2 dropped from a block at {bad:.1f}, "
              f"one column off by 1e-2 at {shift:.2f}, hidden units in bf16 at {bf16:.2f}")
        assert good <= 1 and bad > 1 and shift > 1
    cos, sin = (t.double() for t in rope_tables(1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))))
    for posmode, L, F, qscale in ((0, 150, 1, QSCALE_TIME), (1, 150, 32 // (C // 32), 1.0)):
        ref, bound, gref, gbound = qkv_ref(x, w["wqkv"], w["wg"], w["bg"], cos, sin, L, F, posmode, qscale, H16)
        got, gates = emulate_qkv(x, w["wqkv"], w["wg"], w["bg"], cos, sin, L, F, posmode, qscale)
        good, gr = worst(got, ref, bound), worst(gates, gref, gbound)
        print(f"qkv C={C} posmode={posmode}: emulation at {good:.3f} of the bound, gates at {gr:.3f}")
        assert good <= 1 and gr <= 1
        if posmode == 1:
            bad, _ = emulate_qkv(x, w["wqkv"], w["wg"], w["bg"], cos, sin, L, F, posmode, qscale, pos_mod_f=True)
            print(f"qkv C={C} posmode=1 with position m % F: {worst(bad, ref, bound):.1f} of the bound")
            assert worst(bad, ref, bound) > 1


@pytest.mark.parametrize("C", NORM_CS)
def test_norm_bound_holds_the_emulation(C):
    g = torch.Generator().manual_seed(C)
    x = special_rows(1000, C, g)
    for dt in (None, H16):
        ref, bound = norm_ref(x, dt)
        u = _emu_norm(x.float())
        got = (u if dt is None else _r16(u)).double()
        print(f"norm C={C} {'fp32' if dt is None else 'fp16'}: emulation at {worst(got, ref, bound):.3f} of the bound")
        assert worst(got, ref, bound) <= 1
    wg = torch.randn(4, C, generator=g, dtype=torch.float64) / math.sqrt(C)
    bg = torch.randn(4, generator=g, dtype=torch.float64)
    u = _emu_norm(x.float())
    gates = torch.sigmoid(u @ wg.float().T + bg.float()).double()
    gref, gbound = gates_ref(normalize(x), wg, bg, min(4, C // 32))
    assert worst(gates[:, : gref.shape[1]], gref, gbound) <= 1


def test_every_instantiation_has_a_unit_test(lib_built):
    """The instantiations of the three row kernels in the library are exactly the ones the GPU cases run, and the
    grid-stride cases use the CTAs per SM the launchers use."""
    ff = re.compile(r"_ZN2bt15fused_ff_kernelILi(\d+)ELb([01])EE")
    qkv = re.compile(r"_ZN2bt16fused_qkv_kernelILi(\d+)EE")
    norm = re.compile(r"_ZN2bt11norm_kernelI(f|6__half|13__nv_bfloat16)Li(\d+)EE")
    found = {"ff": set(), "qkv": set(), "norm": set()}
    for line in sass(lib_built).splitlines():
        if "Function :" not in line:
            continue
        if m := ff.search(line):
            found["ff"].add((int(m.group(1)), m.group(2) == "1"))
        elif m := qkv.search(line):
            found["qkv"].add(int(m.group(1)))
        elif m := norm.search(line):
            found["norm"].add((m.group(1) != "f", int(m.group(2))))
    listed = {"ff": {(C, op) for C, op, _, _ in ff_cases(132)},
              "qkv": {c[0] for c in qkv_cases(132)},
              "norm": {(half, C) for C, _, _ in norm_cases() for half in (False, True)}}
    for k in found:
        assert found[k] == listed[k], f"{k}: in the library only {found[k] - listed[k]}, listed only {listed[k] - found[k]}"
    assert len(found["ff"]) == 4 and len(found["qkv"]) == 2 and len(found["norm"]) == 12
    src = open(os.path.join(os.path.dirname(__file__), "..", "beat_this_b200", "csrc", "kernels_fused.cu")).read()
    for fn, table in (("ff_ctas", FF_CTAS), ("qkv_ctas", QKV_CTAS)):
        m = re.search(fn + r"\(\) \{ return C == 32 \? (\d+) : (\d+); \}", src)
        assert m and (int(m.group(1)), int(m.group(2))) == (table[32], table[64]), fn


def test_special_rows():
    x = special_rows(23, 32, torch.Generator().manual_seed(0))
    n = x.norm(dim=1).numpy()
    assert n[3] == 0 and n[14] == 0 and np.count_nonzero(x[4].numpy()) == 1
    assert np.allclose(n[[5, 6, 16, 17]], [1e-3, 1e-8, 1e-3, 1e-8]) and x[7].abs().mean() > 20
