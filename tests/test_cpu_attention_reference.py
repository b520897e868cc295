"""CPU tests (no GPU) of tests/attention_reference.py, the float64 restatement and bounds of the attention kernels:
- without rounding, the restatement is gates x F.scaled_dot_product_attention (with the key mask of chunked cases);
- an fp32 CPU emulation of attn_time_kernel (64-key tiles, base-2 online softmax, ex2_poly bit for bit on the
  AT_POLY_MASK pairs, MUFU as exact +- its stated error, P rounded to fp16, l from the unrounded p) and of
  attn_freq_mma_kernel stays within the bound, and each of a list of single mistakes leaves it;
- ex2_poly meets its stated relative error on a dense grid, clamps at -120 and gives a weight of 0 for -inf;
- the attention kernels in the built library are exactly the ones the GPU cases launch."""
import math
import re

import numpy as np
import pytest
import torch

import attention_reference as R
from numerics import EX2_APPROX_REL, EXPF_REL, QSCALE_H16, fma_f32, worst
from support import sass

H16 = torch.float16


# ---- fp32 building blocks, as the kernels compute them
def ex2_poly_np(x, c0=0.99992895):
    """tc_common.cuh ex2_poly, bit for bit (float32 numpy in and out)."""
    x = np.maximum(x.astype(np.float32), np.float32(-120.0))
    magic = np.float32(12582912.0)
    t = (x + magic).astype(np.float32)
    r = (x - (t - magic).astype(np.float32)).astype(np.float32)
    p = fma_f32(np.full_like(r, 0.05508868), r, np.full_like(r, 0.24260405))
    p = fma_f32(p, r, np.full_like(r, 0.69327623))
    p = fma_f32(p, r, np.full_like(r, np.float32(c0)))
    y = (t.view(np.int32).astype(np.int64) * 8388608 + p.view(np.int32).astype(np.int64)) & 0xFFFFFFFF
    return y.astype(np.uint32).view(np.int32).view(np.float32)


def ex2_mufu(x, rel=EX2_APPROX_REL):
    """ex2.approx.ftz.f32 as the exact 2^x off by its stated relative error, with alternating sign; ftz below 2^-126."""
    xd = x.double()
    sign = 1 - 2 * (torch.arange(x.numel()).view(x.shape) % 2).double()
    y = torch.exp2(xd) * (1 + rel * sign)
    return torch.where(xd < -126, 0.0, y).float()


def ex2_poly_t(x, c0=0.99992895):
    return torch.from_numpy(ex2_poly_np(x.numpy(), c0))


# ---- emulation of attn_time_kernel: one (sequence, head) at a time
def emulate_time_tc(q, k, v, gates, lens, mistake=None):
    """fp32 emulation of attn_time_kernel on the fp32 q, k, v [seqs, L, C], gates [seqs * L, H] the hook gets.
    mistake: None, "drop_last" (the last-tile mask off by one), "alpha_l" (l not rescaled), "poly_c0" (ex2_poly's
    constant 0.9995), "gate_head" (the gate of head h + 1), "v_prev" (key 0 of a tile takes the previous tile's V)."""
    seqs, L, C = q.shape
    H = C // 32
    qh = (q.float() * torch.tensor(QSCALE_H16, dtype=torch.float32)).to(H16).float()
    kh, vh = k.float().to(H16).float(), v.float().to(H16).float()
    poly = R.poly_keys(R.AT_TILE)
    c0 = 0.9995 if mistake == "poly_c0" else 0.99992895
    out = torch.empty(seqs, L, C, dtype=torch.float64)
    for s in range(seqs):
        Lk = int(lens[s])
        nkv = -(-Lk // R.AT_TILE)
        Kp = torch.zeros(nkv * R.AT_TILE, C)
        Vp = torch.zeros(nkv * R.AT_TILE, C)
        Kp[: min(L, nkv * R.AT_TILE)] = kh[s, : nkv * R.AT_TILE]  # TMA: rows past L read as zeros
        Vp[: min(L, nkv * R.AT_TILE)] = vh[s, : nkv * R.AT_TILE]
        for h in range(H):
            cs = slice(32 * h, 32 * h + 32)
            Q = qh[s, :, cs]
            m_run = torch.full((L,), -math.inf)
            l_run = torch.zeros(L)
            o = torch.zeros(L, 32)
            for j in range(nkv):
                Kt, Vt = Kp[64 * j : 64 * j + 64, cs], Vp[64 * j : 64 * j + 64, cs].clone()
                if mistake == "v_prev" and j > 0:
                    Vt[0] = Vp[64 * (j - 1), cs]
                S = Q @ Kt.T
                if j == nkv - 1:
                    lim = Lk - j * 64 - (1 if mistake == "drop_last" else 0)
                    S[:, lim:] = -math.inf
                mref = torch.maximum(m_run, S.amax(1))
                alpha = ex2_mufu(m_run - mref)
                m_run = mref
                if mistake != "alpha_l":
                    l_run = l_run * alpha
                o = o * alpha[:, None]
                x = S - mref[:, None]
                p = torch.where(poly, ex2_poly_t(x, c0), ex2_mufu(x))
                l_run = l_run + p.sum(1)
                o = o + p.to(H16).float() @ Vt
            hg = (h + 1) % H if mistake == "gate_head" else h
            gsc = gates[s * L : (s + 1) * L, hg].float() / l_run
            out[s, :, cs] = (o * gsc[:, None]).to(H16).double()
    return out


def emulate_freq_tc(q, k, v, gates, B, F, cross_mask=True):
    """fp32 emulation of attn_freq_mma_kernel<F>; cross_mask False: F = 8 without the -inf of the other group's keys
    (rows of frame t then also see the keys of frame t ^ 1 of the same 4-frame tile, zeros past L)."""
    M, C = q.shape
    H, L = C // 32, M // (B * F)
    grp = lambda t: t.float().to(H16).float().reshape(B, F, L, H, 32).permute(0, 2, 3, 1, 4)  # [B, L, H, F, 32]
    Q, K, V = grp(q), grp(k), grp(v)
    G = gates.float().reshape(B, F, L, H).permute(0, 2, 3, 1)
    if not cross_mask:
        pad = lambda t: torch.cat([t, torch.zeros_like(t[:, :1])], 1)
        partner = torch.arange(L) ^ 1
        partner = torch.where(partner < L, partner, L)
        K = torch.cat([K, pad(K)[:, partner]], 3)
        V = torch.cat([V, pad(V)[:, partner]], 3)
    S = Q @ K.transpose(-1, -2)
    mx = S.amax(-1, keepdim=True)
    x = ((S - mx) * torch.tensor(QSCALE_H16, dtype=torch.float32)).float()
    p = ex2_mufu(x, EXPF_REL)
    l = p.sum(-1)
    o = p.to(H16).float() @ V
    out = (o * (G / l)[..., None]).to(H16).double()
    return out.permute(0, 3, 1, 2, 4).reshape(M, C)


def _report(got, ref, bound):
    """(ratio, max abs error): a ratio of inf is an error where the bound asks for the exact value."""
    return worst(got, ref, bound), (got - ref).abs().max().item()


# ---- the restatement is the reference operation
@pytest.mark.parametrize("path", ["tc", "simt"])
def test_restatement_is_gated_sdpa(path):
    g = torch.Generator().manual_seed(3)
    case = R.TimeCase(4, 150, 2, (150, 97), 2)
    q, k, v, gates = (t.double() for t in R.time_inputs(case, "random", g, "cpu"))
    lens = torch.tensor(case.lens())
    got = R.time_ref(q, k, v, gates, lens, path, None, exact=True)[0]
    sh = lambda t: t.view(case.seqs, case.L, case.heads, 32).permute(0, 2, 1, 3)
    valid = torch.arange(case.L)[None, :] < lens[:, None]
    ref = torch.nn.functional.scaled_dot_product_attention(sh(q), sh(k), sh(v), attn_mask=valid[:, None, None, :])
    ref = (ref.permute(0, 2, 1, 3) * gates.view(case.seqs, case.L, case.heads, 1)).reshape(q.shape)
    assert (got - ref).abs().max().item() < 1e-12
    fc = R.FreqCase(2, 8, 5, 4)
    q, k, v, gates = (t.double() for t in R.freq_inputs(fc, "random", g, "cpu"))
    got = R.freq_ref(q, k, v, gates, fc.B, fc.F, path, None, exact=True)[0]
    sh = lambda t: t.view(fc.B, fc.F, fc.L, fc.heads, 32).permute(0, 2, 3, 1, 4)
    ref = torch.nn.functional.scaled_dot_product_attention(sh(q), sh(k), sh(v)).permute(0, 3, 1, 2, 4)
    ref = (ref * gates.view(fc.B, fc.F, fc.L, fc.heads, 1)).reshape(q.shape)
    assert (got - ref).abs().max().item() < 1e-12


# ---- the bounds hold the emulation and catch mistakes
MISTAKES = ("drop_last", "alpha_l", "poly_c0", "gate_head", "v_prev")
EMU_CASES = [R.TimeCase(2, 150, 2, (150, 97), 1), R.TimeCase(3, 129, 1), R.TimeCase(1, 13, 2), R.TimeCase(2, 200, 2, (65, 128), 1)]


def test_time_bound_holds_the_emulation_and_catches_mistakes():
    peak = {None: 0.0, **{m: {} for m in MISTAKES}}
    for ci, case in enumerate(EMU_CASES):
        for fam in R.time_families(case):
            g = torch.Generator().manual_seed(100 + ci)
            q, k, v, gates = R.time_inputs(case, fam, g, "cpu")
            lens = torch.tensor(case.lens())
            ref, bound, _, _ = R.time_ref(q.double(), k.double(), v.double(), gates.double(), lens, "tc", H16)
            good = worst(emulate_time_tc(q, k, v, gates, lens), ref, bound)
            print(f"{case.id} {fam}: emulation at {good:.3f} of the bound")
            assert good <= 1, (case.id, fam, good)
            peak[None] = max(peak[None], good)
            if fam in ("random", "dominant", "late_max", "flat_split"):
                for m in MISTAKES:
                    r, e = _report(emulate_time_tc(q, k, v, gates, lens, m), ref, bound)
                    w = peak[m].get(fam, (0.0, 0.0))
                    peak[m][fam] = (max(w[0], r), max(w[1], e))
    for m in MISTAKES:
        print(f"mistake {m}: " + ", ".join(f"{f} {r:.3g} x the bound (max error {e:.2e})" for f, (r, e) in peak[m].items()))
        assert max(r for r, _ in peak[m].values()) > 1, m
    for m in ("drop_last", "v_prev"):  # one misindexed key or value row: an O(1) error where it is the dominant key
        assert peak[m]["dominant"][0] > 100, (m, peak[m])
    # ex2_poly's constant at 0.9995: a bias of 4.9e-4 on 3 of 8 weights, the output itself on the flat_split rows
    assert peak["poly_c0"]["flat_split"][0] > 4 and peak["poly_c0"]["flat_split"][1] > 1e-4, peak["poly_c0"]


def test_freq_bound_holds_the_emulation_and_catches_the_cross_group_mask():
    for F, H in R.FREQ_TC_HEADS.items():
        for L in (1, 5, 13):
            case = R.FreqCase(2, F, L, H)
            for fam in R.freq_families(case):
                g = torch.Generator().manual_seed(F * 100 + L)
                q, k, v, gates = R.freq_inputs(case, fam, g, "cpu")
                ref, bound, _, _ = R.freq_ref(q.double(), k.double(), v.double(), gates.double(), case.B, F, "tc", H16)
                good = worst(emulate_freq_tc(q, k, v, gates, case.B, F), ref, bound)
                msg = f"{case.id} {fam}: emulation at {good:.3f} of the bound"
                if F == 8:
                    bad, e = _report(emulate_freq_tc(q, k, v, gates, case.B, F, cross_mask=False), ref, bound)
                    msg += f", without the cross-group mask at {bad:.3g} (max error {e:.2e})"
                    if fam == "cross_group" and L > 1:  # the other group's value: an O(1) error
                        assert bad > 100 and e > 0.1, (case.id, bad, e)
                print(msg)
                assert good <= 1, (case.id, fam, good)


# ---- ex2_poly
def test_ex2_poly_meets_its_stated_error():
    n = 10_000_000
    x = np.linspace(-130.0, 0.0, n, dtype=np.float64).astype(np.float32)
    ties = np.arange(-120, 1, dtype=np.float32) - np.float32(0.5)  # r = +-0.5: the Cody-Waite split's ties
    x = np.concatenate([x, ties, ties + 1, np.float32([-120.0, -0.0, 0.0])])
    y = ex2_poly_np(x).astype(np.float64)
    inside = x >= -120
    rel = np.abs(y[inside] / np.exp2(x[inside].astype(np.float64)) - 1)
    rel_max = rel.max()
    print(f"ex2_poly: max relative error {rel_max:.3e} at x = {x[inside][rel.argmax()]} over {inside.sum()} points")
    assert rel_max <= R.EX2_POLY_REL
    clamp = ex2_poly_np(np.float32([-120.0]))[0]
    assert np.all(y[~inside] == clamp) and clamp <= 2.0**-119
    neg_inf = ex2_poly_np(np.float32([-np.inf]))
    assert neg_inf[0] == clamp
    assert torch.from_numpy(neg_inf).to(H16).item() == 0  # a masked key's weight in P
    assert ex2_poly_np(np.float32([0.0]))[0] == np.float32(0.99992895)  # the bias at r = 0
    # fma_f32 agrees with an exact rational fmaf on random and constructed midpoint operands
    from fractions import Fraction

    rng = np.random.default_rng(0)
    a, b, c = (rng.standard_normal(2000).astype(np.float32) for _ in range(3))
    got = fma_f32(a, b, c)
    for i in range(0, 2000, 7):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cand = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
        best = min(cand, key=lambda f: (abs(Fraction(float(f)) - exact), int(np.float32(f).view(np.int32)) & 1))
        assert got[i] == best, i


# ---- every instantiation is tested
KERNEL = re.compile(r"_ZN2bt\d+(attn_time_kernel|attn_time_simt_kernel|attn_freq_kernel|attn_freq_mma_kernel)"
                    r"(?:ILi(\d+)EE)?")


def test_every_attention_instantiation_has_a_case(lib_built):
    found = set()
    for line in sass(lib_built).splitlines():
        if "Function :" in line and (m := KERNEL.search(line)):
            found.add((m.group(1), int(m.group(2) or 0)))
    launched = R.launched_kernels("tc") | R.launched_kernels("simt")
    assert found == launched, f"in the library only: {found - launched}, launched only: {launched - found}"
    assert len(found) == 8
    assert all(c.on_tensor_cores() for c in R.freq_cases("tc"))
    # the GPU test checks with the profiler that each context's hooks launch exactly the kernels PATHS names
    assert {p: R.PATHS[p][0] for p in R.PATHS} == {"tc": True, "simt": False}
