"""CPU tests (no GPU) of tests/train_kernels_reference.py: the float64 restatements are gradients of the oracle's
functions (float64 autograd of O.rmsnorm, O.rope, O.batchnorm + F.gelu, softmax attention and the gate), the fp32
emulations of the kernels stay within the bounds on the GPU test's kinds of cases, and each planted single-line
mistake takes its emulation past the bound.  Each mistake's case and ratio are printed (pytest -s)."""
import math

import pytest
import torch
import torch.nn.functional as Fn

import train_kernels_reference as R
from numerics import worst
from oracle import beat_this_oracle as O
from support import rnd


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _bn(C, g):  # running variances 0.5 .. 1.5, as the synthetic checkpoints have them
    return (rnd(C, g=g), rnd(C, g=g), rnd(C, g=g), 0.5 + torch.rand(C, generator=g).float())


def _sd(bn):
    return {"p.weight": R.f64(bn[0]), "p.bias": R.f64(bn[1]), "p.running_mean": R.f64(bn[2]),
            "p.running_var": R.f64(bn[3])}


def close(a, b, rel=1e-12):
    a, b = R.f64(a), R.f64(b)
    assert (a - b).abs().max() <= rel * (1 + b.abs().max()), float((a - b).abs().max())


# ------------------------------------------------------------------------------------ restatements = oracle gradients
def test_rmsnorm_restatement_is_the_oracle_gradient():
    g = _g(0)
    x = rnd(6, 64, g=g).double()
    x[2] *= 1e-14  # clamped
    gamma, dxn = rnd(64, g=g).double(), rnd(6, 64, g=g).double()
    xr = x.clone().requires_grad_(True)
    y = O.rmsnorm(xr, gamma)
    (dx,) = torch.autograd.grad(y, xr, dxn)
    xn, _, inv, _ = R.rms_fwd_ref(x, gamma)
    close(xn, y.detach(), 1e-7)  # the restatement clamps at the kernels' fp32(1e-12)
    ref, _ = R.rms_bwd_ref(dxn, x, inv, gamma)
    close(ref, dx, 1e-7)


def test_bn_gelu_restatements_are_the_oracle_gradients():
    g = _g(1)
    C, n = 8, 8 * 50
    bn = _bn(C, g)
    sd = {k: v.clone().requires_grad_(True) for k, v in _sd(bn).items()}
    z = rnd(n, g=g, scale=3.0).double().reshape(-1, C).requires_grad_(True)
    dy = rnd(n, g=g).double().reshape(-1, C)
    y = Fn.gelu(O.batchnorm(z, sd, "p", 1))
    dz, dw, db = torch.autograd.grad(y, [z, sd["p.weight"], sd["p.bias"]], dy)
    yr, _ = R.bn_gelu_fwd_ref(z.detach().reshape(-1), bn, C)
    close(yr, y.detach().reshape(-1))
    dbn, _, dzr, _ = R.bn_gelu_bwd_ref(dy.reshape(-1), z.detach().reshape(-1), bn, C)
    close(dzr, dz.reshape(-1))
    s_gz = (dbn.reshape(-1, C) * z.detach()).sum(0)
    s_g = dbn.reshape(-1, C).sum(0)
    dwr, _, dbr = R.bn_grads_ref(s_gz, s_g, bn)
    close(dwr, dw)
    close(dbr, db)
    # bn_scale: the gradient at a 1-d BatchNorm's input
    x = rnd(n, g=g).double().reshape(-1, C).requires_grad_(True)
    (dx,) = torch.autograd.grad(O.batchnorm(x, sd, "p", 1), x, dy)
    close(R.bn_scale_ref(dy.reshape(-1), bn, C)[0], dx.reshape(-1))
    h = rnd(n, g=g, scale=4.0).double().requires_grad_(True)
    (dh,) = torch.autograd.grad(Fn.gelu(h), h, dy.reshape(-1))
    close(R.gelu_bwd_ref(dy.reshape(-1), h.detach())[0], dh)


def test_rope_restatement_is_the_oracle_rotation_and_its_adjoint():
    g = _g(2)
    n, C = 40, 64
    qkv = rnd(n, 3 * C, g=g)
    fr = (1.0 / 10000 ** (torch.arange(0, 32, 2).float() / 32)).float()
    ref, _ = R.rope_ref(qkv, fr, n, 1, 0, False)
    q = qkv[:, :C].double().reshape(n, 2, 32).permute(1, 0, 2).requires_grad_(True)
    rq = O.rope(q, fr)
    close(ref[:, :C].reshape(n, 2, 32).permute(1, 0, 2), rq.detach(), 1e-7)  # the oracle's angle is fp32 as well
    dy = rnd(n, 3 * C, g=g)
    (dq,) = torch.autograd.grad(rq, q, dy[:, :C].double().reshape(n, 2, 32).permute(1, 0, 2))
    inv, _ = R.rope_ref(dy, fr, n, 1, 0, True)
    close(inv[:, :C].reshape(n, 2, 32).permute(1, 0, 2), dq, 1e-7)


def test_attention_and_gate_restatements_are_the_oracle_gradients():
    g = _g(3)
    S, n, H = 2, 9, 2
    C = 32 * H
    qkv = rnd(S * n, 3 * C, g=g)
    rows = R.seq_rows(S, n, 1, n, 0, 1)
    q, k, v = (qkv[:, i * C:(i + 1) * C].double().reshape(S, n, H, 32).permute(0, 2, 1, 3).requires_grad_(True)
               for i in range(3))
    gl = rnd(S, n, H, g=g).double().requires_grad_(True)
    att = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(32), -1) @ v
    y = att * gl.permute(0, 2, 1).unsqueeze(-1).sigmoid()
    dy = rnd(S, H, n, 32, g=g).double()
    dq, dk, dv, dgl = torch.autograd.grad(y, [q, k, v, gl], dy)
    Oref, _, lse, _ = R.attn_fwd_ref(qkv, rows, H)
    close(Oref.reshape(S, H, n, 32), att.detach(), 1e-6)  # the restatement scales q by the kernels' fp32 1 / sqrt 32
    Ofull = R.heads_back(Oref, rows, H, S * n, 0, C)
    dG = dy.permute(0, 2, 1, 3).reshape(S * n, C)
    dO, _, dg, _, delta, _ = R.gate_bwd_ref(dG, Ofull, gl.detach().reshape(S * n, H))
    close(dg, dgl.reshape(S * n, H), 1e-6)
    lse_t = lse.reshape(S, H, n).permute(0, 2, 1).reshape(S * n, H)
    dqr, _, dkr, _, dvr, _ = R.attn_bwd_ref(qkv, dO, lse_t, delta, rows, H)
    for a, b in ((dqr, dq), (dkr, dk), (dvr, dv)):
        close(a.reshape(S, H, n, 32), b, 1e-6)


def test_col2im_is_the_adjoint_of_im2col():
    g = _g(4)
    for gm in ((2, 16, 2, 5, 32, 16 * 2 * 5 * 32, 5 * 32, 32, 1), (1, 32, 4, 3, 1, 3 * 128, 1, 128, 0)):
        n_in = gm[0] * gm[1] * gm[2] * gm[3] * gm[4]
        x = rnd(n_in, g=g)
        col, _ = R.im2col_ref(x, gm)
        y = rnd(col.numel(), g=g)
        din, _ = R.col2im_ref(y, gm, n_in)
        lhs, rhs = float((col.reshape(-1) * y.double()).sum()), float((x.double() * din).sum())
        assert abs(lhs - rhs) <= 1e-12 * (1 + abs(lhs))


# ------------------------------------------------------------------------------------ emulations inside the bounds
def _cases():
    """{name: (ratio of the clean emulation, ratio with the planted mistake, case)}: each on a reduced size of a case
    the GPU test runs."""
    g = _g(10)
    out = {}
    # 1, 2: BatchNorm eps, tanh-form GELU'
    C, n = 32, 32 * 200
    bn = _bn(C, g)
    z, dy = rnd(n, g=g, scale=3.0), rnd(n, g=g)
    dbn, e1, dz, e2 = R.bn_gelu_bwd_ref(dy, z, bn, C)
    for m in ("bn_eps", "gelu_tanh"):
        clean = R.emu_bn_gelu_bwd(dy.numpy(), z.numpy(), bn, C)
        bad = R.emu_bn_gelu_bwd(dy.numpy(), z.numpy(), bn, C, m)
        out[m] = (max(worst(torch.tensor(clean[0]), dbn, e1), worst(torch.tensor(clean[1]), dz, e2)),
                  max(worst(torch.tensor(bad[0]), dbn, e1), worst(torch.tensor(bad[1]), dz, e2)), "bn_gelu_bwd C32")
    ref, e = R.bn_scale_ref(dy, bn, C)
    out["bn_eps (bn_scale)"] = (worst(torch.tensor(R.emu_bn_scale_op(dy.numpy(), bn, C)), ref, e),
                                worst(torch.tensor(R.emu_bn_scale_op(dy.numpy(), bn, C, "bn_eps")), ref, e),
                                "bn_scale C32")
    # 3, 4: tr_reduce over Z - 1 parts; the last K tile masked at K (dY^T X over 4099 rows, 7 parts)
    A, B = rnd(9, 4099, g=g), rnd(7, 4099, g=g)
    ref, e, _, _ = R.gemm_ref(A, B, splits=7)
    out["reduce_z_minus_1"] = (worst(torch.tensor(R.emu_gemm(A.numpy(), B.numpy(), 7)), ref, e),
                               worst(torch.tensor(R.emu_gemm(A.numpy(), B.numpy(), 7, "reduce_z_minus_1")), ref, e),
                               "gemm M9 N7 K4099 splits 7")
    out["gemm_mask_at_K"] = (out["reduce_z_minus_1"][0],
                             worst(torch.tensor(R.emu_gemm(A.numpy(), B.numpy(), 7, "gemm_mask_at_K")), ref, e),
                             "gemm M9 N7 K4099 splits 7")
    # 5: colsum lanes all from the part's first row
    A = rnd(1025, 33, g=g)
    ref, e, _, _ = R.colsum_ref(A, splits=3, scale=0.5)
    out["colsum_lane_start"] = (worst(torch.tensor(R.emu_colsum(A.numpy(), 3, 0.5)[0]), ref, e),
                                worst(torch.tensor(R.emu_colsum(A.numpy(), 3, 0.5, "colsum_lane_start")[0]), ref, e),
                                "colsum M1025 N33 splits 3")
    # 6: rms_bwd without its clamped branch (a row of norm 1e-13)
    x = rnd(8, 64, g=g)
    x[3] = 0
    x[4] = x[4] / x[4].norm() * 1e-13
    x[5] = x[5] / x[5].norm() * 1e-12
    gamma, dxn = rnd(64, g=g), rnd(8, 64, g=g)
    _, _, inv, _ = R.rms_fwd_ref(x, gamma)
    inv32 = inv.float()
    ref, e = R.rms_bwd_ref(dxn, x, inv32, gamma)
    args = (dxn.numpy(), x.numpy(), inv32.numpy(), gamma.numpy())
    out["rms_no_clamp"] = (worst(torch.tensor(R.emu_rms_bwd(*args)), ref, e),
                           worst(torch.tensor(R.emu_rms_bwd(*args, "rms_no_clamp")), ref, e), "rms_bwd C64, norm 1e-13")
    # 7, 8: inverse RoPE with +sin; posmode 1 with m % F
    fr = (1.0 / 10000 ** (torch.arange(0, 32, 2).float() / 32)).float()
    for m, (pm, L, F, inv_, M) in (("rope_inverse_plus_sin", (0, 1500, 1, 1, 1600)),
                                   ("rope_pos_mod_F", (1, 17, 16, 0, 16 * 17))):
        qkv = rnd(M, 192, g=g)
        ref, e = R.rope_ref(qkv, fr, L, F, pm, inv_)
        out[m] = (worst(torch.tensor(R.emu_rope(qkv.numpy(), fr.numpy(), L, F, pm, inv_)), ref, e),
                  worst(torch.tensor(R.emu_rope(qkv.numpy(), fr.numpy(), L, F, pm, inv_, m)), ref, e),
                  f"rope posmode {pm} M{M}")
    # 9: dkv without delta
    H, n = 1, 65
    rows = R.seq_rows(2, n, 1, n, 0, 1)
    qkv, dO = rnd(2 * n, 96, g=g), rnd(2 * n, 32, g=g)
    Oref, _, lse, el = R.attn_fwd_ref(qkv, rows, H)
    lse_t = lse.reshape(2, n).reshape(-1, 1)
    delta = (dO.double() * R.heads_back(Oref, rows, H, 2 * n, 0, 32)).sum(-1, keepdim=True)
    _, _, dk, edk, dv, edv = R.attn_bwd_ref(qkv, dO, lse_t.float(), delta.float(), rows, H)
    args = (qkv, dO, lse_t.float(), delta.float(), rows, H)
    ck, cv = R.emu_attn_dkv(*args)
    bk, _ = R.emu_attn_dkv(*args, mistake="dkv_no_delta")
    out["dkv_no_delta"] = (max(worst(ck, dk, edk), worst(cv, dv, edv)), worst(bk, dk, edk), "attn_dkv time n65")
    # 10: lse in log2
    _, _, l2, _ = R.attn_fwd_ref(qkv, rows, H, lse_log2=True)
    out["lse_log2"] = (0.0, worst(l2, lse, el), "attn_fwd time n65")
    # 11: im2col tap t + dt
    gm = (2, 16, 2, 17, 32, 16 * 2 * 17 * 32, 17 * 32, 32, 1)
    x = rnd(2 * 32 * 17 * 32, g=g)
    ref, e = R.im2col_ref(x, gm)
    out["im2col_tap"] = (worst(torch.tensor(R.emu_im2col(x.numpy(), gm)).reshape(ref.shape), ref, e + 0),
                         worst(torch.tensor(R.emu_im2col(x.numpy(), gm, "im2col_tap")).reshape(ref.shape), ref,
                                 e + 0), "im2col conv0 L17 (exact: any difference)")
    # 12: dg without (1 - sg)
    Og, dG = rnd(40, 64, g=g), rnd(40, 64, g=g)
    gl = torch.linspace(-30, 30, 80).float().reshape(40, 2)
    dOr, e0, dg, eg, de, ed = R.gate_bwd_ref(dG, Og, gl)
    c = R.emu_gate_bwd(dG.numpy(), Og.numpy(), gl.numpy())
    b = R.emu_gate_bwd(dG.numpy(), Og.numpy(), gl.numpy(), "dg_no_one_minus")
    out["dg_no_one_minus"] = (max(worst(torch.tensor(c[0]), dOr, e0), worst(torch.tensor(c[1]), dg, eg),
                                  worst(torch.tensor(c[2]), de, ed)), worst(torch.tensor(b[1]), dg, eg),
                              "gate_bwd M40 C64")
    return out


CASES = _cases()


@pytest.mark.parametrize("mistake", sorted(CASES))
def test_emulation_within_bound_and_mistake_exceeds_it(mistake):
    clean, bad, case = CASES[mistake]
    print(f"{mistake:22s} on {case}: clean {clean:.3g} x the bound, with the mistake {bad:.3g}")
    assert clean <= 1.0
    if mistake == "gemm_mask_at_K":
        # tr_gemm_kc rounds every part to whole 16-column tiles, so no tile of a part but the last straddles its end:
        # masking at K instead of the part's end changes nothing, and the emulation is exactly the clean one
        assert bad == clean
        return
    assert bad > 1.0


def test_end_to_end_bound_misses_the_eps_mistake_but_not_the_tanh_one():
    """The BatchNorm-eps and tanh-GELU' mistakes against test_gpu_train.py's normwise 1e-4: the layer's backward
    (dz of a BatchNorm + GELU, and the 1-d BatchNorm's dx) from the emulation with the mistake, against float64."""
    g = _g(20)
    C, n = 32, 32 * 3000
    bn = _bn(C, g)
    z, dy = rnd(n, g=g, scale=2.0), rnd(n, g=g)
    _, _, dz, _ = R.bn_gelu_bwd_ref(dy, z, bn, C)
    rel = {}
    for m in ("bn_eps", "gelu_tanh"):
        got = torch.tensor(R.emu_bn_gelu_bwd(dy.numpy(), z.numpy(), bn, C, m)[1]).double()
        rel[m] = float((got - dz).norm() / dz.norm())
        print(f"{m}: normwise relative error of dz {rel[m]:.3g} against the end-to-end 1e-4")
    assert rel["bn_eps"] < 1e-4     # below the end-to-end check; the unit bound sees it
    assert rel["gelu_tanh"] > 1e-4  # the end-to-end check sees it where this layer sets the gradient's norm
