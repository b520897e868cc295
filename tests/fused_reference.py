"""Float64 restatements of the frontend's row kernels and the elementwise bounds their unit tests hold them to:
norm_kernel<TAct, C> (bt_debug_norm), fused_qkv_kernel<C> (bt_debug_fused_qkv) and fused_ff_kernel<C, OP>
(bt_debug_fused_ff).  Shared by tests/test_gpu_fused.py (runs the cases) and tests/test_cpu_fused_reference.py (ties
the restatements to the oracle, the bounds to a CPU emulation of the kernels and the instantiations to the library).

Each result is written from the definition of the operation, with the 16-bit rounding points the kernel has.
round16 is the activation type (rnd(t, None): no rounding, the reference block itself):
  norm : u = x / max(||x||, 1e-12); gates = sigmoid(u . wg[h] + bg[h]) from the unrounded u
  qkv  : u16 = round16(u), acc = u16 round16(Wqkv)^T; RoPE on the q and k columns at position m % L (posmode 0) or
         (m / L) % F (posmode 1); q times qscale; the result rounded to 16 bits; gates as for norm
  ff   : x' = x (+ round16(O) round16(Wo)^T), u16 = round16(normalize(x')), h16 = round16(gelu_tanh(u16 W1^T + b1)),
         y = x' + b2 + h16 round16(W2)^T; the 16-bit copy is round16(y)

Bounds, elementwise and in float64 from the data, with the error model of tests/numerics.py.  A value the kernel
rounds to 16 bits is off by rounding_error(v, d) of round16(v) when its fp32 value is within d of v; each rounded
intermediate carries that error to first order into the products after it.
ACC = GEMM_ACC_TOL_H16 x (1 + |value|) is the stated fp32 accumulation error of one tensor-core product
(numerics.py).  The fused FFN, whose output is fp32 and whose products are short, uses the derived form
mma_error(K, s) = 2 K 2^-23 s, s = |c| + sum_k |a_k b_k| (numerics.mma_error).  An fp32 addition outside the MMA adds
2^-24 of its result (F32_ADD).
  u    : d_u = norm_rel(C) |u| (the fp32 normalisation, see norm); with the out-projection in front, x' is off by
         e_x and d_u = norm_rel(C) |u| + (e_x + |u| ||e_x||) / ||x'|| (first order);  e_u = rounding_error(u, d_u)
  ff   : e_x = mma_error(C, |x| + |O16| |Wo16|^T)                              (out-projection, x' = x + O16 Wo16^T)
         e_p = |W1| e_u + mma_error(C, |u16| |W1|^T) + 2^-24 |p|               p = u16 W1^T + b1
         d_h = GELU_SLOPE e_p + 0.5 |p| TANH_APPROX_TOL + 2^-21 (|h| + |p|)    h = gelu_tanh(p); tanh.approx.f32
                                                                                and the fp32 arithmetic around it
         e_h = rounding_error(h, d_h)
         bound(y) = |W2| e_h + mma_error(4C, |x' + b2| + |h16| |W2|^T) + 2^-24 |x' + b2|  (+ e_x)
         the 16-bit copy equals round16 of the fp32 y the kernel stored, bitwise: both come from one accumulator
  qkv  : e_a = |Wqkv| e_u + ACC (1 + |acc|); RoPE mixes the two columns of a pair with |cos| + |sin| <= sqrt(2):
         e = sqrt(2) max(e_a of the pair) |qscale| on q and k, e_a on v; bound = e + ulp(round16(ref))
  norm : the fp32 norm factor has relative error <= (C/2 + 2) 2^-24 (sum of C squares, sqrtf, division), the product
         one more 2^-24: norm_rel(C) = (C/2 + 3) 2^-24 of |u| (+ 2^-126, so that a zero row has a bound); the 16-bit
         output adds one ulp of round16(u)
  gates: GATES_TOL (the fp32 sigmoid) + 1/4 (sigmoid slope) x (C + 4) 2^-24 sum_i |u_i wg_i| (u's relative error and
         the fp32 dot product)
"""
import math

import torch

from numerics import (F32_ADD, GATES_TOL, GELU_SLOPE, GEMM_ACC_TOL_H16, TANH_APPROX_TOL, U, gelu_tanh, mma_error,
                      normalize, rnd, rope_positions, rope_ref, rounding_error, ulp16)

ACC = GEMM_ACC_TOL_H16
NORM_CS = (32, 64, 128, 256, 512, 1024)  # the BT_NORM_CASE widths of norm_kernel


def norm_error(x, e_x=None):
    """Bound on |u_kernel - u| for u = normalize(x) in fp32, when the kernel's x is off by at most e_x (elementwise)."""
    n = x.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    u = x / n
    d = norm_rel(x.shape[1]) * u.abs()
    if e_x is not None:
        d = d + (e_x + u.abs() * e_x.norm(dim=-1, keepdim=True)) / n
    return d


def norm_rel(C):
    return (C / 2 + 3) * U


def gates_ref(u, wg, bg, heads):
    """(gates [M, heads], bound) from the unrounded float64 u."""
    C = u.shape[1]
    g = torch.sigmoid(u @ wg[:heads].T + bg[:heads])
    bound = GATES_TOL + 0.25 * (C + 4) * U * (u.abs() @ wg[:heads].abs().T)
    return g, bound


def norm_ref(x, dt):
    """(ref, bound): the norm of x [M, C] float64 as the ctx of activation type dt (None: fp32) stores it."""
    u = normalize(x)
    bound = norm_rel(x.shape[1]) * u.abs() + 2.0**-126  # + the smallest normal fp32: zero rows give exact zeros
    if dt is None:
        return u, bound
    u16 = rnd(u, dt)
    return u16, bound + ulp16(u16, dt)


def qkv_ref(x, wqkv, wg, bg, cos, sin, L, F, posmode, qscale, dt):
    """(qkv, bound, gates, gates bound) of the fused QKV kernel on float64 x [M, C], wqkv [3C, C], wg [>= heads, C],
    bg [>= heads], RoPE tables cos, sin [positions, 16].  dt None: the unrounded block (no bound)."""
    M, C = x.shape
    u = normalize(x)
    u16, W = rnd(u, dt), rnd(wqkv, dt)
    acc = u16 @ W.T
    pos = rope_positions(M, L, F, posmode, x.device)
    c, s = cos[pos], sin[pos]
    out = acc.clone()
    out[:, :C] = rope_ref(acc[:, :C], c, s) * qscale
    out[:, C : 2 * C] = rope_ref(acc[:, C : 2 * C], c, s)
    g, gb = gates_ref(u, wg, bg, C // 32)
    if dt is None:
        return out, None, g, gb
    e_a = rounding_error(u, norm_error(x), dt) @ W.abs().T + ACC * (1 + acc.abs())
    pair = e_a[:, : 2 * C].view(M, C, 2).amax(-1, keepdim=True).expand(M, C, 2).reshape(M, 2 * C)
    e = e_a.clone()
    e[:, :C] = math.sqrt(2) * pair[:, :C] * abs(qscale)
    e[:, C : 2 * C] = math.sqrt(2) * pair[:, C:]
    out16 = rnd(out, dt)
    return out16, e + ulp16(out16, dt), g, gb


def ff_ref(x, w1, b1, w2, b2, o=None, wout=None, dt=None, gelu=gelu_tanh):
    """(y, bound) of the fused FFN on float64 x [M, C] (+ the out-projection o [M, C] wout [C, C] in front).
    dt None: the unrounded block (no bound; pass gelu=gelu_erf for the reference's GELU)."""
    C = x.shape[1]
    xp, e_x = x, None
    if o is not None:
        O16, Wo = rnd(o, dt), rnd(wout, dt)
        xp = x + O16 @ Wo.T
        e_x = mma_error(C, x.abs() + O16.abs() @ Wo.abs().T) if dt is not None else None
    u = normalize(xp)
    u16, W1, W2 = rnd(u, dt), rnd(w1, dt), rnd(w2, dt)
    p = u16 @ W1.T + b1
    h = gelu(p)
    y = xp + b2 + rnd(h, dt) @ W2.T
    if dt is None:
        return y, None
    W1a, W2a = W1.abs(), W2.abs()
    e_p = rounding_error(u, norm_error(xp, e_x), dt) @ W1a.T + mma_error(C, u16.abs() @ W1a.T) + F32_ADD * p.abs()
    d_h = GELU_SLOPE * e_p + 0.5 * p.abs() * TANH_APPROX_TOL + 2.0**-21 * (h.abs() + p.abs())
    xb2 = (xp + b2).abs()
    bound = rounding_error(h, d_h, dt) @ W2a.T + mma_error(4 * C, xb2 + rnd(h, dt).abs() @ W2a.T) + F32_ADD * xb2
    if e_x is not None:
        bound = bound + e_x
    return y, bound


def norm_rows_per_cta(C):
    """Rows of one norm_kernel CTA: 8 warps of 32 / (C / 4) rows (C < 128) or one row (C >= 128)."""
    return 8 * (32 // (C // 4) if C // 4 < 32 else 1)


# ---- inputs and the case matrix of tests/test_gpu_fused.py
def special_rows(M, C, g, device=None):
    """x [M, C] float64: N(0, 1) rows, except rows m with m % 11 in 3..8: all zero (the 1e-12 clamp), one-hot, norm
    1e-3, norm 1e-8, and two rows of |x| ~ 50 (in the fused FFN the residual passes through the MMA accumulator)."""
    x = torch.randn(M, C, generator=g, dtype=torch.float64, device=device)
    m = torch.arange(M, device=device)[:, None]
    k = m % 11
    one_hot = torch.zeros_like(x)
    one_hot[torch.arange(M, device=device), torch.arange(M, device=device) % C] = 2.5
    x = torch.where(k == 3, 0.0, x)
    x = torch.where(k == 4, one_hot, x)
    for kind, norm in ((5, 1e-3), (6, 1e-8)):
        x = torch.where(k == kind, normalize(x) * norm, x)
    return torch.where((k == 7) | (k == 8), x * 50, x)


def random_weights(C, g, device=None):
    """float64 weights of one frontend attention and FFN of width C, at the scales of the synthetic checkpoints (the
    biases wider, so that a missing bias stands out).  wg and bg have all 32 rows of the padded gates weight."""
    r = lambda *shape: torch.randn(*shape, generator=g, dtype=torch.float64, device=device)
    return dict(w1=r(4 * C, C) / math.sqrt(C), b1=r(4 * C) * 0.5, w2=r(C, 4 * C) / math.sqrt(4 * C), b2=r(C) * 0.5,
                wout=r(C, C) / math.sqrt(C), wqkv=r(3 * C, C) * 1.2 / math.sqrt(C), wg=r(32, C) / math.sqrt(C),
                bg=r(32) * 0.5)


# persistent CTAs per SM of the fused kernels (ff_ctas<C>, qkv_ctas<C> in csrc/kernels_fused.cu)
FF_CTAS = {32: 3, 64: 2}
QKV_CTAS = {32: 4, 64: 2}
WARP_ROWS = 16  # a warp of the fused kernels owns 16 rows at a time
FUSED_WARPS = 8


def grid_stride_m(ctas_per_sm, sms):
    """Rows that make every warp of the persistent grid take 3 groups of 16 rows, plus a ragged 9-row tail."""
    return 3 * WARP_ROWS * FUSED_WARPS * ctas_per_sm * sms + 9


def ff_cases(sms):
    """(C, outproj, xb_out, M) of the fused FFN cases."""
    cs = [(C, op, xb, M) for C in (32, 64) for op in (False, True) for xb in (False, True)
          for M in (1, 15, 16, 17, 104, 4800)]
    cs += [(32, True, True, 2 * 32 * 1500), (64, True, True, 2 * 16 * 1500)]  # the forward pass: 2 chunks of F x 1500
    cs += [(C, op, True, grid_stride_m(FF_CTAS[C], sms)) for C in (32, 64) for op in (False, True)]
    return cs


def qkv_cases(sms):
    """(C, posmode, L, F, qscale, M) of the fused QKV cases: ragged M throughout."""
    from gemm_reference import QSCALE_TIME

    cs = []
    for C in (32, 64):
        cs += [(C, 0, L, 1, QSCALE_TIME, M) for L in (1, 13, 150, 1500) for M in (2 * L + 5, 16 * L + 1)]
        cs += [(C, 1, 13, F, 1.0, 2 * F * 13 + 7) for F in (32, 16, 8)]
        cs += [(C, 1, 150, F, 1.0, 3 * F * 150 - 3) for F in (32, 16, 8)]
        cs += [(C, 0, 1500, 1, QSCALE_TIME, grid_stride_m(QKV_CTAS[C], sms)),
               (C, 1, 150, 32 // (C // 32), 1.0, grid_stride_m(QKV_CTAS[C], sms))]
    return cs


def norm_cases():
    """(C, heads, M) of the norm cases; each runs in both contexts."""
    cs = []
    for C in NORM_CS:
        R = norm_rows_per_cta(C)
        for heads in (0, 1, 2, 4):
            if 32 * heads <= C:
                cs += [(C, heads, M) for M in sorted({1, R - 1, R, R + 1, 3 * 1500 + 5})]
    return cs
