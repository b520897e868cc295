"""Float64 restatements of the training kernels (csrc/kernels_train.cu, run alone through bt_debug_train_kernel), the
elementwise bounds their unit tests hold them to, and fp32 emulations of the kernels in numpy with a switch for each
planted mistake.  Shared by tests/test_gpu_train_kernels.py (runs the cases on the device) and
tests/test_cpu_train_kernels.py (ties the restatements to float64 autograd of the oracle, and the bounds to the
emulations, with and without mistakes).

Every restatement is written on the kernel's fp32 operands, converted exactly to float64.  Bounds are first order in
u = 2^-24.  Every multiply and add is charged as its own rounding, so a bound holds whether or not nvcc contracted an
expression into an FMA.  The library is built without -use_fast_math (_lib.NVCC_FLAGS), so the CUDA math library's
ulp figures apply: expf, erff 2 ulp, logf 1 ulp, sinf / cosf 2 ulp over the full range, sqrtf and division correctly
rounded.  Each bound is multiplied by SAFE = 1 + 2^-10 for the second-order terms and gets TINY = 2^-140 for
subnormal flushes.

gemm       C = sum_k A(m, k) B(n, k) (+ bias) (+ resid); gelu_out = GELU(C) (exact erf).  tr_gemm runs one fmaf chain per
           K part of kc columns (tiles of 16; masked columns are exact zeros), tr_reduce adds the Z parts from 0 and
           scales.  With S = sum_k |A B|: e = (kc + Z + 3) u (S + |bias| + |resid|) (+ u |C| for a scale).  gelu_out:
           GELU_SLOPE e + 2^-21 |C| + u |GELU(C)| (erff 2 ulp, the product x / sqrt 2, 1 + erf, the two products).
colsum     out[n] = scale sum_m A[m, n] (B[m, n]) (rs[m]).  A lane sums ceil(rows / 8) of its part's rows, eight lanes
           are added in shared memory, tr_reduce adds the Z parts and scales: with T = sum_m |terms|,
           e = (ceil(rows / 8) + 8 + Z + 3) u T + u |out|  (the 3: the products by B and rs and the scale).
reduce     out = scale sum_z part[z]: e = Z u sum_z |part| + u |out|.
rms_fwd    inv = 1 / max(||x||, 1e-12); xn = x inv sqrt(C) gamma.  ss: lanes of C/32 fmaf terms and five shuffles,
           K = C/32 + 5 roundings of sum x^2; sqrtf halves it and adds u; the clamp constant 1e-12f is u relative off;
           the division adds u: inv is (K/2 + 3) u relative off.  xn: three more products and sqrtf(C) (u each).
rms_bwd    du = dxn sqrt(C) gamma, u_ = x inv; dx = inv (du - u_ (u_ . du)), or du inv where the norm is clamped (the
           derivative of x / 1e-12; F.normalize's gradient there).  Bound from the float64 terms: the dot's
           K = C/32 + 5 + 3 roundings of sum |u_ du|, the products (5 u relative each side), the cancellation
           du - u_ dot charged absolutely, and inv's relative error taken from rms_fwd's bound (inv is an input: the
           restatement reads the kernel's own fp32 inv, as the training pass does).  dres with add: one more add.
bn_*       scale = w / sqrt(rv + 1e-5), shift = b - rm scale (3 u relative in scale: the add, sqrtf, the division).
           bn_gelu_fwd y = GELU(z scale + shift); bn_gelu_bwd dbn = dy GELU'(x), dz = dbn scale; bn_grads dw =
           (S_gz - rm S_g) / sqrt(rv + eps), db = S_g; bn_scale dx = g scale.  GELU'(x) = Phi(x) + x phi(x) from erff and
           expf: its error is GELU2_SLOPE e_x (max |GELU''| = 0.7979 at 0) + u-terms of its five operations, with the
           erff and expf ulps on Phi and phi (2^-22 relative each).
gelu_bwd   dh = da GELU'(h): the GELU' term of bn_gelu_bwd at x = h.
im2col     exact without the BatchNorm (a gather); with it: v scale + shift, a multiply-add pair on an inexact scale.
col2im     at most 3 adds: e = 3 u sum |terms|; also the float64 adjoint of im2col.
concat     exact (a permutation); head_fwd / head_bwd: one add in sum-head mode, else exact.
rope       the angle is fl32(pos fl32(freq)) (rotary_embedding_torch forms it in fp32), rotated in float64.  cosf / sinf
           2 ulp (2^-22 relative + 2^-149), then two products and an add per output: e = 2^-22 (|x0 c| + |x1 s|) + 3 u
           (|x0 c| + |x1 s|) ... per component.
gate_fwd   G = O sigmoid(g): sigmoidf_ = 1 / (1 + expf(-g)): expf 2 ulp, the add and the division: 4 u relative; then
           the product.
gate_bwd   dO = dG sg; dg = sg (1 - sg) sum_d dG O; delta = sum_d dO O: 32-term fmaf chains (32 u of the magnitudes),
           sg's 4 u, the products and 1 - sg (cancellation charged absolutely: u + e_sg).
attention  forward: attention_reference.softmax_ref with one key per online-softmax step (this kernel's schedule) on
           the SIMT score model (q scaled in fp32, 32-term fmaf chains, expf); lse = max + logf(l) in nats, off by the
           max's score error, l's relative error, logf's ulp and the final add.
dq, dkv    ds_ij = p_ij (dp_ij - delta_i), p_ij = expf(a_ij - lse_i); lse and delta are inputs (the tests give them
           in float64 rounded to fp32).  Per term: a's 32-term chain (32 u sum |q k| s), the subtraction and expf
           (p relative error e_p = e_a + u |a - lse| + 2^-22), dp's 32-term chain (32 u sum |dO v|), the cancellation
           dp - delta charged absolutely (u |dp - delta|), and the product; then the sum over the other side's
           positions: a fmaf chain of n terms (n u of the magnitudes), and the final scale (u).
"""
import math

import numpy as np
import torch

from numerics import (EXPF_REL, GELU2_SLOPE, GELU_SLOPE, LOG2E, REL_2ULP, S_F32, U, f32, f64, fma_f32, gelu_erf,
                      rope_positions)

SAFE = 1.0 + 2.0**-10
TINY = 2.0**-140
BN_EPS = 1e-5
KERNELS = {  # op -> the kernels it launches
    "gemm": ("tr_gemm_kernel", "tr_reduce_kernel"), "reduce": ("tr_reduce_kernel",),
    "colsum": ("tr_colsum_kernel", "tr_reduce_kernel"), "rms_fwd": ("tr_rms_fwd_kernel",),
    "rms_bwd": ("tr_rms_bwd_kernel",), "bn_gelu_fwd": ("tr_bn_gelu_fwd_kernel",),
    "bn_gelu_bwd": ("tr_bn_gelu_bwd_kernel",), "bn_grads": ("tr_bn_grads_kernel",), "bn_scale": ("tr_bn_scale_kernel",),
    "gelu_bwd": ("tr_gelu_bwd_kernel",), "im2col": ("tr_im2col_kernel",), "col2im": ("tr_col2im_kernel",),
    "concat": ("tr_concat_kernel",), "rope": ("tr_rope_kernel",), "gate_fwd": ("tr_gate_fwd_kernel",),
    "gate_bwd": ("tr_gate_bwd_kernel",), "head_fwd": ("tr_head_fwd_kernel",), "head_bwd": ("tr_head_bwd_kernel",),
    "attn_fwd": ("tr_attn_fwd_kernel",), "attn_dq": ("tr_attn_dq_kernel",), "attn_dkv": ("tr_attn_dkv_kernel",),
}


# ------------------------------------------------------------------------------------ restatements and bounds
def gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def gelu_grad_err(x, ex):
    """Bound on |gelu_grad_kernel(x^) - gelu_grad(x)| with |x^ - x| <= ex: the slope times ex, plus the roundings of
    cdf = 0.5 (1 + erff(x c)) (erff 2 ulp, x c u, 1 + . u) and pdf = k expf(-0.5 x x) (expf 2 ulp, 3 products), the
    product x pdf and the sum."""
    ax = x.abs()
    cdf = 0.5 * (1 + torch.erf(x / math.sqrt(2)))
    pdf = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    e_cdf = 0.5 * (REL_2ULP + U * ax * 2 / math.sqrt(math.pi) * torch.exp(-0.5 * x * x) / math.sqrt(2) + U * (1 + cdf))
    e_pdf = pdf * (REL_2ULP + 4 * U + U * x * x)  # expf 2 ulp; the argument's 2 products (u x^2 absolute); k, the product
    xp = ax * pdf
    return GELU2_SLOPE * ex + e_cdf + ax * e_pdf + U * xp + U * (cdf + xp) + U * (cdf + xp).abs()


def gemm_kc(K, splits):
    return ((K + splits - 1) // splits + 15) // 16 * 16


def gemm_ref(A, B, bias=None, resid=None, splits=1, scale=1.0):
    """(C, bound, gelu(C), gelu bound) of C[m, n] = scale sum_k A[m, k] B[n, k] (+ bias[n]) (+ resid[m, n])."""
    A, B = f64(A), f64(B)
    K = A.shape[1]
    kc = min(gemm_kc(K, splits), K)
    Z = -(-K // gemm_kc(K, splits))
    C = (A @ B.T) * scale
    S = (A.abs() @ B.abs().T) * abs(scale)
    if bias is not None:
        C, S = C + f64(bias), S + f64(bias).abs()
    if resid is not None:
        C, S = C + f64(resid), S + f64(resid).abs()
    e = SAFE * ((kc + (Z if Z > 1 else 0) + 3) * U * S + U * C.abs()) + TINY
    g = gelu_erf(C)
    eg = SAFE * (GELU_SLOPE * e + 2.0**-21 * C.abs() + U * g.abs()) + TINY
    return C, e, g, eg


def colsum_parts(M, splits):
    rps = -(-M // splits)
    return rps, -(-M // rps)


def colsum_ref(A, B=None, rs=None, splits=1, scale=1.0):
    """(out, bound, parts, parts bound) of out[n] = scale sum_m A[m, n] (B[m, n]) (rs[m]) over `splits` row ranges."""
    T = f64(A)
    if B is not None:
        T = T * f64(B)
    if rs is not None:
        T = T * f64(rs)[:, None]
    M = T.shape[0]
    rps, Z = colsum_parts(M, splits)
    parts = torch.stack([T[z * rps:(z + 1) * rps].sum(0) for z in range(Z)])
    pabs = torch.stack([T[z * rps:(z + 1) * rps].abs().sum(0) for z in range(Z)])
    lane = -(-rps // 8)
    ep = SAFE * (lane + 8 + 2) * U * pabs + TINY
    out = scale * parts.sum(0)
    e = SAFE * abs(scale) * ((lane + 8 + 2 + Z) * U * pabs.sum(0)) + U * out.abs() + TINY
    return out, e, parts, ep


def reduce_ref(part, scale=1.0):
    P = f64(part)
    out = scale * P.sum(0)
    return out, SAFE * (P.shape[0] * U * abs(scale) * P.abs().sum(0) + U * out.abs()) + TINY


def rms_fwd_ref(x, gamma):
    """(xn, bound, inv, inv bound) of F.normalize(x) sqrt(C) gamma and inv = 1 / max(||x||, 1e-12)."""
    x, gamma = f64(x), f64(gamma)
    C = x.shape[1]
    nrm = x.norm(dim=1)
    den = nrm.clamp_min(f32(1e-12))
    inv = 1.0 / den
    K = C // 32 + (1 if C % 32 else 0) + 5
    rel_inv = (K / 2 + 3) * U
    xn = x * inv[:, None] * math.sqrt(C) * gamma
    e = SAFE * xn.abs() * (rel_inv + 4 * U) + TINY
    return xn, e, inv, SAFE * inv * rel_inv + TINY


def rms_bwd_ref(dxn, x, inv, gamma, dres=None):
    """(dx, bound) of the RMSNorm input gradient, read on the kernel's own inv (an fp32 input); clamped rows, where
    ||x|| < 1e-12, take du inv.  dres: the gradient already there (add)."""
    dxn, x, inv, gamma = f64(dxn), f64(x), f64(inv), f64(gamma)
    C = x.shape[1]
    sc = math.sqrt(C)
    du = dxn * sc * gamma
    u_ = x * inv[:, None]
    dot = (u_ * du).sum(1, keepdim=True)
    K = C // 32 + (1 if C % 32 else 0) + 5 + 3
    e_dot = (K * U) * (u_ * du).abs().sum(1, keepdim=True)
    nrm = x.norm(dim=1)[:, None]
    clamped = nrm < f32(1e-12)
    inner = du - u_ * dot
    e_inner = 3 * U * du.abs() + (u_ * dot).abs() * 4 * U + u_.abs() * e_dot + U * inner.abs()
    dc, ec = du * inv[:, None], 4 * U * (du * inv[:, None]).abs()
    dn = inv[:, None] * inner
    en = inv[:, None] * e_inner + U * dn.abs()
    dx = torch.where(clamped, dc, dn)
    e = torch.where(clamped, ec, en)
    # within the kernel's rounding of ||x|| of the clamp, either branch may run: the midpoint, and half the gap
    amb = (nrm - f32(1e-12)).abs() <= (K / 2 + 2) * U * nrm
    dx = torch.where(amb, 0.5 * (dc + dn), dx)
    e = torch.where(amb, 0.5 * (dc - dn).abs() + torch.maximum(ec, en), e)
    if dres is not None:
        dx = dx + f64(dres)
        e = e + U * dx.abs()
    return dx, SAFE * e + TINY


def bn_scale_shift(w, b, rm, rv, eps=BN_EPS):
    w, b, rm, rv = f64(w), f64(b), f64(rm), f64(rv)
    s = w / torch.sqrt(rv + f32(eps))
    return s, b - rm * s, 3 * U * s.abs()


def bn_apply(z, bn, c):
    """(x, bound) of x = z scale + (b - rm scale) at channels c: scale's error, the two products, the difference and
    the sum."""
    s, t, es = bn_scale_shift(*bn)
    rm = f64(bn[2])[c]
    x = z * s[c] + t[c]
    ex = (z.abs() + rm.abs()) * es[c] + U * ((z * s[c]).abs() + (rm * s[c]).abs() + t[c].abs() + x.abs())
    return x, ex


def bn_gelu_fwd_ref(z, bn, C):
    z = f64(z)
    x, ex = bn_apply(z, bn, torch.arange(z.numel()) % C)
    y = gelu_erf(x)
    return y, SAFE * (GELU_SLOPE * ex + 2.0**-21 * x.abs() + U * y.abs()) + TINY


def bn_gelu_bwd_ref(dy, z, bn, C):
    """(dbn, bound, dz, bound)."""
    dy, z = f64(dy), f64(z)
    s, t, es = bn_scale_shift(*bn)
    c = torch.arange(z.numel()) % C
    x, ex = bn_apply(z, bn, c)
    gg = gelu_grad(x)
    dbn = dy * gg
    e_dbn = dy.abs() * gelu_grad_err(x, ex) + U * dbn.abs()
    dz = dbn * s[c]
    e_dz = e_dbn * s.abs()[c] + dbn.abs() * es[c] + U * dz.abs()
    return dbn, SAFE * e_dbn + TINY, dz, SAFE * e_dz + TINY


def bn_grads_ref(s_gz, s_g, bn):
    s_gz, s_g = f64(s_gz), f64(s_g)
    rm, rv = f64(bn[2]), f64(bn[3])
    r = torch.sqrt(rv + f32(BN_EPS))
    num = s_gz - rm * s_g
    dw = num / r
    e = (U * (rm * s_g).abs() * 2 + U * num.abs()) / r + dw.abs() * 3 * U
    return dw, SAFE * e + TINY, s_g


def bn_scale_ref(g, bn, C):
    g = f64(g)
    s, _, es = bn_scale_shift(*bn)
    c = torch.arange(g.numel()) % C
    dx = g * s[c]
    return dx, SAFE * (g.abs() * es[c] + U * dx.abs()) + TINY


def gelu_bwd_ref(da, h):
    da, h = f64(da), f64(h)
    dh = da * gelu_grad(h)
    return dh, SAFE * (da.abs() * gelu_grad_err(h, torch.zeros_like(h)) + U * dh.abs()) + TINY


def im2col_ref(inp, g, bn=None, tap=-1):
    """col [B Fo L, C S 3] from the input read through strides g = (B, Fo, S, L, C, sb, sf, st, sc) of a flat array;
    (col, bound).  tap: the time offset of tap dt is dt + tap (the kernels': -1)."""
    B, Fo, S, L, C, sb, sf, st, sc = g
    flat = f64(inp).reshape(-1)
    b = torch.arange(B)[:, None, None, None, None, None]
    fo = torch.arange(Fo)[None, :, None, None, None, None]
    t = torch.arange(L)[None, None, :, None, None, None]
    c = torch.arange(C)[None, None, None, :, None, None]
    df = torch.arange(S)[None, None, None, None, :, None]
    dt = torch.arange(3)[None, None, None, None, None, :]
    f = fo * S + df
    ti = t + dt + tap
    ok = (ti >= 0) & (ti < L)
    idx = b * sb + f * sf + ti.clamp(0, L - 1) * st + c * sc
    v = flat[idx]
    e = torch.zeros_like(v)
    if bn is not None:
        v, e = bn_apply(v, bn, f.expand_as(v))
    v = torch.where(ok, v, torch.zeros_like(v))
    e = torch.where(ok, e, torch.zeros_like(e))
    return v.reshape(B * Fo * L, C * S * 3), SAFE * e.reshape(B * Fo * L, C * S * 3)


def col2im_ref(dcol, g, n_in):
    """The adjoint of im2col (no BatchNorm) into a flat array of n_in elements (untouched where no input element
    lives: NaN); (din, bound)."""
    B, Fo, S, L, C, sb, sf, st, sc = g
    d = f64(dcol).reshape(B, Fo, L, C, S, 3)
    din = torch.zeros(B, Fo, S, L, C, dtype=torch.float64)
    ab = torch.zeros_like(din)
    for dt in range(3):
        # din(t) += dcol(row t - dt + 1, dt)
        lo, hi = max(0, dt - 1), min(L, L + dt - 1)  # t with 0 <= t - dt + 1 < L
        src = d[:, :, lo - dt + 1:hi - dt + 1, :, :, dt].permute(0, 1, 4, 2, 3)
        din[:, :, :, lo:hi] += src
        ab[:, :, :, lo:hi] += src.abs()
    out = torch.full((n_in,), math.nan, dtype=torch.float64)
    eo = torch.zeros(n_in, dtype=torch.float64)
    b = torch.arange(B)[:, None, None, None, None]
    f = (torch.arange(Fo)[:, None] * S + torch.arange(S)[None, :])[None, :, :, None, None]
    t = torch.arange(L)[None, None, None, :, None]
    c = torch.arange(C)[None, None, None, None, :]
    idx = (b * sb + f * sf + t * st + c * sc).reshape(-1)
    out[idx] = din.reshape(-1)
    eo[idx] = SAFE * 2 * U * ab.reshape(-1)
    return out, eo


def concat_ref(src, B, F, L, C, backward):
    s = f64(src)
    if backward:  # rows [B, L, C F] -> tokens [B, F, L, C]
        return s.reshape(B, L, C, F).permute(0, 3, 1, 2).reshape(-1)
    return s.reshape(B, F, L, C).permute(0, 2, 3, 1).reshape(-1)


def rope_ref(qkv, freqs, L, F, posmode, inverse):
    """(qkv', bound) of rotary_embedding_torch's rotation (angle fl32(pos fl32(freq))) of the q and k columns of qkv
    [M, 3C] by +angle (inverse: -angle); v is untouched."""
    x = f64(qkv).clone()
    M, C3 = x.shape
    C = C3 // 3
    pos = rope_positions(M, L, F, posmode).float()
    fr = torch.as_tensor(freqs).float()
    cols = torch.arange(2 * C)  # the q columns, then the k columns
    ang = (pos[:, None] * fr[(cols[::2] % 32) // 2][None, :]).double()  # fp32 product, as the reference forms it
    co, si = torch.cos(ang), torch.sin(ang)
    if inverse:
        si = -si
    x0, x1 = x[:, 0:2 * C:2], x[:, 1:2 * C:2]
    y0, y1 = x0 * co - x1 * si, x1 * co + x0 * si
    t0, t1 = (x0 * co).abs() + (x1 * si).abs(), (x1 * co).abs() + (x0 * si).abs()
    e = torch.zeros_like(x)
    x[:, 0:2 * C:2], x[:, 1:2 * C:2] = y0, y1
    e[:, 0:2 * C:2] = SAFE * ((REL_2ULP + 3 * U) * t0) + 2.0**-148 * (x0.abs() + x1.abs())
    e[:, 1:2 * C:2] = SAFE * ((REL_2ULP + 3 * U) * t1) + 2.0**-148 * (x0.abs() + x1.abs())
    return x, e


def sigmoid_err(g):
    sg = torch.sigmoid(g)
    # expf(-g) 2 ulp relative, 1 + e and the division: the relative error of 1 / (1 + e) is (e / (1 + e)) 2^-22 + 2 u
    return sg, sg * ((1 - sg) * REL_2ULP + 2 * U)


def gate_fwd_ref(O, g):
    O, g = f64(O), f64(g)
    M, C = O.shape
    sg, es = sigmoid_err(g)
    sgx = sg.repeat_interleave(32, 1)
    G = O * sgx
    return G, SAFE * (O.abs() * es.repeat_interleave(32, 1) + U * G.abs()) + TINY


def gate_bwd_ref(dG, O, g):
    """(dO, bound, dg, bound, delta, bound) from dG [M, C], O [M, C], g [M, C / 32]."""
    dG, O, g = f64(dG), f64(O), f64(g)
    M, C = O.shape
    H = C // 32
    sg, es = sigmoid_err(g)
    sgx, esx = sg.repeat_interleave(32, 1), es.repeat_interleave(32, 1)
    dO = dG * sgx
    e_dO = dG.abs() * esx + U * dO.abs()
    pr = (dG * O).reshape(M, H, 32)
    s = pr.sum(-1)
    e_s = 32 * U * pr.abs().sum(-1)
    one = 1 - sg
    e_one = es + U * one.abs()
    fac = sg * one
    e_fac = es * one.abs() + sg * e_one + U * fac.abs()
    dg = s * fac
    e_dg = e_s * fac.abs() + s.abs() * e_fac + 2 * U * dg.abs()
    dOO = (dO * O).reshape(M, H, 32)
    delta = dOO.sum(-1)
    e_delta = 32 * U * dOO.abs().sum(-1) + (e_dO * O.abs()).reshape(M, H, 32).sum(-1)
    return dO, SAFE * e_dO + TINY, dg, SAFE * e_dg + TINY, delta, SAFE * e_delta + TINY


def head_fwd_ref(o, sum_head):
    o = f64(o).reshape(-1, 2)
    beat = o[:, 0] + o[:, 1] if sum_head else o[:, 0]
    return beat, o[:, 1]


def head_bwd_ref(dbeat, ddown, sum_head):
    db, dd = f64(dbeat), f64(ddown)
    return torch.stack([db, dd + db if sum_head else dd], 1).reshape(-1)


def seq_rows(seqs, n, seq_in, s_out, s_in, s_pos):
    """[seqs, n] token rows of the TrSeqs layout."""
    s = torch.arange(seqs)[:, None]
    i = torch.arange(n)[None, :]
    return (s // seq_in) * s_out + (s % seq_in) * s_in + i * s_pos


def _heads(t, rows, H, off, width):
    """[seqs * H, n, 32] of the `off` block (of `width` heads' columns) of a row-major array at token rows."""
    seqs, n = rows.shape
    x = t[rows.reshape(-1)][:, off:off + width].reshape(seqs, n, H, 32)
    return x.permute(0, 2, 1, 3).reshape(seqs * H, n, 32)


def attn_fwd_ref(qkv, rows, H, lse_log2=False):
    """(O, bound, lse, lse bound) [seqs * H, n, 32] / [seqs * H, n] of the forward over sequences `rows` [seqs, n]."""
    from attention_reference import softmax_ref

    C = 32 * H
    t = f64(qkv)
    q = (_heads(t, rows, H, 0, C).float() * torch.tensor(S_F32, dtype=torch.float32)).double()
    k, v = _heads(t, rows, H, C, C), _heads(t, rows, H, 2 * C, C)
    G, n, _ = q.shape
    T2 = LOG2E * (q @ k.transpose(1, 2))
    E2 = 32 * U * (q.abs() @ k.abs().transpose(1, 2)) * LOG2E
    valid = torch.ones(G, n, dtype=torch.bool)
    nk = torch.full((G,), n, dtype=torch.float64)
    ref, err, _, _ = softmax_ref(T2, E2, valid, v, torch.ones(G, n, dtype=torch.float64), step=1,
                                 exp_rel=lambda x, e: torch.full_like(x, EXPF_REL), alpha_rel=EXPF_REL + U, sub_ops=1,
                                 p_dt=None, n_sum=nk, pv_error=lambda s, nnz: nk[:, None, None] * U * s, out_dt=None,
                                 n_pad=0)
    a = T2 / LOG2E
    lse = torch.logsumexp(a, -1)
    mx = a.amax(-1)
    l = torch.exp(a - mx[..., None]).sum(-1)
    e_max = (E2 / LOG2E).amax(-1)
    # l's relative error: each p_j off by expf and its argument (e_max + the key's score error + u |a - m|), plus the
    # running rescales (expf per step) and one add per key
    e_l = (torch.exp(a - mx[..., None]) * (EXPF_REL * 2 + U * (a - mx[..., None]).abs() + 2 * e_max[..., None]
                                           + (E2 / LOG2E))).sum(-1) / l + n * (EXPF_REL + 2 * U)
    e_lse = SAFE * (e_max + e_l + 2.0**-23 * torch.log(l).abs() + U * lse.abs() + 2 * U * mx.abs()) + TINY
    if lse_log2:
        lse = lse / math.log(2)
    return ref, err, lse, e_lse


def attn_bwd_ref(qkv, dO, lse, delta, rows, H):
    """(dq, dq bound, dk, dk bound, dv, dv bound) [seqs * H, n, 32] of the flash backward read on the given lse and
    delta (fp32 inputs, [tokens, H]), over sequences `rows`."""
    C = 32 * H
    t, d = f64(qkv), f64(dO)
    q, k, v = _heads(t, rows, H, 0, C), _heads(t, rows, H, C, C), _heads(t, rows, H, 2 * C, C)
    do = _heads(d, rows, H, 0, C)
    seqs, n = rows.shape
    L_ = f64(lse)[rows.reshape(-1)].reshape(seqs, n, H).permute(0, 2, 1).reshape(seqs * H, n)
    D_ = f64(delta)[rows.reshape(-1)].reshape(seqs, n, H).permute(0, 2, 1).reshape(seqs * H, n)
    a = S_F32 * (q @ k.transpose(1, 2))  # the kernels scale q (dq) or the score (dkv) by fp32(1 / sqrt 32)
    e_a = (32 + 2) * U * S_F32 * (q.abs() @ k.abs().transpose(1, 2))
    x = a - L_[..., None]
    p = torch.exp(x)
    e_p = p * (e_a + U * x.abs() + REL_2ULP)
    dp = do @ v.transpose(1, 2)
    e_dp = 32 * U * (do.abs() @ v.abs().transpose(1, 2))
    diff = dp - D_[..., None]
    e_diff = e_dp + U * diff.abs()
    ds = p * diff
    e_ds = e_p * diff.abs() + p * e_diff + U * ds.abs()
    dq = S_F32 * (ds @ k)
    e_dq = S_F32 * (e_ds @ k.abs() + (n + 1) * U * (ds.abs() @ k.abs()))
    dk = S_F32 * (ds.transpose(1, 2) @ q)
    e_dk = S_F32 * (e_ds.transpose(1, 2) @ q.abs() + (n + 1) * U * (ds.abs().transpose(1, 2) @ q.abs()))
    dv = p.transpose(1, 2) @ do
    e_dv = e_p.transpose(1, 2) @ do.abs() + n * U * (p.transpose(1, 2) @ do.abs())
    return (dq, SAFE * e_dq + TINY, dk, SAFE * e_dk + TINY, dv, SAFE * e_dv + TINY)


def heads_back(x, rows, H, n_rows, off, width, base=None):
    """Scatter [seqs * H, n, 32] back into the `off` block of a [n_rows, width...] float64 array (NaN elsewhere)."""
    seqs, n = rows.shape
    out = base if base is not None else torch.full((n_rows, width), math.nan, dtype=torch.float64)
    out[rows.reshape(-1), off:off + 32 * H] = x.reshape(seqs, H, n, 32).permute(0, 2, 1, 3).reshape(seqs * n, 32 * H)
    return out


# ------------------------------------------------------------------------------------ fp32 emulations
# numpy fp32 in the kernels' operation order (fmaf: numerics.fma_f32).  `mistake` plants one single-line error.
F = np.float32


def emu_bn_scale(w, rv, mistake=None):
    eps = F(0) if mistake == "bn_eps" else F(1e-5)
    return (w / np.sqrt(rv + eps)).astype(F)


def emu_gelu_grad(x, mistake=None):
    x = x.astype(F)
    if mistake == "gelu_tanh":
        k = F(math.sqrt(2 / math.pi))
        inner = k * (x + F(0.044715) * x * x * x)
        th = np.tanh(inner).astype(F)
        return (F(0.5) * (1 + th) + F(0.5) * x * (1 - th * th) * k * (1 + F(3 * 0.044715) * x * x)).astype(F)
    from scipy.special import erf

    cdf = F(0.5) * (F(1) + erf((x * F(0.70710678118654752440)).astype(np.float64)).astype(F))
    pdf = F(0.3989422804014327) * np.exp((F(-0.5) * x * x).astype(np.float64)).astype(F)
    return (cdf + x * pdf).astype(F)


def emu_bn_gelu_bwd(dy, z, bn, C, mistake=None):
    w, b, rm, rv = (np.asarray(a, F) for a in bn)
    s = emu_bn_scale(w, rv, mistake)
    c = np.arange(z.size) % C
    x = (z * s[c] + (b[c] - rm[c] * s[c])).astype(F)
    g = (dy * emu_gelu_grad(x, mistake)).astype(F)
    return g, (g * s[c]).astype(F)


def emu_bn_scale_op(g, bn, C, mistake=None):
    w, b, rm, rv = (np.asarray(a, F) for a in bn)
    s = emu_bn_scale(w, rv, mistake)
    return (g * s[np.arange(g.size) % C]).astype(F)


def emu_gemm(A, B, splits=1, mistake=None):
    """tr_gemm (+ tr_reduce) of C = A B^T: one fmaf chain per K part, 16-wide tiles."""
    A, B = np.asarray(A, F), np.asarray(B, F)
    M, K = A.shape
    kc = gemm_kc(K, splits)
    Z = -(-K // kc)
    parts = []
    for z in range(Z):
        kb, ke = z * kc, min(K, z * kc + kc)
        acc = np.zeros((M, B.shape[0]), F)
        for k0 in range(kb, ke, 16):
            for k in range(k0, k0 + 16):
                lim = K if mistake == "gemm_mask_at_K" else ke
                if k < lim:
                    acc = fma_f32(A[:, k:k + 1], B[:, k][None, :], acc)
        parts.append(acc)
    return emu_reduce(np.stack(parts), 1.0, mistake) if Z > 1 else parts[0]


def emu_reduce(part, scale, mistake=None):
    Z = part.shape[0] - (1 if mistake == "reduce_z_minus_1" else 0)
    s = np.zeros(part.shape[1:], F)
    for z in range(Z):
        s = (s + part[z]).astype(F)
    return (s * F(scale)).astype(F)


def emu_colsum(A, splits, scale=1.0, mistake=None):
    A = np.asarray(A, F)
    M, N = A.shape
    rps, Z = colsum_parts(M, splits)
    parts = np.zeros((Z, N), F)
    for z in range(Z):
        r0, r1 = z * rps, min(M, z * rps + rps)
        red = np.zeros((8, N), F)
        for ty in range(8):
            start = r0 if mistake == "colsum_lane_start" else r0 + ty
            s = np.zeros(N, F)
            for m in range(start, r1, 8):
                s = (s + A[m]).astype(F)
            red[ty] = s
        t = np.zeros(N, F)
        for i in range(8):
            t = (t + red[i]).astype(F)
        parts[z] = t
    return emu_reduce(parts, scale), parts


def emu_rms_bwd(dxn, x, inv, gamma, mistake=None):
    dxn, x, inv, gamma = (np.asarray(a, F) for a in (dxn, x, inv, gamma))
    C = x.shape[1]
    sc = F(np.sqrt(F(C)))
    du = (dxn * sc * gamma).astype(F)
    ss = (x.astype(np.float64) ** 2).sum(1).astype(F)
    dot = ((x * inv[:, None]).astype(F).astype(np.float64) * du).sum(1).astype(F)
    clamped = np.sqrt(ss) < F(1e-12)
    if mistake == "rms_no_clamp":
        clamped = np.zeros_like(clamped)
    full = (inv[:, None] * (du - (x * inv[:, None]).astype(F) * dot[:, None]).astype(F)).astype(F)
    return np.where(clamped[:, None], (du * inv[:, None]).astype(F), full)


def emu_rope(qkv, freqs, L, Fq, posmode, inverse, mistake=None):
    x = np.asarray(qkv, F).copy()
    M, C3 = x.shape
    C = C3 // 3
    m = np.arange(M)
    pos = m % L if posmode == 0 else ((m % Fq) if mistake == "rope_pos_mod_F" else (m // L) % Fq)
    p = np.arange(C)
    col = np.where(p < C // 2, 2 * p, C + 2 * (p - C // 2))
    ang = (pos[:, None].astype(F) * np.asarray(freqs, F)[(col % 32) // 2][None, :]).astype(F)
    co, si = np.cos(ang.astype(np.float64)).astype(F), np.sin(ang.astype(np.float64)).astype(F)
    if inverse and mistake != "rope_inverse_plus_sin":
        si = -si
    x0, x1 = x[:, col].copy(), x[:, col + 1].copy()
    x[:, col] = (x0 * co - x1 * si).astype(F)
    x[:, col + 1] = (x1 * co + x0 * si).astype(F)
    return x


def emu_im2col(inp, g, mistake=None):
    return im2col_ref(np.asarray(inp, F), g, tap=0 if mistake == "im2col_tap" else -1)[0].float().numpy()


def emu_gate_bwd(dG, O, g, mistake=None):
    dG, O, g = (np.asarray(a, F) for a in (dG, O, g))
    M, C = O.shape
    sg = (F(1) / (F(1) + np.exp(-g.astype(np.float64)).astype(F))).astype(F)
    s = (dG.astype(np.float64) * O).reshape(M, C // 32, 32).sum(-1).astype(F)
    fac = (sg * (F(1) - sg)).astype(F) if mistake != "dg_no_one_minus" else sg
    dO = (dG * np.repeat(sg, 32, 1)).astype(F)
    delta = (dO.astype(np.float64) * O).reshape(M, C // 32, 32).sum(-1).astype(F)
    return dO, (s * fac).astype(F), delta


def emu_attn_dkv(qkv, dO, lse, delta, rows, H, mistake=None):
    """dk, dv [seqs * H, n, 32] in fp32 with fp64-accumulated dot products (each rounded once)."""
    C = 32 * H
    t, d = torch.as_tensor(qkv).double(), torch.as_tensor(dO).double()
    q, k, v = _heads(t, rows, H, 0, C), _heads(t, rows, H, C, C), _heads(t, rows, H, 2 * C, C)
    do = _heads(d, rows, H, 0, C)
    seqs, n = rows.shape
    L_ = torch.as_tensor(lse).double()[rows.reshape(-1)].reshape(seqs, n, H).permute(0, 2, 1).reshape(seqs * H, n)
    D_ = torch.as_tensor(delta).double()[rows.reshape(-1)].reshape(seqs, n, H).permute(0, 2, 1).reshape(seqs * H, n)
    if mistake == "dkv_no_delta":
        D_ = torch.zeros_like(D_)
    a = (q @ k.transpose(1, 2)).float().double()
    p = torch.exp((a * S_F32).float().double() - L_[..., None]).float().double()
    dp = (do @ v.transpose(1, 2)).float().double()
    ds = (p * (dp - D_[..., None]).float().double()).float().double()
    dk = ((ds.transpose(1, 2) @ q).float().double() * S_F32).float()
    dv = (p.transpose(1, 2) @ do).float()
    return dk, dv
