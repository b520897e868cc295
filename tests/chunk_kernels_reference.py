"""Float64 restatements of the three kernels that read the chunk table (ChunkSrc, csrc/bt_kernels.h), the elementwise
bounds their unit tests hold them to, and fp32 emulations of the kernels: stem_kernel (bt_debug_stem),
zero_tail_kernel (bt_debug_zero_tail) and head_kernel (bt_debug_head).  Shared by tests/test_gpu_chunk_kernels.py (runs
the cases on the device) and tests/test_cpu_chunk_kernels.py (ties the restatements to the oracle and the bounds to the
emulations, with and without mistakes).

A chunk is the tuple (frame_base, T, start, out_base, write_lo, write_hi, len) of bt_debug_chunk.  Every restatement is
written on the kernel's fp32 operands (the packed parameters), converted exactly to float64.

stem, per chunk, output [32 f, L, 32 c], time tap tl = t + dt - 1 (dt < 3), frequency tap 4 f + df (df < 4):
  v   = spect[frame_base + start + tl] if 0 <= start + tl < T else 0        (clip padding: zero BEFORE BN1d)
  in  = v bn1_scale + bn1_shift          if 0 <= tl < len else 0            (chunk padding: zero AFTER BN1d)
  a   = bias[c] + sum_{df, dt} in w[c, df, dt];   out = gelu(a) = 0.5 a (1 + erf(a / sqrt 2))   (exact erf)
Bound, first order, u = 2^-24:
  in    one fmaf: e_in = u |in|
  a     a 12-term fmaf chain from the bias: each rounding loses <= u of the running sum, which is at most
        S = |bias| + sum |in w|, so 12 u S; the inputs' errors add sum |w| e_in.  e_a = (12 u S + sum |w| e_in)(1 + 2^-20)
  gelu  |gelu(a^) - gelu(a)| <= GELU_SLOPE e_a (max |gelu'| = 1.1290 at a = sqrt 2); gelu_fast's erf is within E_ERF of
        erf(|a^| / sqrt 2), which moves the output by 0.5 |a^| E_ERF; its final fp32 product and sum add <= 2 u |a^|.
        bound = GELU_SLOPE e_a + (0.5 E_ERF + 2 u)(|a| + e_a) + 2^-148
  E_ERF (erf_error_bound) is the maximum over z >= 0 of the error of gelu_fast's erf(z) (csrc/epilogue.cuh), whose
        terms are:
        - Abramowitz & Stegun 7.1.26 itself: AS_ERF = 1.5e-7;
        - the fp32 rounding of its six coefficients, carried through the polynomial;
        - z = fp32(|x| * fp32(1/sqrt 2)) is 2u off relative: erf'(z) z 2u;
        - t = rcp.approx.ftz(fp32(1 + a z)): RCP_APPROX_REL = 2^-23 (PTX ISA, rcp.approx.f32: at most 1 ulp) + u relative,
          carried through p(t) = sum a_i t^(i+1) as |t p'(t)| e^(-z^2);
        - Horner's fmaf chain on t <= 1: the running error err <- err t + u |partial|, times e^(-z^2);
        - e = ex2.approx.ftz(fp32(fp32(z z) * fp32(-log2 e))): EX2_APPROX_REL = 2^-22 (PTX ISA, ex2.approx.f32: 2 ulp)
          relative, plus 3u of the argument's relative error, which is 3u z^2 relative in e; results below 2^-126 are
          flushed to 0 (p 2^-126);
        - fmaf(-p, e, 1): u.
head, per owned frame t of chunk b, row x = x[b, t] of D:
  o_j = (x . w_j) / max(||x||, 1e-12) + b_j;  beat = o_0 + o_1 (sum_head) or o_0;  down = o_1
Bound: each lane runs a D/32-term fmaf chain of ss = sum x^2, a_j = sum x w_j, and five shuffle additions combine the
lanes: K = D/32 + 5 roundings, each <= u of the sum of magnitudes, so ss is K u relative off and a_j off by
K u sum |x w_j|.  sqrtf halves the first and adds u, the 1e-12f clamp constant is u relative off, the division adds u:
the reciprocal is e_inv = (K/2 + 3) u relative off.  Then the product a_j inv (u) and the bias add (u |o_j|):
  e_j = (K u sum|x w_j| / den + |a_j / den| (e_inv + u) + u |o_j|)(1 + 2^-20) + K 2^-149 / den   (den = max(||x||, 1e-12))
  beat bound e_0 + e_1 + u |o_0 + o_1| (sum_head) or e_0;  down bound e_1.  A zero row is the bias, exactly.
zero_tail: exact.  Rows [len, L) of every plane of a chunk are 0, every other byte keeps its value.
"""
import math

import numpy as np
import torch

from numerics import EX2_APPROX_REL, GELU_SLOPE, LOG2E, RCP_APPROX_REL, U, f32, fma_f32, gelu_erf

AS_ERF = 1.5e-7
AS_P = 0.3275911
AS_A = (0.254829592, -0.284496736, 1.421413741, -1.453152027, 1.061405429)  # a1 .. a5 of A&S 7.1.26
FIELDS = ("frame_base", "T", "start", "out_base", "write_lo", "write_hi", "len")


def erf_error_bound(n=200001, z_max=10.0):
    """E_ERF: the largest error of gelu_fast's erf(z), z >= 0, from the terms in the module docstring (float64 on a
    grid of n points, times 1.01 for what falls between them)."""
    z = np.linspace(0.0, z_max, n)
    t = 1.0 / (1.0 + AS_P * z)
    e = np.exp(-z * z)
    a = np.array(AS_A)
    powers = np.stack([t ** (i + 1) for i in range(5)])
    p = a @ powers
    tdp = (np.arange(1, 6) * a) @ powers  # t p'(t)
    coef = np.abs(np.array([f32(c) for c in AS_A]) - a) @ powers + abs(tdp) * abs(f32(AS_P) - AS_P) / AS_P
    horner_p, err = np.full_like(z, a[4]), np.zeros_like(z)
    for c in a[3::-1]:
        horner_p = horner_p * t + c
        err = err * t + U * np.abs(horner_p)
    err = err * t + U * np.abs(horner_p * t)
    total = (AS_ERF + coef * e + 2.0 / math.sqrt(math.pi) * e * z * 2 * U + np.abs(tdp) * e * (RCP_APPROX_REL + U)
             + err * e + np.abs(p) * e * (EX2_APPROX_REL + 3 * U * z * z) + np.abs(p) * 2.0**-126 + U)
    return 1.01 * float(total.max())


E_ERF = erf_error_bound()


# ------------------------------------------------------------------------------------------ restatements and bounds
def stem_ref(spect, chunks, L, bn1_scale, bn1_shift, w, bias):
    """(ref, bound) [n, 32, L, 32] float64 for spect [frames, 128] and the packed stem parameters (float64 tensors of
    fp32 values: bn1 [128], w [32, 12] or [32, 4, 3], bias [32])."""
    dev = spect.device
    w = w.reshape(32, 4, 3)
    refs, bounds = [], []
    tl = torch.arange(-1, L + 1, device=dev)
    for fb, T, start, _, _, _, ln in chunks:
        fr = start + tl
        clip_ok = (fr >= 0) & (fr < T)
        conv_ok = (tl >= 0) & (tl < ln)
        zero = torch.zeros((), dtype=spect.dtype, device=dev)
        v = torch.where(clip_ok[:, None], spect[fb + fr.clamp(0, T - 1)], zero)
        x = torch.where(conv_ok[:, None], v * bn1_scale + bn1_shift, zero)
        cols = torch.stack([x[dt : dt + L] for dt in range(3)], dim=-1).view(L, 32, 4, 3)  # t, f, df, dt
        a = torch.einsum("lfdt,cdt->flc", cols, w) + bias
        s = torch.einsum("lfdt,cdt->flc", cols.abs(), w.abs()) + bias.abs()
        e_in = torch.einsum("lfdt,cdt->flc", U * cols.abs(), w.abs())
        e_a = (12 * U * s + e_in) * (1 + 2.0**-20)
        refs.append(gelu_erf(a))
        bounds.append(GELU_SLOPE * e_a + (0.5 * E_ERF + 2 * U) * (a.abs() + e_a) + 2.0**-148)
    return torch.stack(refs), torch.stack(bounds)


def head_ref(x, w, b, sum_head):
    """(beat, down, beat bound, down bound) [n, L] float64 for x [n, L, D], w [2, D], b [2] (fp32 values)."""
    D = x.shape[-1]
    w = w.reshape(2, D)
    K = D // 32 + 5
    den = x.norm(dim=-1).clamp_min(1e-12)
    a = x @ w.T  # [n, L, 2]
    sa = x.abs() @ w.abs().T
    o = a / den[..., None] + b
    e_inv = (K / 2 + 3) * U
    e = (K * U * sa / den[..., None] + (a / den[..., None]).abs() * (e_inv + U) + U * o.abs()) * (1 + 2.0**-20)
    e = e + K * 2.0**-149 / den[..., None]
    if sum_head:
        return o[..., 0] + o[..., 1], o[..., 1], e[..., 0] + e[..., 1] + U * (o[..., 0] + o[..., 1]).abs(), e[..., 1]
    return o[..., 0], o[..., 1], e[..., 0], e[..., 1]


def head_scatter(chunks, L, vals, out_count):
    """Places per-chunk rows vals [n, L] at out_base + start + t for every owned t: (out [out_count], owned mask)."""
    out = torch.full((out_count,), float("nan"), dtype=vals.dtype, device=vals.device)
    owned = torch.zeros(out_count, dtype=torch.int32, device=vals.device)
    for i, (_, _, start, ob, lo, hi, _) in enumerate(chunks):
        if lo < hi:
            out[ob + start + lo : ob + start + hi] = vals[i, lo:hi]
            owned[ob + start + lo : ob + start + hi] += 1
    return out, owned


def zero_tail_ref(buf, chunks, F, L, C):
    """buf [n, F, L, C] (any dtype) with rows [len, L) of every plane of each chunk cleared."""
    out = buf.clone()
    for i, c in enumerate(chunks):
        out[i, :, c[6]:] = 0
    return out


# ------------------------------------------------------------------------------------------ chunk tables
def wave(clips, plan, guard=3):
    """The chunk table of one mixed-length wave over clips of the given lengths, laid out back to back with `guard`
    guard frames before, between and after them, in the spectrogram and in the outputs alike.  plan(T) -> (starts,
    lens, own_lo, own_hi) of the clip's chunks.  Chunks are sorted longest first (stable), as run_chunks sorts them.
    Returns (chunks, L, frames, clip_offsets)."""
    chunks, offs, pos = [], [], guard
    for T in clips:
        offs.append(pos)
        for s, ln, lo, hi in zip(*plan(T)):
            chunks.append((pos, T, s, pos, lo - s, hi - s, ln))
        pos += T + guard
    chunks.sort(key=lambda c: -c[6])
    return chunks, max(c[6] for c in chunks), pos, offs


def sweep_lengths(chunk_size, border):
    """Clip lengths around the planner's edges for one chunking: 1, 2, a border's worth, the chunk and the step
    +- 1, two chunks and some, and an odd long one."""
    step = chunk_size - 2 * border
    v = {1, 2, border + 1, 2 * border + 1, step - 1, step, step + 1, chunk_size - 1, chunk_size, chunk_size + 1,
         2 * step + 3, 3 * chunk_size + 7}
    return sorted(x for x in v if x >= 1)


# ------------------------------------------------------------------------------------------ fp32 emulations (numpy)
def _approx(exact, rel, sign):
    """An fp32 result within `rel` (relative) of the float64 `exact`, off by about `rel` in direction `sign`."""
    y = exact * (1.0 + sign * rel)
    r = y.astype(np.float32)
    over = np.abs(r.astype(np.float64) - exact) > np.abs(y - exact)
    toward = np.where(exact > y, np.inf, -np.inf).astype(np.float32)
    return np.where(over, np.nextafter(r, toward), r).astype(np.float32)


def gelu_fast_np(x, sign=1.0, p_const=AS_P):
    """gelu_fast (csrc/epilogue.cuh) in fp32 on float32 x, rcp / ex2 off by their stated error in direction sign.
    Returns (gelu, erf_abs)."""
    x = np.asarray(x, np.float32)
    z = (np.abs(x) * np.float32(0.70710678118654752440)).astype(np.float32)
    d = fma_f32(np.float32(p_const), z, np.float32(1.0))
    t = _approx(1.0 / d.astype(np.float64), RCP_APPROX_REL, sign)
    p = fma_f32(np.float32(AS_A[4]), t, np.float32(AS_A[3]))
    for c in AS_A[2::-1]:
        p = fma_f32(p, t, np.float32(c))
    p = (p * t).astype(np.float32)
    arg = ((z * z).astype(np.float32) * np.float32(-LOG2E)).astype(np.float32)
    exact = np.exp2(arg.astype(np.float64))
    e = np.where(exact < 2.0**-126, np.float32(0), _approx(exact, EX2_APPROX_REL, sign)).astype(np.float32)
    erf_abs = fma_f32(-p, e, np.float32(1.0))
    half = (np.float32(0.5) * x).astype(np.float32)
    return fma_f32((np.float32(0.5) * np.abs(x)).astype(np.float32), erf_abs, half), erf_abs


STEM_MISTAKES = ("conv_by_clip", "bn_on_chunk_pad", "clip_pad_after_bn", "gelu_const")
HEAD_MISTAKES = ("drop_first", "ignore_sum_head", "ss_no_sqrt")
ZERO_TAIL_MISTAKES = ("plane_mod", "from_len_plus_1")


def stem_np(spect, chunks, L, bn1_scale, bn1_shift, w, bias, sign=1.0, mistake=None):
    """stem_kernel in fp32 (numpy), in the kernel's order of operations: [n, 32, L, 32] float32."""
    w = np.asarray(w, np.float32).reshape(32, 12)
    out = np.empty((len(chunks), 32, L, 32), np.float32)
    t = np.arange(L)
    for b, (fb, T, start, _, _, _, ln) in enumerate(chunks):
        ins = np.empty((32, 4, 3, L), np.float32)  # f, df, dt, t
        for dt in range(3):
            tl = t + dt - 1
            fr = start + tl
            clip_ok = (fr >= 0) & (fr < T)
            conv_ok = (tl >= 0) & ((fr < T) if mistake == "conv_by_clip" else (tl < ln))
            v = np.where((conv_ok & clip_ok)[:, None], spect[fb + np.clip(fr, 0, T - 1)], np.float32(0)).astype(np.float32)
            x = fma_f32(v, bn1_scale[None, :], bn1_shift[None, :])  # [L, 128]
            if mistake == "clip_pad_after_bn":
                x = np.where(clip_ok[:, None], x, np.float32(0))
            pad = np.broadcast_to(bn1_shift, x.shape) if mistake == "bn_on_chunk_pad" else np.float32(0)
            x = np.where(conv_ok[:, None], x, pad).astype(np.float32)
            ins[:, :, dt, :] = x.T.reshape(32, 4, L)
        for co in range(32):
            a = np.broadcast_to(np.float32(bias[co]), (32, L)).astype(np.float32)
            for df in range(4):
                for dt in range(3):
                    a = fma_f32(ins[:, df, dt, :], w[co, df * 3 + dt], a)
            out[b, :, :, co] = gelu_fast_np(a, sign, 0.3275 if mistake == "gelu_const" else AS_P)[0]
    return out


def head_np(x, w, bias, chunks, L, sum_head, out_count, mistake=None):
    """head_kernel in fp32 (numpy): (beat, down) [out_count] float32, NaN where no chunk writes."""
    n, _, D = x.shape
    w = np.asarray(w, np.float32).reshape(2, D)
    xl = x.reshape(n, L, D // 32, 32)
    wl = w.reshape(2, D // 32, 32)
    ss = np.zeros((n, L, 32), np.float32)
    a0, a1 = ss.copy(), ss.copy()
    for i in range(D // 32):  # lane chains over i = lane, lane + 32, ...
        v = xl[:, :, i, :]
        ss = fma_f32(v, v, ss)
        a0 = fma_f32(v, wl[0, i], a0)
        a1 = fma_f32(v, wl[1, i], a1)
    for o in (16, 8, 4, 2, 1):  # warp_sum: lane l adds lane l ^ o
        idx = np.arange(32) ^ o
        ss, a0, a1 = [(s + s[..., idx]).astype(np.float32) for s in (ss, a0, a1)]
    ss, a0, a1 = ss[..., 0], a0[..., 0], a1[..., 0]
    nrm = ss if mistake == "ss_no_sqrt" else np.sqrt(ss).astype(np.float32)
    inv = (np.float32(1.0) / np.maximum(nrm, np.float32(1e-12))).astype(np.float32)
    o0 = fma_f32(a0, inv, np.float32(bias[0]))
    o1 = fma_f32(a1, inv, np.float32(bias[1]))
    beat_v = (o0 + o1).astype(np.float32) if (sum_head or mistake == "ignore_sum_head") else o0
    beat = np.full(out_count, np.nan, np.float32)
    down = beat.copy()
    for b, (_, _, start, ob, lo, hi, _) in enumerate(chunks):
        lo = lo + 1 if mistake == "drop_first" else lo
        if lo < hi:
            beat[ob + start + lo : ob + start + hi] = beat_v[b, lo:hi]
            down[ob + start + lo : ob + start + hi] = o1[b, lo:hi]
    return beat, down


def zero_tail_np(buf, chunks, F, L, mistake=None):
    """zero_tail_kernel on buf [n, F, L, C] (numpy, any dtype), returning a cleared copy."""
    out = buf.copy()
    n = len(chunks)
    for plane in range(n * F):
        b = plane % n if mistake == "plane_mod" else plane // F
        first = chunks[b][6] + (1 if mistake == "from_len_plus_1" else 0)
        out[plane // F, plane % F, first:] = 0
    return out
