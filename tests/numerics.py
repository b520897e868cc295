"""The error model the kernel unit tests derive their bounds from: the stated error figures of the hardware and the CUDA
math library, the tolerances several test files share, and the float64 and fp32 helpers the restatements
(tests/*_reference.py) are written with.  Pure torch and numpy, no CUDA.

Figures (relative to the exact result unless stated):
  U                one fp32 rounding to nearest: 2^-24 (IEEE 754 binary32, 24-bit significand).  F32_ADD names the same
                   figure for an fp32 addition outside an MMA.
  RCP_APPROX_REL   rcp.approx.ftz.f32: at most 1 ulp, 2^-23 (PTX ISA, rcp.approx.f32).
  REL_2ULP         2 ulp of an fp32 result, 2^-22.  EX2_APPROX_REL: ex2.approx.ftz.f32 (PTX ISA, ex2.approx.f32: 2 ulp);
                   EXPF_REL: expf and exp2f, and the same figure for erff, sinf and cosf over the full range (CUDA
                   Programming Guide, mathematical functions; the library is built without -use_fast_math).
  TANH_APPROX_TOL  tanh.approx.f32: absolute error at most 2^-10.987 (PTX ISA), taken as 2^-10.
  mma_error        an fp32 mma.sync accumulation of K products of 16-bit operands onto c: the products are exact in
                   fp32, and each of the K + K/16 additions of an m16n8k16 chain (aligned to its largest term, rounded
                   or truncated) loses at most 2^-23 of s = |c| + sum |a_k b_k|: 2 K 2^-23 s (derivation).
  GELU_SLOPE       max |GELU'| = 1.1290 at x = sqrt 2, for the erf and the tanh form alike (GELU'' = 0 there).
  GELU2_SLOPE      max |GELU''| = 0.7979 = 2 phi(0), at x = 0.
Constants of the kernels: LOG2E; S_F32 = fp32(1 / sqrt 32), the attention scale; QSCALE_H16 = fp32(S_F32 * log2 e),
the q scale bt_debug_attention applies in the 16-bit context (api_debug.cu), which is also the SL2 score scale of
attn_freq_mma_kernel.

Rounding to 16 bits: the kernels compute in fp32, so the value a kernel rounds to 16 bits differs from its float64
value v by up to some d, and the rounded value can land on the other neighbour of round16(v).  Rounding is monotonic,
so the kernel's rounded value lies in [round16(v - d), round16(v + d)]:
  rounding_error(v, d) = max |round16(v +- d) - round16(v)|
is 0 where v is farther than d from a rounding midpoint, one ulp near one (d below half an ulp), and stays sound for
any d (fp16 subnormals below 2^-14 included).
"""
import math

import numpy as np
import torch

U = 2.0**-24
F32_ADD = U
RCP_APPROX_REL = 2.0**-23
REL_2ULP = 2.0**-22
EX2_APPROX_REL = REL_2ULP
EXPF_REL = REL_2ULP
TANH_APPROX_TOL = 2.0**-10
GELU_SLOPE = 1.13
GELU2_SLOPE = 0.8
LOG2E = 1.4426950408889634
S_F32 = float(np.float32(0.17677669529663687))
QSCALE_H16 = float(np.float32(np.float32(S_F32) * np.float32(LOG2E)))

# Flat tolerances (bt_debug_gemm against the float64 reference of tests/gemm_reference.py, on the operands the kernel
# multiplies: rounded to the 16-bit type in the 16-bit context):
#   fp32 outputs  : fp32 accumulation over K <= 2048 of unit-scale products, |ref| ~ 1:
#                   GEMM_ACC_TOL_H16 (wgmma) / GEMM_ACC_TOL_F32 (CUDA-core fmaf chain) x (1 + |ref|)
#   16-bit outputs: 1 ulp of the 16-bit-rounded float64 value (the fp32 result may sit on the other side of a rounding
#                   boundary) + the fp32 bound above, which only matters near zero where the ulp is tiny
#   GELU          : the 16-bit path evaluates the tanh form with tanh.approx.f32 (TANH_APPROX_TOL), so 0.5 |x| 2^-10
#                   on top; the fp32 path the exact erf form (erff)
#   gates         : GATES_TOL absolute on sigmoid values (slope <= 1/4 of the fp32 accumulation error)
GEMM_ACC_TOL_H16 = 1e-4
GEMM_ACC_TOL_F32 = 3e-5
GATES_TOL = 1e-6
# frame logits against the fp32 reference: the fp32 path (measured ~1e-4), and the 16-bit path (fp16 operands, fp32
# accumulation and residual stream; logits have std ~2, range +-8)
F32_TOL = 1e-3
H16_TOL = 0.05


def f32(v):
    """v rounded to fp32, as a Python float."""
    return float(np.float32(v))


def f64(t):
    return torch.as_tensor(t).double()


def fma_f32(a, b, c):
    """fmaf on fp32 values (numpy arrays or scalars), correctly rounded: the float64 sum of the exact product and c,
    with the one case where rounding twice differs from rounding once (a float64 result exactly between two floats)
    resolved by the exact remainder of the float64 addition."""
    a, b, c = (np.asarray(x, np.float32) for x in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)  # exact: 24 + 24 bits
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)  # s + err == p + c exactly
    f = s.astype(np.float32)
    r = f.astype(np.float64)
    nb = np.nextafter(f, np.where(s > r, np.float32(np.inf), np.float32(-np.inf)))
    tie = (s != r) & (s == (r + nb.astype(np.float64)) / 2) & (err != 0)
    past = np.sign(err) == np.sign(s - r)  # the exact value lies beyond the midpoint: the far neighbour
    return np.where(tie & past, nb, f).astype(np.float32)


def rnd(t, dt):
    """t rounded to the 16-bit type dt, back in float64; dt None: t unchanged."""
    return t if dt is None else t.to(dt).double()


def rounding_error(v, d, dt):
    """max |round16(v +- d) - round16(v)|: how far the 16-bit rounding of a value within d of float64 v can land from
    round16(v) (round to nearest is monotonic)."""
    r = rnd(v, dt)
    return torch.maximum((rnd(v + d, dt) - r).abs(), (rnd(v - d, dt) - r).abs())


def ulp16(x, dt):
    """Spacing of the 16-bit floating-point type dt at its representable values x (float64)."""
    mant, emin = (10, -14) if dt == torch.float16 else (7, -126)
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0**emin))) - mant)


def mma_error(K, s):
    """Error bound of an fp32 mma.sync accumulation of K products of 16-bit operands onto c: s = |c| + sum |a_k b_k|."""
    return 2 * K * 2.0**-23 * s


def normalize(x):
    return x / x.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x**3)))


def rope_positions(M, L, F, posmode, device=None):
    """The RoPE position of token row m: m % L (posmode 0, time) or (m / L) % F (posmode 1, frequency plane)."""
    m = torch.arange(M, device=device)
    return m % L if posmode == 0 else (m // L) % F


def rope_ref(x, cos, sin):
    """Interleaved-pair rotation (oracle.rope / rotary_embedding_torch) of x [M, heads * 32] by per-row tables
    cos, sin [M, 16]: out[2i] = x[2i] cos_i - x[2i+1] sin_i, out[2i+1] = x[2i+1] cos_i + x[2i] sin_i."""
    M = x.shape[0]
    p = x.reshape(M, -1, 16, 2)
    c, s = cos[:, None, :], sin[:, None, :]
    return torch.stack((p[..., 0] * c - p[..., 1] * s, p[..., 1] * c + p[..., 0] * s), dim=-1).reshape(x.shape)


def worst(got, ref, bound):
    """max |got - ref| / bound (NaN in got or a non-finite difference: inf)."""
    got, ref, bound = f64(got), f64(ref), f64(bound)
    d = (got - ref).abs()
    if not torch.isfinite(d).all():
        return math.inf
    r = torch.where(d == 0, torch.zeros_like(d), d / bound)
    return float(r.max()) if d.numel() else 0.0
