"""Float64 restatements of the time- and frequency-direction attention kernels and the elementwise bounds their unit
tests hold them to: attn_time_kernel (16-bit context) and attn_time_simt_kernel (fp32) through bt_debug_attention,
attn_freq_mma_kernel<F> (16-bit) and attn_freq_kernel<F> (fp32) through bt_debug_attention_freq.  Shared by
tests/test_gpu_attention.py (runs the cases) and tests/test_cpu_attention_reference.py (ties the restatement to SDPA,
the bounds to a CPU emulation of the kernels, and the cases to the instantiations in the library).

Operands, as the hooks pack them (round16: the activation type; the fp32 context does not round):
  time, tensor cores : q^ = round16(fp32(q * QSCALE_H16)), QSCALE_H16 = fp32(s * log2 e), s = fp32(1 / sqrt(32));
                       k^ = round16(k), v^ = round16(v); scores in base-2 units: t_ij = q^_i . k^_j
  time, SIMT         : qs = fp32(q * s); t_ij = log2 e * (qs_i . k_j)      (the kernel takes expf of qs . k)
  frequency, TC      : q^, k^, v^ = round16(q, k, v); t = SL2 * (q^ . k^), SL2 = fp32(s * log2 e) = QSCALE_H16
  frequency, SIMT    : as the SIMT time path (__expf)
Restatement, per (sequence or group, head, query row i), over the keys j a row may see (the first len of its chunk in
time; the F planes of its (chunk, frame, head) in frequency):
  M_k = max of t_ij over the keys of the online-softmax steps 0..k (64-key tiles on tensor cores, 8-key blocks in the
  SIMT time kernel, one step in frequency); W_j = 2^(t_j - M_last)
  numerator weight  Wn_j = round16(2^(t_j - M_k(j))) 2^(M_k(j) - M_last)    (16-bit paths: P is packed per step)
                         = W_j                                               (fp32 paths)
  o_i = g_i sum_j Wn_j v^_j / sum_j W_j     (the denominator l sums the UNROUNDED p); 16-bit paths store round16(o)

Bound per output element, first order in each term, in float64 from the data (all exponents base 2):
  scores     e_j = mma_error(32, sum_d |q^_d k^_jd|) on tensor cores (numerics.mma_error: products of 16-bit
             operands are exact in fp32, each of the K + K/16 additions of an m16n8k16 chain loses <= 2^-23 of the
             sum of magnitudes); SIMT: a 32-term fmaf chain, 32 2^-24 sum_d |qs_d k_jd| (times log2 e).  SL2 e_j on
             the frequency tensor-core path.  The row maximum of step k is off by at most Ek_j = max e over the keys of
             steps <= k.
  exponent   x_j = fp32(s_j - m_k): 2^-24 |x_j| (one more 2^-24 |x_j| for the SL2 product of the frequency TC path)
  exp        ex2.approx.ftz.f32 (MUFU): 2 ulp, EX2_APPROX_REL = 2^-22 relative (PTX ISA, ex2);
             ex2_poly (tc_common.cuh) on the AT_POLY_MASK score pairs: EX2_POLY_REL = 8e-5 relative, as its comment
             states (test_cpu_attention_reference checks it on >= 10^7 points: 7.74e-5 at r = +-0.5; its constant
             0.99992895 makes it a bias low by ~7e-5, not noise);
             expf, exp2f: 2 ulp, EXPF_REL = 2^-22 (CUDA Programming Guide, mathematical functions);
             __expf(x): 2 + floor(1.173 |x|) ulp (CUDA Programming Guide, intrinsic functions);
             results below 2^-126 are flushed (ftz) and ex2_poly clamps its argument at -120: an absolute
             TINY = 2^-119 per key, and per masked key of the last tile (ex2_poly(-inf) = 2^-120 goes into l)
  P          16-bit paths: the kernel rounds p_j, within d_j = p_ref_j ((1 + exp) 2^(e_j + Ek_j + x) - 1) + TINY of
             p_ref_j = 2^(t_j - M_k(j)); rounding_error(p_ref_j, d_j) (fp16 subnormals below 2^-14 included).  In the
             numerator only: l sums the unrounded p.
  rescale    alpha = ex2(m_old - m_new) multiplies o and l alike, so its value cancels up to the keys it does not
             scale: per later step one exp error + one fp32 product (2^-24), and the 2^-24 |m_old - m_new| of its
             argument; the product telescopes, so the numerator weight also carries 2^(+-Ek_j) (the running max
             against M_k) on top of its rounded p
  l          fp32 sum: (16 nkv + 2) 2^-24 (each thread adds 16 of every 64 keys, then two quad shuffles), 2NT + 2 on
             the frequency TC path, one addition per key in the SIMT kernels
  P V        mma_error(nnz, sum_j p^_j |v^_j|) on tensor cores, nnz the keys of the row whose rounded p may not be 0
             (a product that is exactly 0 adds nothing, and an MMA step without a nonzero product leaves the
             accumulator as it is; a dominant key or a late maximum leaves few); an fp32 fmaf chain in the SIMT
             kernels: one 2^-24 per key
  output     g / l and the product: 2 2^-24; the 16-bit store: rounding_error(o, bound).
With A_j, B_j the absolute errors of the numerator and denominator weights (relative to W_j's scale):
  |dO| <= g (sum_j A_j |v^_j| + PV + |o/g| (sum_j B_j + l)) / (sum_j W_j - sum_j B_j - l)
(the denominator keeps the second-order term, so the bound also holds for large relative errors).
"""
import math
from dataclasses import dataclass

import torch

from numerics import EX2_APPROX_REL, EXPF_REL, LOG2E, QSCALE_H16, S_F32, U, mma_error, rnd, rounding_error

EX2_POLY_REL = 8e-5
TINY = 2.0**-119
AT_TILE = 64  # keys per step of attn_time_kernel (AT_BKV)
AT_POLY_MASK = 0x52  # score pairs nb of a tile (keys 8 nb .. 8 nb + 7) that take ex2_poly (kernels_attn.cu)
SA_BLOCK = 8  # keys per online-softmax step of attn_time_simt_kernel
FREQ_TC_HEADS = {32: 1, 16: 2, 8: 4}  # the (F, heads) pairs of attn_freq_mma_kernel<F>
# path -> whether the hooks run it (the 16-bit context) and the kernels they launch there (time, frequency)
PATHS = {"tc": (True, "attn_time_kernel", "attn_freq_mma_kernel"),
         "simt": (False, "attn_time_simt_kernel", "attn_freq_kernel")}


def poly_keys(K, device=None):
    """[K] bool: key positions whose exponential attn_time_kernel takes with ex2_poly."""
    nb = (torch.arange(K, device=device) % AT_TILE) // 8
    return ((AT_POLY_MASK >> nb) & 1).bool()


def _f32mul(t, c):
    return (t.float() * torch.tensor(c, dtype=torch.float32, device=t.device)).double()


def softmax_ref(T2, E2, valid, v, gates, step, exp_rel, alpha_rel, sub_ops, p_dt, n_sum, pv_error, out_dt, n_pad):
    """(ref, bound, o, err) of g * sum_j Wn_j v_j / sum_j W_j for one batch of rows.
    T2, E2 [G, R, K]: scores in base-2 units and bounds on the kernel's score error; valid [G, K]: the keys the rows
    see (a prefix); v [G, K, 32]; gates [G, R]; step: keys per online-softmax step; exp_rel(x2, e2) -> [G, R, K]
    relative error of the exponential at base-2 argument x2 <= 0; alpha_rel: error of one rescale (exp + product);
    sub_ops: fp32 operations forming the exponent; p_dt: type P is rounded to (None: not rounded); n_sum [G]:
    additions per chain of l; pv_error(s, nnz) [G, R, 32] (nnz [G, R, 1]: the keys whose rounded p may not be 0, on
    the 16-bit paths); out_dt: the stored type; n_pad: masked keys whose p may be TINY.
    o and err are the value and bound before the output is stored (the fp32 result); ref and bound those of the
    stored value (ref = round16(o) on the 16-bit paths)."""
    G, R, K = T2.shape
    ns = -(-K // step)
    pad = ns * step - K
    vmask = valid[:, None, :].expand(G, R, K)
    t = T2.masked_fill(~vmask, -math.inf)
    e = E2.masked_fill(~vmask, 0.0)
    tp = torch.nn.functional.pad(t, (0, pad), value=-math.inf).view(G, R, ns, step)
    ep = torch.nn.functional.pad(e, (0, pad), value=0.0).view(G, R, ns, step)
    Ms = tp.amax(-1).cummax(-1).values  # running max after each step
    Es = ep.amax(-1).cummax(-1).values
    Mt = Ms.repeat_interleave(step, -1)[..., :K]
    Ek = Es.repeat_interleave(step, -1)[..., :K]
    Mfin, Efin = Ms[..., -1:], Es[..., -1:]
    x = (t - Mt).masked_fill(~vmask, 0.0)  # <= 0
    scale = torch.exp2(Mt - Mfin).masked_fill(~vmask, 0.0)
    p_ref = torch.exp2(x).masked_fill(~vmask, 0.0)
    W = p_ref * scale
    eps = exp_rel(x, e + Ek)
    rsub = ((1 + U) ** sub_ops - 1) * x.abs()
    nkv = (valid.sum(-1) + step - 1) // step  # steps the kernel runs per group
    after = (nkv[:, None, None] - 1 - torch.arange(K, device=T2.device) // step).clamp_min(0)
    chain = (1 + alpha_rel) ** after * torch.exp2(U * (Mfin - Mt + 2 * Efin)) - 1
    B = W * ((1 + eps) * torch.exp2(e + rsub) * (1 + chain) - 1) + TINY * scale
    if p_dt is not None:
        d = p_ref * ((1 + eps) * torch.exp2(e + Ek + rsub) - 1) + TINY
        p16 = rnd(p_ref, p_dt)
        Rr = rounding_error(p_ref, d, p_dt)
        Wn = p16 * scale
        A = (Rr + (p16 + Rr) * ((1 + chain) * torch.exp2(Ek) - 1)) * scale + TINY * scale
    else:
        Wn, A = W, B
    zero = ~vmask
    W, Wn, A, B = (z.masked_fill(zero, 0.0) for z in (W, Wn, A, B))
    nnz = ((Wn + A) > 0).sum(-1, keepdim=True) if p_dt is not None else None  # products P V may have that are not 0
    SW = W.sum(-1)
    SB = B.sum(-1) + n_pad * TINY
    den_err = SB + n_sum[:, None] * U * (SW + SB)
    va = v.abs()
    on = (Wn @ v) / SW[..., None]
    num_err = A @ va + pv_error((Wn + A) @ va, nnz)
    g = gates[..., None]
    ref = g * on
    err = g * (num_err + on.abs() * den_err[..., None]) / (SW - den_err)[..., None]
    err = err + ((1 + U) ** 2 - 1) * (ref.abs() + err)
    if out_dt is None:
        return ref, err, ref, err
    return rnd(ref, out_dt), rounding_error(ref, err, out_dt), ref, err


def _batches(G, per_group, budget=1 << 25):
    n = max(1, budget // max(1, per_group))
    return [(a, min(G, a + n)) for a in range(0, G, n)]


def time_ref(q, k, v, gates, lens, path, dt, exact=False):
    """(ref, bound, o, err) (softmax_ref) of the time-direction attention on q, k, v [seqs, L, heads * 32] (float64 of the fp32 values the
    hook gets), gates [seqs * L, heads], lens [seqs] keys per sequence; path "tc" or "simt"; dt: the 16-bit type of
    the tc path.  exact: the unrounded operation (no fp32 constants, no rounding), bounds None."""
    seqs, L, C = q.shape
    H = C // 32
    hv = lambda t: t.reshape(seqs, L, H, 32).permute(0, 2, 1, 3).reshape(seqs * H, L, 32)
    if exact:
        qh, kh, vh, sc = hv(q), hv(k), hv(v), LOG2E / math.sqrt(32)
    elif path == "tc":
        qh, kh, vh, sc = hv(rnd(_f32mul(q, QSCALE_H16), dt)), hv(rnd(k, dt)), hv(rnd(v, dt)), 1.0
    else:
        qh, kh, vh, sc = hv(_f32mul(q, S_F32)), hv(k), hv(v), LOG2E
    g = gates.reshape(seqs, L, H).permute(0, 2, 1).reshape(seqs * H, L)
    lens_g = torch.as_tensor(lens, device=q.device).repeat_interleave(H)
    valid = torch.arange(L, device=q.device)[None, :] < lens_g[:, None]
    out = [torch.empty_like(qh) if i % 2 == 0 or not exact else None for i in range(4)]
    for a, b in _batches(seqs * H, L * L):
        T2 = sc * (qh[a:b] @ kh[a:b].transpose(1, 2))
        vm = valid[a:b]
        if exact:
            w = torch.exp2(T2.masked_fill(~vm[:, None, :], -math.inf))
            out[0][a:b] = out[2][a:b] = g[a:b, :, None] * (w @ vh[a:b]) / w.sum(-1, keepdim=True)
            continue
        S = qh[a:b].abs() @ kh[a:b].abs().transpose(1, 2)
        nkv = (vm.sum(-1) + AT_TILE - 1) // AT_TILE
        if path == "tc":
            pk = poly_keys(L, q.device)
            kw = dict(step=AT_TILE, alpha_rel=EX2_APPROX_REL + U, sub_ops=1, p_dt=dt, n_sum=16 * nkv + 2,
                      pv_error=lambda s, nnz: mma_error(nnz, s), out_dt=dt, n_pad=AT_TILE,
                      exp_rel=lambda x, e: torch.where(pk, EX2_POLY_REL, EX2_APPROX_REL).expand_as(x))
            E2 = mma_error(32, S)
        else:
            nk = SA_BLOCK * ((vm.sum(-1) + SA_BLOCK - 1) // SA_BLOCK)
            kw = dict(step=SA_BLOCK, alpha_rel=EXPF_REL + U, sub_ops=1, p_dt=None, n_sum=nk,
                      pv_error=lambda s, nnz: nk[:, None, None] * U * s, out_dt=None, n_pad=0,
                      exp_rel=lambda x, e: torch.full_like(x, EXPF_REL))
            E2 = 32 * U * S * LOG2E
        for o, r in zip(out, softmax_ref(T2, E2, vm, vh[a:b], g[a:b], **kw)):
            o[a:b] = r
    back = lambda t: None if t is None else t.view(seqs, H, L, 32).permute(0, 2, 1, 3).reshape(seqs, L, C)
    return tuple(back(t) for t in out)


def freq_ref(q, k, v, gates, B, F, path, dt, exact=False):
    """(ref, bound, o, err) (softmax_ref) of the frequency-direction attention on q, k, v [B * F * L, heads * 32] (token (b F + f) L + t),
    gates [B * F * L, heads]; path "tc" (attn_freq_mma_kernel) or "simt" (attn_freq_kernel)."""
    M, C = q.shape
    H, L = C // 32, M // (B * F)
    grp = lambda t: t.reshape(B, F, L, H, -1).permute(0, 2, 3, 1, 4).reshape(B * L * H, F, -1)  # [groups, F, 32]
    if exact:
        qh, kh, vh, sc = grp(q), grp(k), grp(v), LOG2E / math.sqrt(32)
    elif path == "tc":
        qh, kh, vh, sc = grp(rnd(q, dt)), grp(rnd(k, dt)), grp(rnd(v, dt)), QSCALE_H16
    else:
        qh, kh, vh, sc = grp(_f32mul(q, S_F32)), grp(k), grp(v), LOG2E
    g = grp(gates)[..., 0]
    G = qh.shape[0]
    valid = torch.ones(G, F, dtype=torch.bool, device=q.device)
    T2 = sc * (qh @ kh.transpose(1, 2))
    if exact:
        w = torch.exp2(T2 - T2.amax(-1, keepdim=True))
        ref = g[..., None] * (w @ vh) / w.sum(-1, keepdim=True)
        res = (ref, None, ref, None)
    else:
        S = qh.abs() @ kh.abs().transpose(1, 2)
        if path == "tc":
            NT = 4 if F == 32 else 2
            ones = torch.ones(G, dtype=torch.float64, device=q.device)
            res = softmax_ref(T2, QSCALE_H16 * mma_error(32, S), valid, vh, g, step=F, alpha_rel=0.0,
                                     sub_ops=2, p_dt=dt, n_sum=(2 * NT + 2) * ones,
                                     pv_error=lambda s, nnz: mma_error(nnz, s), out_dt=dt, n_pad=0,
                                     exp_rel=lambda x, e: torch.full_like(x, EXPF_REL))
        else:
            ones = torch.ones(G, dtype=torch.float64, device=q.device)
            expf_fast = lambda x, e: (2 + 1.173 * (x.abs() + 2 * e) / LOG2E) * 2.0**-23  # x, e base 2 -> natural
            res = softmax_ref(T2, 32 * U * S * LOG2E, valid, vh, g, step=F, alpha_rel=0.0, sub_ops=1,
                                     p_dt=None, n_sum=F * ones, pv_error=lambda s, nnz: F * U * s, out_dt=None, n_pad=0,
                                     exp_rel=expf_fast)
    back = lambda t: None if t is None else t.reshape(B, L, H, F, 32).permute(0, 3, 1, 2, 4).reshape(M, C)
    return tuple(back(t) for t in res)


# ---- cases
@dataclass(frozen=True)
class TimeCase:
    seqs: int
    L: int
    heads: int
    key_lens: tuple | None = None  # keys per chunk of spc sequences (None: all L)
    spc: int = 1

    @property
    def id(self):
        lens = "" if self.key_lens is None else f" lens={list(self.key_lens)} per {self.spc}"
        return f"time seqs={self.seqs} L={self.L} heads={self.heads}{lens}"

    def lens(self):
        return [self.L] * self.seqs if self.key_lens is None else [self.key_lens[s // self.spc] for s in range(self.seqs)]


@dataclass(frozen=True)
class FreqCase:
    B: int
    F: int
    L: int
    heads: int

    @property
    def id(self):
        return f"freq B={self.B} F={self.F} L={self.L} heads={self.heads}"

    def on_tensor_cores(self):
        return FREQ_TC_HEADS[self.F] == self.heads


RAGGED = (1, 13, 63, 64, 65, 127, 128, 129, 1499, 1500)  # chunk lengths at every tile edge


def time_cases():
    cs = [TimeCase(2, 1500, 4), TimeCase(2, 1500, 16)]  # main layers: small0 (D = 128), final0 (D = 512)
    for L in (150, 1500):  # frontend: (heads, planes per chunk) of the three blocks, two chunks
        cs += [TimeCase(2 * P, L, H, (L, L * 2 // 3), P) for H, P in ((1, 32), (2, 16), (4, 8))]
    cs += [TimeCase(len(RAGGED), 1500, 2, RAGGED, 1)]  # a wave of chunks of every tile-edge length
    cs += [TimeCase(2, 13, 2), TimeCase(3, 129, 1), TimeCase(1, 1001, 4)]  # L not a multiple of 128
    # the cases of the earlier flat-tolerance test
    cs += [TimeCase(3, 1500, 2), TimeCase(2, 200, 1), TimeCase(1, 13, 4), TimeCase(2, 128, 1),
           TimeCase(7, 1500, 16, (1, 13, 63, 64, 65, 150, 1500)), TimeCase(96, 150, 1, (150, 65, 13), 32),
           TimeCase(64, 1500, 1, (1500, 64), 32)]
    return cs


def freq_cases(path):
    pairs = [(32, 1), (16, 2), (8, 4)] + ([(16, 1), (8, 2)] if path == "simt" else [])
    return [FreqCase(B, F, L, H) for F, H in pairs for L in (1, 3, 4, 5, 13, 1500) for B in (1, 3)]


def launched_kernels(path):
    """{(kernel, F)} the GPU cases of `path` launch (F 0 for the time kernels)."""
    _, time_k, freq_k = PATHS[path]
    return ({(time_k, 0)} if time_cases() else set()) | {(freq_k, c.F) for c in freq_cases(path)}


# ---- input families: (q, k, v, gates) fp32 on `device`
FAMILIES = ("random", "dominant", "late_max", "early_max", "flat_split", "masked_garbage")
MASKED_KV = 3e4


def time_families(case):
    return [f for f in FAMILIES if f != "masked_garbage" or case.key_lens is not None]


def freq_families(case):
    return ["random", "dominant"] + (["cross_group"] if case.F == 8 else [])


def _unit(*shape, g, device):
    x = torch.randn(*shape, generator=g, device=device)
    return x / x.norm(dim=-1, keepdim=True)


def _dominant_q(k, kappa, exclude, g):
    """q [.., R, 32] (fp32) whose score QSCALE_H16 q_i . k_kappa(i) beats every rival key of its row by >= 32 base-2
    units: q_i = c_i k_kappa(i).  k [.., K, 32] unit rows; kappa [.., R]; exclude [.., R, K]: keys that are no
    rivals (kappa itself, keys the row does not see)."""
    kk = torch.gather(k, -2, kappa[..., None].expand(*kappa.shape, 32))  # [.., R, 32]
    cos = kk @ k.transpose(-1, -2)  # [.., R, K]
    rival = cos.masked_fill(exclude, -1.0)
    gap = 1 - rival.amax(-1)
    assert gap.min().item() > 0.05, f"dominant-key family: gap {gap.min().item():.3f}"
    c = 32 / (QSCALE_H16 * gap)
    return kk * c[..., None]


def time_inputs(case, family, g, device):
    seqs, L, H = case.seqs, case.L, case.heads
    C = 32 * H
    lens = torch.tensor(case.lens(), device=device)
    gates = torch.rand(seqs * L, H, generator=g, device=device)
    if family in ("random", "masked_garbage"):
        q = torch.randn(seqs, L, C, generator=g, device=device) * 1.5
        k = torch.randn(seqs, L, C, generator=g, device=device)
        v = torch.randn(seqs, L, C, generator=g, device=device)
        if family == "masked_garbage":
            valid = (torch.arange(L, device=device)[None, :] < lens[:, None])[..., None]
            sign = torch.randint(0, 2, (seqs, L, C), generator=g, device=device) * 2 - 1
            k = torch.where(valid, k, MASKED_KV * sign)
            v = torch.where(valid, v, -MASKED_KV * sign)
        return q, k, v, gates
    j = torch.arange(L, device=device)
    if family == "flat_split":
        # q = 0: every score is exactly 0, so every key a row sees has the same weight, and the kernel's exponentials
        # are ex2_poly(0) and ex2.approx(0).  V is +u on the ex2_poly keys (3 of 8 pairs) and -0.6 u on the others:
        # a full tile averages to 0, and any bias between the two exponentials is the output itself.
        u = 1 + torch.rand(seqs, 1, H, 32, generator=g, device=device)
        v = torch.where(poly_keys(L, device)[None, :, None, None], u, -0.6 * u)
        q = torch.zeros(seqs, L, C, device=device)
        k = torch.randn(seqs, L, C, generator=g, device=device)
        return q, k, v.reshape(seqs, L, C).contiguous(), gates
    v = torch.randn(seqs, L, H, 32, generator=g, device=device)
    if family == "dominant":
        # key kappa(i) = (i + shift) % len: every key of a chunk (first and last of every tile, the last valid one) is
        # the dominant key of some row
        n = lens[:, None]  # [seqs, 1]
        k = _unit(seqs, L, H, 32, g=g, device=device)
        shift = torch.arange(seqs, device=device)[:, None] * 7 + torch.arange(H, device=device)[None, :] * 3 + 5
        kappa = (j[None, None, :] + shift[..., None] + n[..., None] // 2) % n[..., None]  # [seqs, H, L]
        jk = j[None, None, None, :]
        exclude = (jk >= n[..., None, None]) | (jk == kappa[..., None])
        q = _dominant_q(k.permute(0, 2, 1, 3), kappa, exclude, g).permute(0, 2, 1, 3)
    else:
        # one direction u carries the score: q_i = c u + noise, k_j = beta_j u + noise; beta ~ 1 in the last (late_max)
        # or first (early_max) tile of each chunk, <= 0.85 elsewhere (>= 20 base-2 units lower), down to 0 (< -120)
        c = 200 / QSCALE_H16
        ntile = (lens + AT_TILE - 1) // AT_TILE
        tile = j[None, :] // AT_TILE
        top = tile == (ntile[:, None] - 1) if family == "late_max" else tile == 0
        u = torch.rand(seqs, L, H, generator=g, device=device)
        beta = torch.where(top[..., None], 0.95 + 0.05 * u, 0.85 * u)
        k = torch.randn(seqs, L, H, 32, generator=g, device=device) * 0.02
        k[..., 0] = beta
        q = torch.randn(seqs, L, H, 32, generator=g, device=device) * 0.02
        q[..., 0] = c
    return q.reshape(seqs, L, C).contiguous(), k.reshape(seqs, L, C).contiguous(), v.reshape(seqs, L, C).contiguous(), gates


def freq_inputs(case, family, g, device):
    B, F, L, H = case.B, case.F, case.L, case.heads
    M, C = B * F * L, 32 * H
    gates = torch.rand(M, H, generator=g, device=device)
    v = torch.randn(M, C, generator=g, device=device)
    if family == "random":
        return (torch.randn(M, C, generator=g, device=device) * 1.5, torch.randn(M, C, generator=g, device=device), v,
                gates)
    # one group per (b, t, h): plane f's dominant key is plane (f + 1 + (t + h) % (F - 1)) % F, never itself.
    # cross_group (F = 8, where a 16-row tile of attn_freq_mma_kernel holds frames t and t ^ 1): q aims at that plane
    # of frame t ^ 1 instead, 32 base-2 units above every key of its own group; a row that sees the other group's keys
    # then returns the other group's value.  Frames without a partner (t ^ 1 = L) keep their own dominant key.
    k = _unit(B, L, H, F, 32, g=g, device=device)
    f = torch.arange(F, device=device)
    sh = 1 + (torch.arange(L, device=device)[:, None] + torch.arange(H, device=device)[None, :]) % (F - 1)  # [L, H]
    kappa = ((f[None, None, :] + sh[..., None]) % F).expand(B, L, H, F)
    own = torch.gather(k, 3, kappa[..., None].expand(B, L, H, F, 32))
    target = own
    exclude = f[None, None, None, None, :] == kappa[..., None]
    if family == "cross_group":
        t = torch.arange(L, device=device)
        has = (t ^ 1) < L
        partner = torch.gather(k[:, (t ^ 1).clamp(max=L - 1)], 3, kappa[..., None].expand(B, L, H, F, 32))
        target = torch.where(has[None, :, None, None, None], partner, own)
        exclude = exclude & ~has[None, :, None, None, None]
    rival = (target @ k.transpose(-1, -2)).masked_fill(exclude, -1.0)
    gap = 1 - rival.amax(-1)
    assert gap.min().item() > 0.05, f"{family} family: gap {gap.min().item():.3f}"
    q = target * (32 / (QSCALE_H16 * gap))[..., None]
    to_tok = lambda t: t.permute(0, 3, 1, 2, 4).reshape(M, C)  # [B, L, H, F, 32] -> token-major
    return to_tok(q).contiguous(), to_tok(k).contiguous(), v, gates


# ---- production activations: final0 on the stage-parity input of test_gpu_kernels._stage_errors_full_chunks
def _pre_attention(z, sd, p, heads):
    """oracle.pre_attention on z [S, n, C] in the hooks' layout: q, k, v [S, n, C] and gates [S, n, heads]."""
    from oracle import beat_this_oracle as O

    S, n, C = z.shape
    q, k, v, gates = O.pre_attention(z, sd, p, heads)
    back = lambda t: t.permute(0, 2, 1, 3).reshape(S, n, C)
    return back(q), back(k), back(v), torch.sigmoid(gates)


def production_inputs():
    """{name: (case, (q, k, v, gates) fp32 CPU)}: final0's first frontend time attention (b0.attnT), its first
    frequency attention (b0.attnF) and main layer 0, on the oracle's activations at their inputs."""
    from beat_this_b200 import synthetic
    from oracle import beat_this_oracle as O

    sd = synthetic.make_state_dict(synthetic.model_hparams("final0"), 0)
    torch.manual_seed(4)
    B, T = 2, 1500
    chunks = torch.rand(B, T, 128) * 7
    taps = {}
    with torch.inference_mode():
        O.forward(sd, chunks, taps)
        out = {}
        st = taps["stem"]  # [B, F, L, C]
        Fq, C = st.shape[1], st.shape[3]
        z = st.permute(0, 2, 1, 3).reshape(B * T, Fq, C)
        q, k, v, g = _pre_attention(z, sd, "frontend.blocks.0.partial.attnF", C // 32)
        tok = lambda t: t.reshape(B, T, Fq, -1).permute(0, 2, 1, 3).reshape(B * Fq * T, -1).contiguous()
        out["b0.attnF"] = (FreqCase(B, Fq, T, C // 32), tuple(tok(t) for t in (q, k, v, g)))
        z = taps["b0.ffF"].reshape(B * Fq, T, C)
        q, k, v, g = _pre_attention(z, sd, "frontend.blocks.0.partial.attnT", C // 32)
        out["b0.attnT"] = (TimeCase(B * Fq, T, C // 32, (T,) * B, Fq),
                           (q.contiguous(), k.contiguous(), v.contiguous(), g.reshape(-1, C // 32).contiguous()))
        h = taps["frontend"]
        D = h.shape[-1]
        q, k, v, g = _pre_attention(h, sd, "transformer_blocks.layers.0.0", D // 32)
        out["l0.attn"] = (TimeCase(B, T, D // 32), (q.contiguous(), k.contiguous(), v.contiguous(),
                                                    g.reshape(-1, D // 32).contiguous()))
    return out
