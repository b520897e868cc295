"""The forward pass of BeatThis as a list of steps, each a chain of kernel test hooks (bt_debug_*), restated from the
hyper-parameters, the layer stack of the reference model (oracle.forward) and the hook contracts of
include/beatthis.h.  Shared by tests/test_gpu_forward_steps.py (runs every chain on the tap in front of its step and
compares it with the step's tap by bits) and tests/test_cpu_forward_steps.py (ties the list to the oracle's taps and to
the packed parameters, and the chains, evaluated in float64 by Eval64, to oracle.forward in float64).

A step maps the tap in front of it (its input) to its own tap (its output).  Its chain lists every hook call with
every argument the forward pass gives the kernel it stands for:

- the packed parameters by name (``b0.attnF.wqkv``, ``b1.conv.w``, ``lin.w``, ``l3.ff.w2``, ...);
- GEMM shapes as tests/gemm_reference.py builds them (plain_shape, conv_shape, lin_shape), the epilogue kind, bias,
  GELU, residual, the fp32 and 16-bit outputs and the tile policy of a residual epilogue;
- C, heads, RoPE position mode (0: time t, 1: frequency plane p % F), F and the q scale;
- the keys per chunk and sequences per chunk of the time attentions in a wave of chunks of different lengths;
- where the 16-bit copy of the residual stream comes from (written by the FFN in front of a convolution, or rounded
  from the fp32 stream when there is no FFN), and zero_tail's element size.

Each call also names ``prod``: the profile name of the forward pass's launch it stands for, so that the chains of a
pass can be counted against the launches the pass makes.

The layer stack (oracle.forward, reference beat_tracker.py:188-192 and roformer.py):
  stem -> 3 frontend blocks of [attnF, ffF, attnT, ffT] (partial transformers only) + conv (C -> 2C, F -> F / 2)
       -> frontend.linear -> n_layers x [attn, ff] -> head.
The choices of the 16-bit path (include/beatthis.h, DESIGN.md):
  - the sub-blocks of width 32 and 64 (the first two frontend blocks) run fused: RMSNorm + gates + QKV + RoPE in one
    kernel, and the FFN in one kernel that also adds the attention's out-projection in front of it; a tap on the
    attention keeps that residual stream visible, so a pass tapping it runs the out-projection as its own GEMM
    (steps with ``tap_mode``: they do not run in the production pass);
  - the time attentions take q scaled by log2(e) / sqrt(32) (softmax in base 2); the frequency attention scales its
    scores itself;
  - the convolutions read the 16-bit copy of the stream.
The fp32 path runs everything unfused; attentions of at most two heads compute their gates in the norm kernel.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch

from gemm_reference import QSCALE_TIME, conv_shape, lin_shape, plain_shape
from numerics import normalize

FUSED_WIDTHS = (32, 64)
HOOK_ROPE_ROWS = 1500  # bt_debug_fused_qkv takes L <= BT_CHUNK: longer planes run as pieces of at most this many rows


@dataclass
class Call:
    op: str    # stem, norm, gemm, fused_qkv, attention, attention_freq, fused_ff, zero_tail, round16, head
    prod: str  # the profile name of the forward pass's launch this call stands for
    args: dict = field(default_factory=dict)


@dataclass
class Step:
    name: str    # the output tap ("logits" for the head)
    input: str   # the tap in front ("spect" for the stem)
    kind: str    # stem, attn_freq, attn_time, ff, pair_freq, pair_time, conv, linear, head
    chain: list
    C: int = 0   # width of the step's input rows
    F: int = 1   # planes per chunk of the step's input
    out: str = "x"  # the register holding the step's output
    tap_mode: bool = False  # the variant a tap on this attention runs (not part of the production pass)
    params: tuple = ()  # packed parameters the step reads


@dataclass
class Wave:
    nb: int
    L: int
    lens: list | None = None  # keys per chunk, wave order; None: every chunk is L long

    @property
    def varlen(self):
        return self.lens is not None and any(n != self.L for n in self.lens)


def _attn_calls(p, half, C, F, freq, wave):
    """The hook calls of x -> o (gates * attention, before the out-projection) of attention layer p."""
    heads, front, planes, L = C // 32, F > 1, wave.nb * F, wave.L
    posmode, qscale = (1, 1.0) if freq else (0, QSCALE_TIME if half else 1.0)
    sfx = "_front" if front else ""
    if half and C in FUSED_WIDTHS:
        calls = [Call("fused_qkv", f"qkv_fused_c{C}", dict(w=p + ".wqkv", wg=p + ".wg", bg=p + ".bg", C=C, L=L, F=F,
                                                           posmode=posmode, qscale=qscale))]
    else:
        gates_in_norm = heads <= 2  # fp32 path only: the 16-bit path fuses those widths
        calls = [Call("norm", "norm_gates" if gates_in_norm else "norm" + sfx,
                      dict(C=C, heads=heads if gates_in_norm else 0, wg=p + ".wg" if gates_in_norm else None,
                           bg=p + ".bg" if gates_in_norm else None))]
        if not gates_in_norm:
            calls.append(Call("gemm", "gemm_gates" + sfx, dict(shape=plain_shape(planes, L, 32, C), a="xn", w=p + ".wg",
                                                               bias=p + ".bg", kind=2, heads=heads, out_f32="gates")))
        calls.append(Call("gemm", "gemm_qkv" + sfx, dict(shape=plain_shape(planes, L, 3 * C, C), a="xn", w=p + ".wqkv",
                                                         kind=1, C=C, heads=heads, posmode=posmode, F=F, qscale=qscale,
                                                         out_act="qkv")))
    if freq:
        calls.append(Call("attention_freq", "attn_freq", dict(B=wave.nb, F=F, L=L, heads=heads)))
    else:
        calls.append(Call("attention", "attn_time_tc" if half else "attn_time_simt",
                          dict(seqs=planes, L=L, heads=heads, key_lens=list(wave.lens) if wave.varlen else None,
                               seqs_per_chunk=F, qscale=qscale)))
    return calls


def _out_call(p, C, F, wave):
    return Call("gemm", "gemm_attn_out" + ("_front" if F > 1 else ""),
                dict(shape=plain_shape(wave.nb * F, wave.L, C, C), a="o", w=p + ".wout", resid=True, out_f32="x",
                     resid_epilogue=True))


def _ff_calls(p, half, C, F, mult, wave, wout=None, copy=False):
    """The hook calls of x += ff(x) of FFN layer p (wout: the out-projection in front it adds first, fused kernels
    only; copy: it also writes the 16-bit copy xb that the convolution after it reads)."""
    if half and C in FUSED_WIDTHS and mult == 4:
        return [Call("fused_ff", f"ff_fused_c{C}", dict(w1=p + ".w1", b1=p + ".b1", w2=p + ".w2", b2=p + ".b2", C=C,
                                                        wout=wout, xb=copy))]
    assert wout is None
    planes, L, sfx = wave.nb * F, wave.L, "_front" if F > 1 else ""
    return [
        Call("norm", "norm" + sfx, dict(C=C, heads=0, wg=None, bg=None)),
        Call("gemm", "gemm_ff1" + sfx, dict(shape=plain_shape(planes, L, mult * C, C), a="xn", w=p + ".w1", bias=p + ".b1",
                                            gelu=True, out_act="h")),
        Call("gemm", "gemm_ff2" + sfx, dict(shape=plain_shape(planes, L, C, mult * C), a="h", w=p + ".w2", bias=p + ".b2",
                                            resid=True, out_f32="x", out_act="xb" if copy else None,
                                            resid_epilogue=True)),
    ]


def _attn_params(p):
    return tuple(p + s for s in (".wqkv", ".wg", ".bg", ".wout"))


def _ff_params(p):
    return tuple(p + s for s in (".w1", ".b1", ".w2", ".b2"))


def forward_steps(hp: dict, half: bool, wave: Wave, tap_variants: bool = True) -> list:
    """The steps of one forward pass of the model of hyper-parameters hp over `wave`, on the 16-bit (half) or fp32
    path, in order.  tap_variants: also list the tap-mode variants of the fused attention steps."""
    steps = [Step("stem", "spect", "stem", [Call("stem", "stem", dict(
        params=("stem.bn1_scale", "stem.bn1_shift", "stem.w", "stem.bias")))], C=128, F=1,
        params=("stem.bn1_scale", "stem.bn1_shift", "stem.w", "stem.bias"))]
    prev, C, F = "stem", hp["stem_dim"], hp["spect_dim"] // 4
    for i in range(3):
        b = f"b{i}"
        ff_in_front = False
        if hp["partial_transformers"]:
            for d, freq in (("F", True), ("T", False)):
                pa, pf = f"{b}.attn{d}", f"{b}.ff{d}"
                copy = half and d == "T"  # the FFN in front of the convolution writes its 16-bit copy
                attn = _attn_calls(pa, half, C, F, freq, wave)
                kind = "freq" if freq else "time"
                if half and C in FUSED_WIDTHS:  # the out-projection runs inside the fused FFN
                    steps.append(Step(pf, prev, "pair_" + kind, attn + _ff_calls(pf, half, C, F, 4, wave, pa + ".wout",
                                                                                  copy), C, F,
                                      params=_attn_params(pa) + _ff_params(pf)))
                    if tap_variants:
                        steps.append(Step(pa, prev, "attn_" + kind, attn + [_out_call(pa, C, F, wave)], C, F,
                                          tap_mode=True, params=_attn_params(pa)))
                else:
                    steps.append(Step(pa, prev, "attn_" + kind, attn + [_out_call(pa, C, F, wave)], C, F,
                                      params=_attn_params(pa)))
                    steps.append(Step(pf, pa, "ff", _ff_calls(pf, half, C, F, 4, wave, None, copy), C, F,
                                      params=_ff_params(pf)))
                prev = pf
            ff_in_front = True
        last = i == 2  # the last convolution feeds frontend.linear in the activation type
        chain = []
        if half and not ff_in_front:
            chain.append(Call("round16", "f32_to_h16", {}))
        a = "xb" if half else "x"
        if wave.varlen:
            chain.append(Call("zero_tail", "zero_tail", dict(buf=a, elem_bytes=2 if half else 4, F=F, C=C)))
        chain.append(Call("gemm", "gemm_conv", dict(shape=conv_shape(wave.nb, F, wave.L, C), a=a, w=b + ".conv.w",
                                                    bias=b + ".conv.bias", gelu=True,
                                                    out_f32=None if last else "x", out_act="xn" if last else None)))
        steps.append(Step(b + ".conv", prev, "conv", chain, C, F, out="xn" if last else "x",
                          params=(b + ".conv.w", b + ".conv.bias")))
        prev, C, F = b + ".conv", 2 * C, F // 2
    D = hp["transformer_dim"]
    steps.append(Step("frontend", prev, "linear", [Call("gemm", "gemm_frontend_linear", dict(
        shape=lin_shape(wave.nb, wave.L, D, F, C), a="xn", w="lin.w", bias="lin.b", out_f32="x"))], C, F,
        params=("lin.w", "lin.b")))
    prev = "frontend"
    for k in range(hp["n_layers"]):
        pa, pf = f"l{k}.attn", f"l{k}.ff"
        steps.append(Step(pa, prev, "attn_time", _attn_calls(pa, half, D, 1, False, wave) + [_out_call(pa, D, 1, wave)],
                          D, 1, params=_attn_params(pa)))
        steps.append(Step(pf, pa, "ff", _ff_calls(pf, half, D, 1, hp["ff_mult"], wave), D, 1, params=_ff_params(pf)))
        prev = pf
    steps.append(Step("logits", prev, "head", [Call("head", "head", dict(w="head.w", b="head.b",
                                                                          sum_head=bool(hp["sum_head"])))], D, 1,
                      out="logits", params=("head.w", "head.b")))
    return steps


def tap_names(hp: dict) -> list:
    """Every activation the forward pass can tap, in order (oracle.forward's tap names)."""
    names = ["stem"]
    for i in range(3):
        if hp["partial_transformers"]:
            names += [f"b{i}.{s}" for s in ("attnF", "ffF", "attnT", "ffT")]
        names.append(f"b{i}.conv")
    names.append("frontend")
    for k in range(hp["n_layers"]):
        names += [f"l{k}.attn", f"l{k}.ff"]
    return names


def production_taps(hp: dict, half: bool) -> list:
    """The taps a production pass materialises: all but the attentions whose out-projection runs inside the fused
    FFN after them (16-bit path, widths 32 and 64)."""
    steps = forward_steps(hp, half, Wave(1, 16), tap_variants=False)
    return [s.name for s in steps if s.kind != "head"]


# ---------------------------------------------------------------------------------------------------------------------
# float64 evaluation of the chains, from the hook contracts of include/beatthis.h.  Composed over a pass, it must give
# oracle.forward in float64 (tests/test_cpu_forward_steps.py): that ties every argument of every chain -- weights, F,
# position modes, q scales, key lengths, zero_tail -- to the reference model independently of the library, and the GPU
# test ties the forward pass to the chains bit for bit.  Rounding points (round16, the 16-bit operands) are identities
# here.
def _attend(q, k, v, mask=None):
    """softmax(q k^T / sqrt(32)) v over the last two dims of [..., n, 32] (mask [.., n]: keys kept)."""
    s = q @ k.transpose(-1, -2) / math.sqrt(32)
    if mask is not None:
        s = s.masked_fill(~mask[..., None, :], float("-inf"))
    return torch.softmax(s, dim=-1) @ v


def slab_gemm(shape, a, w):
    """acc [planes_out * L, N] of bt_debug_gemm's shape contract: row p_out * L + t sums, over the slabs s, the columns
    [0, Kslab) of the row of plane p_out * plane_mul + plane_add[s] at time t + t_shift[s] of a [planes_in * L, lda]
    (zeros outside [0, L)) times W[:, s * Kslab : (s + 1) * Kslab] of w [N, nslab * Kslab]."""
    L, N, K = shape["L"], shape["N"], shape["Kslab"]
    A = a.reshape(shape["planes_in"], L, shape["lda"])[..., :K]
    w = w.reshape(N, shape["nslab"] * K)
    acc = torch.zeros(shape["planes_out"] * L, N, dtype=a.dtype)
    p_out = torch.arange(shape["planes_out"])
    for s in range(shape["nslab"]):
        x = A[p_out * shape["plane_mul"] + shape["plane_add"][s]]
        sh, y = shape["t_shift"][s], torch.zeros_like(x)
        if sh >= 0:
            y[:, : L - sh] = x[:, sh:]
        else:
            y[:, -sh:] = x[:, : L + sh]
        acc += y.reshape(-1, K) @ w[:, s * K : (s + 1) * K].T
    return acc


class Eval64:
    """Runs the calls of a step in float64 on registers of [rows, cols] float64 tensors, as Chain does on the device.
    P: packed parameters as float64 tensors; chunks: the wave's chunk table; spect: [frames, 128] float64."""

    def __init__(self, P, wave, chunks, spect, regs):
        self.P, self.wave, self.chunks, self.spect, self.regs = P, wave, chunks, spect, regs

    def run(self, step):
        for c in step.chain:
            getattr(self, "_" + c.op)(**c.args)
        return self.regs[step.out]

    def _stem(self, params):
        from chunk_kernels_reference import stem_ref

        ref, _ = stem_ref(self.spect, self.chunks, self.wave.L, *(self.P[p] for p in params))
        self.regs["x"] = ref.reshape(-1, 32)

    def _norm(self, C, heads, wg, bg):
        xn = normalize(self.regs["x"])
        self.regs["xn"] = xn
        if heads:
            self.regs["gates"] = torch.sigmoid(xn @ self.P[wg].view(32, C)[:heads].T + self.P[bg][:heads])

    def _gemm(self, shape, a, w, bias=None, kind=0, gelu=False, resid=False, out_f32=None, out_act=None,
              resid_epilogue=False, C=0, heads=0, posmode=0, F=1, qscale=1.0):
        from gemm_reference import GemmCase, epilogue_ref

        acc = slab_gemm(shape, self.regs[a], self.P[w])
        case = GemmCase("", shape, kind=kind, bias=bias is not None, gelu=gelu, resid=resid, C=C, heads=heads,
                        posmode=posmode, F=F, qscale=qscale)
        rope = (self.P["rope.cos"].view(-1, 16), self.P["rope.sin"].view(-1, 16)) if kind == 1 else (None, None)
        y, _ = epilogue_ref(case, acc, self.P[bias] if bias else None, self.regs["x"] if resid else None, False, *rope)
        for r in (out_f32, out_act):
            if r:
                self.regs[r] = y

    def _fused_qkv(self, w, wg, bg, C, L, F, posmode, qscale):
        heads = C // 32
        self._norm(C, heads, wg, bg)
        shape = plain_shape(self.regs["x"].shape[0] // L, L, 3 * C, C)
        self._gemm(shape, "xn", w, kind=1, C=C, heads=heads, posmode=posmode, F=F, qscale=qscale, out_act="qkv")

    def _heads(self, t, seqs, n, heads):
        return t.reshape(seqs, n, heads, 32).transpose(1, 2)  # [seqs, heads, n, 32]

    def _gate(self, o, heads):
        return (o.reshape(-1, heads, 32) * self.regs["gates"].reshape(-1, heads, 1)).reshape(-1, heads * 32)

    def _attention(self, seqs, L, heads, key_lens, seqs_per_chunk, qscale):
        C = heads * 32
        qkv = self.regs["qkv"]
        q, k, v = (self._heads(qkv[:, i * C : (i + 1) * C], seqs, L, heads) for i in range(3))
        mask = None
        if key_lens is not None:
            lens = torch.tensor(key_lens).repeat_interleave(seqs_per_chunk)
            mask = (torch.arange(L)[None, :] < lens[:, None])[:, None, :]  # [seqs, 1, L]
        o = _attend(q / qscale, k, v, mask)  # q arrives scaled by the q scale of the QKV call
        self.regs["o"] = self._gate(o.transpose(1, 2).reshape(-1, C), heads)

    def _attention_freq(self, B, F, L, heads):
        C = heads * 32
        qkv = self.regs["qkv"].reshape(B, F, L, 3 * C).transpose(1, 2)  # sequences over the F planes of (b, t)
        q, k, v = (self._heads(qkv[..., i * C : (i + 1) * C], B * L, F, heads) for i in range(3))
        o = _attend(q, k, v).transpose(1, 2).reshape(B, L, F, C).transpose(1, 2).reshape(-1, C)
        self.regs["o"] = self._gate(o, heads)

    def _fused_ff(self, w1, b1, w2, b2, C, wout, xb):
        x = self.regs["x"]
        if wout:
            x = x + self.regs["o"] @ self.P[wout].view(C, C).T
        h = torch.nn.functional.gelu(normalize(x) @ self.P[w1].view(4 * C, C).T + self.P[b1])
        x = x + h @ self.P[w2].view(C, 4 * C).T + self.P[b2]
        self.regs["x"] = x
        if xb:
            self.regs["xb"] = x

    def _round16(self):
        self.regs["xb"] = self.regs["x"]

    def _zero_tail(self, buf, elem_bytes, F, C):
        t = self.regs[buf].reshape(self.wave.nb, F, self.wave.L, C).clone()
        for i, n in enumerate(self.wave.lens):
            t[i, :, n:] = 0
        self.regs[buf] = t.reshape(-1, C)

    def _head(self, w, b, sum_head):
        from chunk_kernels_reference import head_ref, head_scatter

        x = self.regs["x"].reshape(self.wave.nb, self.wave.L, -1)
        beat, down, _, _ = head_ref(x, self.P[w], self.P[b], sum_head)
        frames = self.spect.shape[0]
        self.regs["logits"] = torch.stack([head_scatter(self.chunks, self.wave.L, v, frames)[0] for v in (beat, down)])


# ---------------------------------------------------------------------------------------------------------------------
def mutations(half: bool, wave: Wave, steps: list) -> list:
    """(what, step, the step with one wrong but valid argument) for one step of each kind: the wiring errors a check
    must catch.  Each is a valid hook call: it computes wrong numbers, never out of bounds."""
    import copy

    prod = [s for s in steps if not s.tap_mode]

    def first(kinds, pred=lambda s: True):
        return next((s for s in prod if s.kind in kinds and pred(s)), None)

    def mutate(s, pred, **kw):
        m = copy.deepcopy(s)
        c = next(c for c in m.chain if pred(c))
        c.args.update(kw)
        return m

    qkv = lambda c: "posmode" in c.args  # the fused QKV or the kind 1 GEMM
    out = []
    s = first(("attn_freq", "pair_freq"))
    if s:
        out.append(("posmode 0", s, mutate(s, qkv, posmode=0)))
        F = next(c.args["F"] for c in s.chain if qkv(c))
        out.append((f"F {F // 2} for {F}", s, mutate(s, qkv, F=F // 2)))
    if half:
        s = first(("attn_time", "pair_time"))
        out.append(("qscale 1", s, mutate(s, qkv, qscale=1.0)))
    if wave.varlen:
        s = first(("attn_time", "pair_time"))
        out.append(("every key length L", s, mutate(s, lambda c: c.op == "attention", key_lens=[wave.L] * wave.nb)))
    s = first(("ff",), lambda s: s.name.startswith("l0."))
    out.append(("the next layer's w2", s, mutate(s, lambda c: c.args.get("w", "").endswith(".w2"), w="l1.ff.w2")))
    s = first(("pair_time",))
    if s:
        c = next(c for c in s.chain if c.op == "fused_ff")
        out.append(("attnF's wout in the time pair", s,
                    mutate(s, lambda c: c.op == "fused_ff", wout=c.args["wout"].replace(".attnT.", ".attnF."))))
    s = first(("conv",))
    shape = dict(next(c for c in s.chain if c.op == "gemm").args["shape"])
    shape["t_shift"] = [-t for t in shape["t_shift"]]
    out.append(("t_shift reversed", s, mutate(s, lambda c: c.op == "gemm", shape=shape)))
    s = first(("linear",))
    out.append(("l0.ff.b2 for lin.b", s, mutate(s, lambda c: c.op == "gemm", bias="l0.ff.b2")))
    return out
