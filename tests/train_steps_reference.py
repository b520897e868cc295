"""The training passes of BeatThis (bt_train_forward_ex / bt_train_backward_ex) as a list of steps, each a forward
and a backward chain of training-kernel test hook calls (bt_debug_train_kernel), restated from the hyper-parameters,
the reference model's layer stack (oracle.forward, tests/train_mode_reference.forward_train), the parameter table
(BeatThis.state_dict() order), the dropout numbering and the activation-store layout documented in include/beatthis.h.
Shared by tests/test_cpu_train_steps.py (the chains, evaluated in float64 by Eval64 and composed over whole passes,
give float64 autograd of the reference) and tests/test_gpu_train_steps.py (the passes equal the chains bit for bit,
step by step).

A step's forward chain maps its stored input (region ``in`` of the store) to every activation it stores and to the
next step's input (the head: the logits); in training mode it also computes the batch statistics of its BatchNorms
into the store's statistics region and moves the running statistics (two reductions with beta = 0.9).  Its backward
chain maps the gradient at its output (scratch ``dcur``) to the gradient at its input (``dcur`` again; the stem:
``dspect``) and to the gradient of every trainable entry it reads.

Every call is (op, slots, desc, prod): the bt_debug_train_kernel op, its array slots in the header's order as
references into the memory of a pass, every descriptor field the pass gives the kernel, and the profile names of the
pass launches it stands for (train_gemm, train_gemm_dx, train_gemm_dw, train_reduce, ...).  References:
  ("P", i) / ("G", i) / ("R", i)  parameter, gradient and running-statistics table entry i;
  ("A", off, n)                   n floats of the activation store at float offset off;
  ("S", name)                     the pass's scratch: dcur (gradient of the stream), s1, s2, big, dqkv, hd1, hd2, part;
  ("X", name)                     beat, down (logits), dbeat, ddown (their gradients), dspect.
"""
from __future__ import annotations

import copy
import math
from dataclasses import dataclass, field

import numpy as np
import torch

PART_FLOATS = 8 << 20  # the pass's split-K / column-sum partials (kTrPartFloats)
PROFILE = {"rms_fwd": "train_rmsnorm", "rms_bwd": "train_rmsnorm_bwd", "bn_gelu_fwd": "train_bn_gelu",
           "bn_gelu_bwd": "train_bn_gelu_bwd", "bn_grads": "train_bn_grads", "bn_scale": "train_bn_scale",
           "gelu_bwd": "train_gelu_bwd", "im2col": "train_im2col", "col2im": "train_col2im", "concat": "train_concat",
           "rope": "train_rope", "gate_fwd": "train_gate", "gate_bwd": "train_gate_bwd", "head_fwd": "train_head",
           "head_bwd": "train_head", "attn_fwd": "train_attention", "attn_dq": "train_attention_dq",
           "attn_dkv": "train_attention_dkv", "reduce": "train_reduce"}


def _f32(x):
    return float(np.float32(x))


def r4(n):
    return (n + 3) // 4 * 4


def dw_splits(M, N, K):
    """tr_dw_splits: the parts of a weight gradient dW [N, K] summed over M rows (two CTAs per SM of 132, at least 256
    rows a part, all parts inside the partials)."""
    tiles = -(-N // 64) * -(-K // 64)
    s = min(-(-264 // tiles), max(1, M // 256))
    return max(1, min(s, PART_FLOATS // (N * K)))


def gemm_parts(K, splits):
    kc = (-(-K // splits) + 15) // 16 * 16
    return -(-K // kc)


def colsum_splits(M, N):
    return min(-(-M // 512), PART_FLOATS // N)


def scratch_sizes(BL):
    return dict(dcur=BL * 1024, s1=BL * 1024, s2=BL * 1024, big=BL * 4096, dqkv=BL * 3072, hd1=BL * 32 + 1024,
                hd2=BL * 32 + 1024, part=PART_FLOATS)


@dataclass
class Call:
    op: str
    slots: list
    desc: dict
    prod: tuple
    exact: dict = field(default_factory=dict)  # float64 evaluation: the values desc's fp32 constants round

    def params(self, kind):
        return {r[1] for r in self.slots if r is not None and r[0] == kind}


@dataclass
class TrStep:
    index: int
    kind: str       # stem, attn_freq, attn_time, ffn, conv, linear, head
    module: str     # state_dict prefix
    C: int
    F: int
    mult: int
    p: int          # table index of the step's first entry
    regions: dict   # store regions: name -> (offset, floats)
    fwd: list = field(default_factory=list)
    bwd: list = field(default_factory=list)

    def A(self, name):
        off, n = self.regions[name]
        return ("A", off, n)


# ---------------------------------------------------------------------------------------------- table and layout
def _layer_list(hp):
    """(kind, module, C, F, mult) of model_steps: the stem, per frontend block attnF, ffF, attnT, ffT (partial
    transformers only) and the convolution, frontend.linear, per main layer its attention and FFN, the head."""
    C, F = hp["stem_dim"], hp["spect_dim"] // 4
    out = [("stem", "frontend.stem", C, F, 0)]
    for i in range(3):
        m = f"frontend.blocks.{i}"
        if hp["partial_transformers"]:
            out += [("attn_freq", m + ".partial.attnF", C, F, 0), ("ffn", m + ".partial.ffF", C, F, 4),
                    ("attn_time", m + ".partial.attnT", C, F, 0), ("ffn", m + ".partial.ffT", C, F, 4)]
        out.append(("conv", m, C, F, 0))
        C, F = 2 * C, F // 2
    out.append(("linear", "frontend.linear", C, F, 0))
    D = hp["transformer_dim"]
    for k in range(hp["n_layers"]):
        out += [("attn_time", f"transformer_blocks.layers.{k}.0", D, 1, 0),
                ("ffn", f"transformer_blocks.layers.{k}.1", D, 1, hp["ff_mult"])]
    out.append(("head", "", D, 1, 0))
    return out


def _bn_names(p):
    return [p + s for s in (".weight", ".bias", ".running_mean", ".running_var", ".num_batches_tracked")]


def table(hp):
    """The parameter table: state_dict names in BeatThis.state_dict() order, one list per step of _layer_list."""
    out = []
    for kind, m, C, F, mult in _layer_list(hp):
        if kind == "stem":
            out.append(_bn_names(m + ".bn1d") + [m + ".conv2d.weight"] + _bn_names(m + ".bn2d"))
        elif kind.startswith("attn"):
            out.append([m + s for s in (".rotary_embed.freqs", ".norm.gamma", ".to_qkv.weight", ".to_gates.weight",
                                        ".to_gates.bias", ".to_out.0.weight")])
        elif kind == "ffn":
            out.append([m + s for s in (".net.0.gamma", ".net.1.weight", ".net.1.bias", ".net.4.weight",
                                        ".net.4.bias")])
        elif kind == "conv":
            out.append([m + ".conv2d.weight"] + _bn_names(m + ".norm"))
        elif kind == "linear":
            out.append([m + ".weight", m + ".bias"])
        else:
            out.append(["transformer_blocks.norm.gamma", "task_heads.beat_downbeat_lin.weight",
                        "task_heads.beat_downbeat_lin.bias"])
    return out


def trainable(name):
    return not name.endswith((".running_mean", ".running_var", ".num_batches_tracked", ".freqs"))


def layout(hp, B, L, train):
    """The activation store of include/beatthis.h: per step (in model_steps order) its regions, each rounded up to 4
    floats, then in training mode the batch statistics (mean, then variance, each of ch channels rounded up to 4) of the
    stem's bn1d and bn2d and of each convolution's norm.  Returns (regions per step, total floats)."""
    BL, Fs = B * L, hp["spect_dim"]
    total = 0
    regs = []

    def alloc(n):
        nonlocal total
        off = total
        total += r4(n)
        return off, n

    for kind, _, C, F, mult in _layer_list(hp):
        M = BL * F
        if kind == "stem":
            names = [("in", BL * Fs), ("z", M * C)]
        elif kind.startswith("attn"):
            names = [("in", M * C), ("xn", M * C), ("inv", M), ("qkv", 3 * M * C), ("gate", M * C // 32),
                     ("lse", M * C // 32), ("o", M * C)]
        elif kind == "ffn":
            names = [("in", M * C), ("xn", M * C), ("inv", M), ("h", M * mult * C), ("a", M * mult * C)]
        elif kind == "conv":
            names = [("in", M * C), ("z", M // 2 * 2 * C)]
        elif kind == "linear":
            names = [("in", M * C), ("xl", M * C)]
        else:
            names = [("in", M * C), ("xn", M * C), ("inv", M)]
        regs.append({k: alloc(n) for k, n in names})
    if train:
        for r, (kind, _, C, F, _) in zip(regs, _layer_list(hp)):
            for bn, ch in (("bn1", Fs), ("bn2", C)) if kind == "stem" else (("bn2", 2 * C),) if kind == "conv" else ():
                r[bn + ".mean"] = alloc(ch)
                r[bn + ".var"] = alloc(ch)
    return regs, total


# ---------------------------------------------------------------------------------------------- the chains
class _Builder:
    def __init__(self, hp, B, L, mode):
        self.hp, self.B, self.L, self.mode = hp, B, L, mode  # mode: None or (seed, p_front, p_trans)

    def drop(self, step, k, F):
        """The descriptor fields of dropout site 2 s + k of step s (none in eval mode or at rate 0)."""
        if self.mode is None:
            return {}
        seed, pf, pt = self.mode
        p = pf if F > 1 else pt
        if math.floor(float(np.float32(p)) * 2.0**32) == 0:
            return {}
        return dict(seed=int(seed), p=float(p), site=2 * step + k)

    @staticmethod
    def linear(X, M, K, W, N, out, bias=None, resid=None, gelu_out=None, drop=None):
        """out[M, N] = X[M, K] W[N, K]^T (+ bias) (+ resid), GELU of it into gelu_out: the pass's train_gemm."""
        return Call("gemm", [X, W, out, bias, resid, gelu_out],
                    dict(M=M, N=N, K=K, a_rs=K, a_cs=1, b_rs=K, b_cs=1, ldc=N, ldr=N, splits=1, scale=1.0,
                         **(drop or {})), ("train_gemm",))

    @staticmethod
    def grad_input(dY, M, N, W, K, dX, resid=None):
        """dX[M, K] = dY[M, N] W[N, K] (+ resid): train_gemm_dx."""
        return Call("gemm", [dY, W, dX, None, resid], dict(M=M, N=K, K=N, a_rs=N, a_cs=1, b_rs=1, b_cs=K, ldc=K, ldr=K,
                                                           splits=1, scale=1.0), ("train_gemm_dx",))

    @staticmethod
    def grad_weight(dY, M, N, X, K, dW, splits=0):
        """dW[N, K] = dY[M, N]^T X[M, K] in the pass's split policy (splits 0): train_gemm_dw (+ train_reduce)."""
        parts = gemm_parts(M, splits or dw_splits(M, N, K))
        return Call("gemm", [dY, X, dW, None, None, None, ("S", "part")],
                    dict(M=N, N=K, K=M, a_rs=1, a_cs=N, b_rs=1, b_cs=K, ldc=K, ldr=K, splits=splits, scale=1.0),
                    ("train_gemm_dw",) + (("train_reduce",) if parts > 1 else ()))

    @staticmethod
    def colsum(A, M, N, scale, out, B=None, rs=None, shift=None):
        """out[N] = scale sum_m A (B) (rs[m]) (A centred by shift); scale: (fp32, exact) or exact 1.0."""
        f32, exact = scale if isinstance(scale, tuple) else (scale, scale)
        return Call("colsum", [A, B, rs, ("S", "part"), out, shift], dict(M=M, N=N, splits=0, scale=f32),
                    ("train_colsum", "train_reduce"), dict(scale=exact))

    @staticmethod
    def call(op, slots, exact=None, **desc):
        return Call(op, slots, desc, (PROFILE[op],), exact or {})

    def bn(self, s, p, stats, ch):
        """The four BatchNorm slots of the entry at table index p: running statistics (eval mode) or the step's batch
        statistics in the store."""
        if self.mode is None:
            return [("P", p), ("P", p + 1), ("P", p + 2), ("P", p + 3)]
        return [("P", p), ("P", p + 1), s.A(stats + ".mean"), s.A(stats + ".var")]

    def stats(self, s, x, N, ch, p, stats):
        """Training mode: the batch mean and biased variance of x [N, ch] and the running statistics moved to them."""
        mean, var = s.A(stats + ".mean"), s.A(stats + ".var")
        inv_n = (_f32(1.0 / N), 1.0 / N)
        return [self.colsum(x, N, ch, inv_n, mean), self.colsum(x, N, ch, inv_n, var, shift=mean),
                self.call("reduce", [mean, ("R", p + 2)], M=ch, splits=1, scale=0.1, beta=0.9,
                          exact=dict(scale=0.1, beta=0.9)),
                self.call("reduce", [var, ("R", p + 3)], M=ch, splits=1, scale=_f32(0.1 * N / (N - 1)), beta=0.9,
                          exact=dict(scale=0.1 * N / (N - 1), beta=0.9))]

    def img(self, s):
        B, L, C, F = self.B, self.L, s.C, s.F
        if s.kind == "stem":  # the [B, L, 128] input: F output frequencies of 4, one channel
            return dict(B=B, F=F, S=4, L=L, C=1, sb=L * 4 * F, sf=1, st=4 * F, sc=0)
        return dict(B=B, F=F // 2, S=2, L=L, C=C, sb=F * L * C, sf=L * C, st=C, sc=1)

    def seqs(self, s):
        B, L, heads = self.B, self.L, s.C // 32
        if s.kind == "attn_freq":  # sequences (b, t) over the F planes
            return dict(seqs=B * L, n=s.F, heads=heads, seq_in=L, s_out=s.F * L, s_in=1, s_pos=L)
        return dict(seqs=B * s.F, n=L, heads=heads, seq_in=1, s_out=L, s_in=0, s_pos=1)

    # ---- forward
    def forward(self, s, nxt):
        M, C, p, BL, Fs = self.B * self.L * s.F, s.C, s.p, self.B * self.L, self.hp["spect_dim"]
        S = lambda n: ("S", n)  # noqa: E731
        P = lambda i: ("P", i)  # noqa: E731
        ch = []
        if s.kind == "stem":
            if self.mode is not None:
                ch += self.stats(s, s.A("in"), BL, Fs, p, "bn1")
            ch.append(self.call("im2col", [s.A("in"), S("big")] + self.bn(s, p, "bn1", Fs), flag=1, **self.img(s)))
            ch.append(self.linear(S("big"), M, 12, P(p + 5), C, s.A("z")))
            if self.mode is not None:
                ch += self.stats(s, s.A("z"), M, C, p + 6, "bn2")
            ch.append(self.call("bn_gelu_fwd", [s.A("z")] + self.bn(s, p + 6, "bn2", C) + [nxt], M=M * C, C=C))
        elif s.kind.startswith("attn"):
            heads = C // 32
            ch += [self.call("rms_fwd", [s.A("in"), P(p + 1), s.A("xn"), s.A("inv")], M=M, C=C),
                   self.linear(s.A("xn"), M, C, P(p + 2), 3 * C, s.A("qkv")),
                   self.linear(s.A("xn"), M, C, P(p + 3), heads, s.A("gate"), bias=P(p + 4)),
                   self.call("rope", [s.A("qkv"), P(p)], M=M, C=C, L=self.L, F=s.F,
                             posmode=int(s.kind == "attn_freq"), flag=0),
                   self.call("attn_fwd", [s.A("qkv"), s.A("o"), s.A("lse")], **self.seqs(s),
                             **self.drop(s.index, 0, s.F)),
                   self.call("gate_fwd", [s.A("o"), s.A("gate"), S("s1")], M=M, C=C),
                   self.linear(S("s1"), M, C, P(p + 5), C, nxt, resid=s.A("in"), drop=self.drop(s.index, 1, s.F))]
        elif s.kind == "ffn":
            H = s.mult * C
            ch += [self.call("rms_fwd", [s.A("in"), P(p), s.A("xn"), s.A("inv")], M=M, C=C),
                   self.linear(s.A("xn"), M, C, P(p + 1), H, s.A("h"), bias=P(p + 2), gelu_out=s.A("a"),
                               drop=self.drop(s.index, 0, s.F)),
                   self.linear(s.A("a"), M, H, P(p + 3), C, nxt, bias=P(p + 4), resid=s.A("in"),
                               drop=self.drop(s.index, 1, s.F))]
        elif s.kind == "conv":
            Mo = M // 2
            ch += [self.call("im2col", [s.A("in"), S("big")], flag=0, **self.img(s)),
                   self.linear(S("big"), Mo, 6 * C, P(p), 2 * C, s.A("z"))]
            if self.mode is not None:
                ch += self.stats(s, s.A("z"), Mo, 2 * C, p + 1, "bn2")
            ch.append(self.call("bn_gelu_fwd", [s.A("z")] + self.bn(s, p + 1, "bn2", 2 * C) + [nxt], M=Mo * 2 * C,
                                C=2 * C))
        elif s.kind == "linear":
            ch += [self.call("concat", [s.A("in"), s.A("xl")], B=self.B, F=s.F, L=self.L, C=C, flag=0),
                   self.linear(s.A("xl"), BL, C * s.F, P(p), self.hp["transformer_dim"], nxt, bias=P(p + 1))]
        else:
            ch += [self.call("rms_fwd", [s.A("in"), P(p), s.A("xn"), s.A("inv")], M=M, C=C),
                   self.linear(s.A("xn"), M, C, P(p + 1), 2, S("s1"), bias=P(p + 2)),
                   self.call("head_fwd", [S("s1"), ("X", "beat"), ("X", "down")], M=M,
                             flag=int(bool(self.hp["sum_head"])))]
        return ch

    # ---- backward
    def rms_backward(self, s, gamma, dxn, M, add):
        sc = (float(np.sqrt(np.float32(s.C))), math.sqrt(s.C))  # sqrtf(C)
        return [self.call("rms_bwd", [dxn, s.A("in"), s.A("inv"), ("P", gamma), ("S", "dcur")], M=M, C=s.C,
                          flag=int(add)),
                self.colsum(dxn, M, s.C, sc, ("G", gamma), B=s.A("in"), rs=s.A("inv"))]

    def backward(self, s):
        M, C, p, BL, Fs = self.B * self.L * s.F, s.C, s.p, self.B * self.L, self.hp["spect_dim"]
        S = lambda n: ("S", n)  # noqa: E731
        P, G = (lambda i: ("P", i)), (lambda i: ("G", i))
        ch = []
        if s.kind == "head":
            ch += [self.call("head_bwd", [("X", "dbeat"), ("X", "ddown"), S("s1")], M=M,
                             flag=int(bool(self.hp["sum_head"]))),
                   self.grad_weight(S("s1"), M, 2, s.A("xn"), C, G(p + 1)),
                   self.colsum(S("s1"), M, 2, 1.0, G(p + 2)),
                   self.grad_input(S("s1"), M, 2, P(p + 1), C, S("s2"))]
            ch += self.rms_backward(s, p, S("s2"), M, False)
        elif s.kind.startswith("attn"):
            heads = C // 32
            d1 = self.drop(s.index, 1, s.F)
            ch.append(self.call("gate_fwd", [s.A("o"), s.A("gate"), S("s1")], M=M, C=C))
            dy = S("dcur")
            if d1:  # to_out's dropout: the masked gradient to its GEMMs (in dqkv), the plain one to the residual path
                ch.append(self.call("reduce", [S("dcur"), S("dqkv")], M=M * C, splits=1, scale=1.0, **d1))
                dy = S("dqkv")
            ch += [self.grad_weight(dy, M, C, S("s1"), C, G(p + 5)),
                   self.grad_input(dy, M, C, P(p + 5), C, S("s2")),
                   self.call("gate_bwd", [S("s2"), s.A("o"), s.A("gate"), S("hd1"), S("hd2")], M=M, C=C)]
            for op in ("attn_dq", "attn_dkv"):
                ch.append(self.call(op, [s.A("qkv"), S("s2"), s.A("lse"), S("hd2"), S("dqkv")], **self.seqs(s),
                                    **self.drop(s.index, 0, s.F)))
            ch += [self.call("rope", [S("dqkv"), P(p)], M=M, C=C, L=self.L, F=s.F,
                             posmode=int(s.kind == "attn_freq"), flag=1),
                   self.grad_weight(S("dqkv"), M, 3 * C, s.A("xn"), C, G(p + 2)),
                   self.grad_weight(S("hd1"), M, heads, s.A("xn"), C, G(p + 3)),
                   self.colsum(S("hd1"), M, heads, 1.0, G(p + 4)),
                   self.grad_input(S("dqkv"), M, 3 * C, P(p + 2), C, S("s1")),
                   self.grad_input(S("hd1"), M, heads, P(p + 3), C, S("s1"), resid=S("s1"))]
            ch += self.rms_backward(s, p + 1, S("s1"), M, True)
        elif s.kind == "ffn":
            H = s.mult * C
            d1 = self.drop(s.index, 1, s.F)
            dy = S("dcur")
            if d1:  # net.5's dropout: the masked gradient to net.4, the plain one to the residual path
                ch.append(self.call("reduce", [S("dcur"), S("s2")], M=M * C, splits=1, scale=1.0, **d1))
                dy = S("s2")
            ch += [self.grad_weight(dy, M, C, s.A("a"), H, G(p + 3)),
                   self.colsum(dy, M, C, 1.0, G(p + 4)),
                   self.grad_input(dy, M, C, P(p + 3), H, S("big")),
                   self.call("gelu_bwd", [S("big"), s.A("h"), S("big")], M=M * H, **self.drop(s.index, 0, s.F)),
                   self.grad_weight(S("big"), M, H, s.A("xn"), C, G(p + 1)),
                   self.colsum(S("big"), M, H, 1.0, G(p + 2)),
                   self.grad_input(S("big"), M, H, P(p + 1), C, S("s1"))]
            ch += self.rms_backward(s, p, S("s1"), M, True)
        elif s.kind == "linear":
            D, K = self.hp["transformer_dim"], C * s.F
            ch += [self.grad_weight(S("dcur"), BL, D, s.A("xl"), K, G(p)),
                   self.colsum(S("dcur"), BL, D, 1.0, G(p + 1)),
                   self.grad_input(S("dcur"), BL, D, P(p), K, S("s1")),
                   self.call("concat", [S("s1"), S("dcur")], B=self.B, F=s.F, L=self.L, C=C, flag=1)]
        else:  # conv, stem: the convolution's output is Mo rows of Co channels, im2col has K = Ci S 3 columns
            stem = s.kind == "stem"
            g = self.img(s)
            Co, K = (C if stem else 2 * C), g["C"] * g["S"] * 3
            bn2, wc = (p + 6, p + 5) if stem else (p + 1, p)
            Mo = g["B"] * g["F"] * g["L"]
            b2 = self.bn(s, bn2, "bn2", Co)
            ch += [self.call("bn_gelu_bwd", [S("dcur"), s.A("z")] + b2 + [S("s1"), S("s2")], M=Mo * Co, C=Co),
                   self.colsum(S("s1"), Mo, Co, 1.0, S("hd1"), B=s.A("z")),
                   self.colsum(S("s1"), Mo, Co, 1.0, S("hd2")),
                   self.call("bn_grads", [S("hd1"), S("hd2")] + b2 + [G(bn2), G(bn2 + 1)], C=Co)]
            if self.mode is not None:  # batch statistics: the terms through the mean and the variance
                ch.append(self.call("bn_scale", [S("s1")] + b2 + [S("s2"), s.A("z"), S("hd1"), S("hd2")], M=Mo * Co,
                                    C=Co, bn_n=Mo))
            b1 = self.bn(s, p, "bn1", Fs) if stem else []
            ch += [self.call("im2col", [s.A("in"), S("big")] + b1, flag=int(stem), **g),
                   self.grad_weight(S("s2"), Mo, Co, S("big"), K, G(wc)),
                   self.grad_input(S("s2"), Mo, Co, P(wc), K, S("big")),
                   self.call("col2im", [S("big"), S("s1") if stem else S("dcur")], **g)]
            if stem:
                batch = [s.A("in"), S("hd1"), S("hd2")] if self.mode is not None else []
                ch += [self.colsum(S("s1"), BL, Fs, 1.0, S("hd1"), B=s.A("in")),
                       self.colsum(S("s1"), BL, Fs, 1.0, S("hd2")),
                       self.call("bn_grads", [S("hd1"), S("hd2")] + b1 + [G(p), G(p + 1)], C=Fs),
                       self.call("bn_scale", [S("s1")] + b1 + [("X", "dspect")] + batch, M=BL * Fs, C=Fs,
                                 **(dict(bn_n=BL) if batch else {}))]
        return ch


def train_steps(hp, B, L, mode=None):
    """The steps of one training forward and backward over a [B, L, 128] batch; mode None (eval mode) or (seed,
    dropout_frontend, dropout_transformer)."""
    regs, _ = layout(hp, B, L, mode is not None)
    b = _Builder(hp, B, L, mode)
    steps, p = [], 0
    for i, ((kind, m, C, F, mult), names) in enumerate(zip(_layer_list(hp), table(hp))):
        steps.append(TrStep(i, kind, m, C, F, mult, p, regs[i]))
        p += len(names)
    for i, s in enumerate(steps):
        nxt = steps[i + 1].A("in") if i + 1 < len(steps) else None
        s.fwd = b.forward(s, nxt)
        s.bwd = b.backward(s)
    return steps


def step_outputs(steps, s, direction):
    """The references a step's chain must reproduce: forward, every stored activation but its input, the next step's
    input (the head: the logits) and its batch statistics; backward, its gradient entries and the gradient at its
    input (dcur, the stem: dspect) over the input's floats."""
    if direction == "fwd":
        out = [s.A(k) for k in s.regions if k != "in"]
        return out + ([steps[s.index + 1].A("in")] if s.index + 1 < len(steps) else [("X", "beat"), ("X", "down")])
    out = sorted({r for c in s.bwd for r in c.slots if r is not None and r[0] == "G"}, key=lambda r: r[1])
    return out + [("X", "dspect") if s.kind == "stem" else ("D", s.regions["in"][1])]


# ---------------------------------------------------------------------------------------------- mutations
def mutations(hp, B, L, steps, mode):
    """(what, step index, "fwd" | "bwd", the chain with one wrong but valid argument, bitwise_only): the wiring errors
    the ties must catch, one per kind of step.  bitwise_only: the same value in exact arithmetic (another dW split),
    which only the bitwise tie sees."""
    out = []
    train = mode is not None
    dropt = train and bool(_Builder(hp, 1, 1, mode).drop(0, 0, 1))

    def first(kind, pred=lambda s: True):
        return next((s for s in steps if s.kind == kind and pred(s)), None)

    def mutate(what, s, d, pick, bitwise_only=False, **kw):
        chain = copy.deepcopy(getattr(s, d))
        c = [c for c in chain if pick(c)][0]
        for k, v in kw.items():
            if k == "slots":
                c.slots = v(c.slots)
            elif v is None:
                c.desc.pop(k, None)
            else:
                c.desc[k] = v
            c.exact.pop(k, None)
        out.append((what, s.index, d, chain, bitwise_only))

    af, at, main = first("attn_freq"), first("attn_time"), first("attn_time", lambda s: s.F == 1)
    ffm = first("ffn", lambda s: s.F == 1)
    if af is not None:
        mutate("posmode 0 in attnF's RoPE", af, "fwd", lambda c: c.op == "rope", posmode=0)
        mutate("attnT's TrSeqs in attnF", af, "fwd", lambda c: c.op == "attn_fwd",
               **_Builder(hp, B, L, mode).seqs(at))
    mutate("RoPE not inverted in the backward", main, "bwd", lambda c: c.op == "rope", flag=0)
    mutate("gamma column sum at scale 1", ffm, "bwd", lambda c: c.op == "colsum" and c.slots[1] is not None, scale=1.0)
    mutate("rms_bwd without add", main, "bwd", lambda c: c.op == "rms_bwd", flag=0)
    stem = steps[0]
    mutate("the stem's im2col without bn1d", stem, "bwd", lambda c: c.op == "im2col", flag=0,
           slots=lambda sl: sl[:2])
    if train:
        mutate("bn1's statistics for bn2", stem, "fwd", lambda c: c.op == "bn_gelu_fwd",
               slots=lambda sl: sl[:3] + [stem.A("bn1.mean"), stem.A("bn1.var")] + sl[5:])
        conv = first("conv")
        mutate("eval-mode bn_scale", conv, "bwd", lambda c: c.op == "bn_scale", bn_n=None, slots=lambda sl: sl[:6])
    else:
        mutate("bn1d's running statistics for bn2d", stem, "fwd", lambda c: c.op == "bn_gelu_fwd",
               slots=lambda sl: sl[:3] + [("P", stem.p + 2), ("P", stem.p + 3)] + sl[5:])
    mutate("concat backward off", first("linear"), "bwd", lambda c: c.op == "concat", flag=0)
    mutate("sum_head flipped", steps[-1], "bwd", lambda c: c.op == "head_bwd", flag=int(not hp["sum_head"]))
    if dropt:
        s = ffm
        mutate("site k swapped in the FFN", s, "fwd", lambda c: c.op == "gemm" and c.slots[5] is not None,
               site=2 * s.index + 1)
        mutate("the next step's site in the attention", main, "fwd", lambda c: c.op == "attn_fwd",
               site=2 * main.index + 2)
        mutate("the FFN's masked and plain gradients swapped", s, "bwd", lambda c: c.op == "gemm" and
               c.prod == ("train_gemm_dx",) and c.slots[2] == ("S", "big"),
               slots=lambda sl: [("S", "dcur")] + sl[1:])
    # bitwise only: another split of the widest frontend (or main) weight gradient
    for s in steps:
        c = next((c for c in s.bwd if c.prod[0] == "train_gemm_dw" and dw_splits(c.desc["K"], c.desc["M"],
                                                                                     c.desc["N"]) > 1), None)
        if c is not None:
            k = dw_splits(c.desc["K"], c.desc["M"], c.desc["N"])
            parts = (gemm_parts(c.desc["K"], k), gemm_parts(c.desc["K"], k // 2))  # another partition of the rows
            assert parts[0] != parts[1]
            mutate(f"dW in {parts[1]} parts for {parts[0]}", s, "bwd", lambda x, c=c: x == c, bitwise_only=True,
                   splits=k // 2)
            break
    return out



# ---------------------------------------------------------------------------------------------- memory of a pass
class Mem:
    """The arrays a pass's references name, as flat tensors: the store, the table entries (P, G, R: lists indexed like
    the table, None where absent), the scratch and the logits.  ("D", n): the first n floats of dcur."""

    def __init__(self, store, P, G, R, S, X):
        self.store, self.P, self.G, self.R, self.S, self.X = store, P, G, R, S, X

    def get(self, ref):
        if ref is None:
            return None
        k = ref[0]
        if k == "A":
            return self.store[ref[1] : ref[1] + ref[2]]
        if k == "D":
            return self.S["dcur"][: ref[1]]
        if k == "S":
            return self.S.get(ref[1])  # float64 runs keep no partials
        if k == "X":
            return self.X.get(ref[1])
        return {"P": self.P, "G": self.G, "R": self.R}[k][ref[1]]


# ---------------------------------------------------------------------------------------------- float64 evaluation
def dropout_mask(desc, n, e0=0):
    """keep / (1 - p) in float64 of elements e0 .. e0 + n of the call's dropout site, or None without dropout."""
    from oracle import philox

    if not desc.get("p") or philox.threshold(desc["p"]) == 0:
        return None
    keep = philox.keep(desc["seed"], desc["site"], desc["p"], n, e0 + desc.get("e0", 0))
    return torch.from_numpy(keep.astype(np.float64) * philox.scale(desc["p"]))


def _rope_tables(freqs, pos):
    """cos, sin [rows, 16] as the reference forms them: angle fl32(pos fl32(freq)), its cos and sin in fp32."""
    ang = pos.float()[:, None] * freqs.float()[None, :]
    return ang.cos().double(), ang.sin().double()


class Eval64:
    """Runs calls on a Mem of float64 tensors: each op restated in float64 from the hook contract of
    include/beatthis.h (the sums, BatchNorms and GELUs exact; RoPE on the reference's fp32 angle tables, as
    oracle.rope; dropout from oracle.philox), so a chain composed over a pass is the reference model's value."""

    ATTN_ROWS = 1 << 22  # probabilities per block of sequences

    def __init__(self, mem):
        self.m = mem

    def run(self, chain):
        for c in chain:
            getattr(self, "_" + c.op)([self.m.get(r) for r in c.slots], {**c.desc, **c.exact})

    @staticmethod
    def _mat(t, rows, cols, rs, cs):
        return torch.as_strided(t, (rows, cols), (rs, cs))

    def _gemm(self, a, d):
        a = a + [None] * (7 - len(a))
        M, N, K = d["M"], d["N"], d["K"]
        y = self._mat(a[0], M, K, d["a_rs"], d["a_cs"]) @ self._mat(a[1], N, K, d["b_rs"], d["b_cs"]).T
        if a[3] is not None:
            y = y + a[3][:N]
        mask = dropout_mask(d, M * N)
        if a[5] is not None:
            g = torch.nn.functional.gelu(y)
            self._mat(a[5], M, N, d["ldc"], 1).copy_(g if mask is None else g * mask.view(M, N))
        elif mask is not None:
            y = y * mask.view(M, N)
        if a[4] is not None:
            y = y + self._mat(a[4], M, N, d["ldr"], 1)
        self._mat(a[2], M, N, d["ldc"], 1).copy_(y)

    def _reduce(self, a, d):
        n, Z = d["M"], d["splits"]
        y = d["scale"] * a[0][: Z * n].view(Z, n).sum(0)
        mask = dropout_mask(d, n)
        if mask is not None:
            y = y * mask
        if d.get("beta"):
            y = y + d["beta"] * a[1][:n]
        a[1][:n] = y

    def _colsum(self, a, d):
        a = a + [None] * (6 - len(a))
        M, N = d["M"], d["N"]
        A = a[0][: M * N].view(M, N)
        if a[5] is not None:
            A = A - a[5][:N]
            t = A * a[1][: M * N].view(M, N) if a[1] is not None else A * A
        else:
            t = A * a[1][: M * N].view(M, N) if a[1] is not None else A
        if a[2] is not None:
            t = t * a[2][:M, None]
        a[4][:N] = d["scale"] * t.sum(0)

    def _rms_fwd(self, a, d):
        M, C = d["M"], d["C"]
        x = a[0][: M * C].view(M, C)
        inv = 1.0 / x.norm(dim=1).clamp_min(1e-12)
        a[2][: M * C] = (x * inv[:, None] * math.sqrt(C) * a[1][:C]).reshape(-1)
        a[3][:M] = inv

    def _rms_bwd(self, a, d):
        M, C = d["M"], d["C"]
        dxn, x, inv = a[0][: M * C].view(M, C), a[1][: M * C].view(M, C), a[2][:M]
        du = dxn * math.sqrt(C) * a[3][:C]
        u = x * inv[:, None]
        clamped = (x.norm(dim=1) < 1e-12)[:, None]
        dx = torch.where(clamped, du * inv[:, None], inv[:, None] * (du - u * (u * du).sum(1, keepdim=True)))
        out = a[4][: M * C].view(M, C)
        out.copy_(out + dx if d.get("flag") else dx)

    @staticmethod
    def _bn(a, C):
        """scale, shift, mean, variance of a BatchNorm; eps 1e-5 exactly (the kernels' 1e-5f is a rounding point)."""
        w, b, rm, rv = (t[:C] for t in a)
        s = w / torch.sqrt(rv + 1e-5)
        return s, b - rm * s, rm, rv

    def _bn_gelu_fwd(self, a, d):
        n, C = d["M"], d["C"]
        s, t, _, _ = self._bn(a[1:5], C)
        c = torch.arange(n) % C
        a[5][:n] = torch.nn.functional.gelu(a[0][:n] * s[c] + t[c])

    def _bn_gelu_bwd(self, a, d):
        from train_kernels_reference import gelu_grad

        n, C = d["M"], d["C"]
        s, t, _, _ = self._bn(a[2:6], C)
        c = torch.arange(n) % C
        dbn = a[0][:n] * gelu_grad(a[1][:n] * s[c] + t[c])
        a[6][:n] = dbn
        a[7][:n] = dbn * s[c]

    def _bn_grads(self, a, d):
        C = d["C"]
        _, _, rm, rv = self._bn(a[2:6], C)
        if a[6] is not None:
            a[6][:C] = (a[0][:C] - rm * a[1][:C]) / torch.sqrt(rv + 1e-5)
        if a[7] is not None:
            a[7][:C] = a[1][:C]

    def _bn_scale(self, a, d):
        n, C = d["M"], d["C"]
        a = a + [None] * (9 - len(a))
        s, _, rm, rv = self._bn(a[1:5], C)
        c = torch.arange(n) % C
        g = a[0][:n]
        if a[6] is None:
            a[5][:n] = g * s[c]
            return
        r = torch.sqrt(rv + 1e-5)
        xhat = (a[6][:n] - rm[c]) / r[c]
        sgx = (a[7][:C] - rm * a[8][:C]) / r  # sum g xhat
        a[5][:n] = s[c] * (g - a[8][:C][c] / d["bn_n"] - xhat * sgx[c] / d["bn_n"])

    def _gelu_bwd(self, a, d):
        from train_kernels_reference import gelu_grad

        n = d["M"]
        dh = a[0][:n] * gelu_grad(a[1][:n])
        mask = dropout_mask(d, n)
        a[2][:n] = dh if mask is None else dh * mask

    @staticmethod
    def _img(d):
        return (d["B"], d["F"], d["S"], d["L"], d["C"], d["sb"], d["sf"], d["st"], d["sc"])

    def _im2col(self, a, d):
        from train_kernels_reference import im2col_ref

        g = self._img(d)
        n_in = (d["B"] - 1) * d["sb"] + (d["F"] * d["S"] - 1) * d["sf"] + (d["L"] - 1) * d["st"] + (d["C"] - 1) * d["sc"] + 1
        x = a[0][:n_in]
        if d.get("flag"):  # the 1-d BatchNorm of the input's F S frequencies, at stride sf = 1 (the stem's input)
            assert d["sf"] == 1
            s, t, _, _ = self._bn(a[2:6], d["F"] * d["S"])
            f = torch.arange(n_in) % (d["F"] * d["S"])
            x = x * s[f] + t[f]
        col, _ = im2col_ref(x, g)
        a[1][: col.numel()] = col.reshape(-1)

    def _col2im(self, a, d):
        from train_kernels_reference import col2im_ref

        g = self._img(d)
        n_in = (d["B"] - 1) * d["sb"] + (d["F"] * d["S"] - 1) * d["sf"] + (d["L"] - 1) * d["st"] + (d["C"] - 1) * d["sc"] + 1
        rows = d["B"] * d["F"] * d["L"]
        din, _ = col2im_ref(a[0][: rows * d["C"] * d["S"] * 3], g, n_in)
        ok = ~torch.isnan(din)
        a[1][:n_in][ok] = din[ok]

    def _concat(self, a, d):
        from train_kernels_reference import concat_ref

        n = d["B"] * d["F"] * d["L"] * d["C"]
        a[1][:n] = concat_ref(a[0][:n], d["B"], d["F"], d["L"], d["C"], d.get("flag", 0))

    def _rope(self, a, d):
        M, C = d["M"], d["C"]
        x = a[0][: M * 3 * C].view(M, 3 * C)
        m = torch.arange(M)
        pos = m % d["L"] if d["posmode"] == 0 else (m // d["L"]) % d["F"]
        co, si = _rope_tables(a[1][:16], pos)
        co, si = co.repeat(1, 2 * C // 32), si.repeat(1, 2 * C // 32)  # pair i of each head of q, then of k
        if d.get("flag"):
            si = -si
        x0, x1 = x[:, 0 : 2 * C : 2].clone(), x[:, 1 : 2 * C : 2].clone()
        x[:, 0 : 2 * C : 2] = x0 * co - x1 * si
        x[:, 1 : 2 * C : 2] = x1 * co + x0 * si

    def _gate_fwd(self, a, d):
        M, C = d["M"], d["C"]
        sg = torch.sigmoid(a[1][: M * C // 32].view(M, C // 32)).repeat_interleave(32, 1)
        a[2][: M * C] = (a[0][: M * C].view(M, C) * sg).reshape(-1)

    def _gate_bwd(self, a, d):
        M, C = d["M"], d["C"]
        H = C // 32
        dG, O = a[0][: M * C].view(M, C), a[1][: M * C].view(M, C)
        sg = torch.sigmoid(a[2][: M * H].view(M, H))
        a[3][: M * H] = ((dG * O).view(M, H, 32).sum(-1) * sg * (1 - sg)).reshape(-1)
        dO = dG * sg.repeat_interleave(32, 1)
        a[4][: M * H] = (dO * O).view(M, H, 32).sum(-1).reshape(-1)
        dG.copy_(dO)

    def _head_fwd(self, a, d):
        M = d["M"]
        o = a[0][: 2 * M].view(M, 2)
        a[1][:M] = o[:, 0] + o[:, 1] if d.get("flag") else o[:, 0]
        a[2][:M] = o[:, 1]

    def _head_bwd(self, a, d):
        M = d["M"]
        db, dd = a[0][:M], a[1][:M]
        a[2][: 2 * M] = torch.stack([db, dd + db if d.get("flag") else dd], 1).reshape(-1)

    # ---- attention over TrSeqs, in blocks of sequences
    def _blocks(self, d):
        from train_kernels_reference import seq_rows

        rows = seq_rows(d["seqs"], d["n"], d["seq_in"], d["s_out"], d["s_in"], d["s_pos"])
        step = max(1, self.ATTN_ROWS // (d["heads"] * d["n"] * d["n"]))
        for s0 in range(0, d["seqs"], step):
            yield s0, rows[s0 : s0 + step]

    @staticmethod
    def _heads(t, rows, H, off, width):
        n_tok = int(rows.max()) + 1
        x = t[: n_tok * width].view(n_tok, width)[rows.reshape(-1), off : off + 32 * H]
        return x.reshape(rows.shape[0], rows.shape[1], H, 32).permute(0, 2, 1, 3)  # [seqs, H, n, 32]

    @staticmethod
    def _put(t, rows, H, off, width, v):
        n_tok = int(rows.max()) + 1
        t[: n_tok * width].view(n_tok, width)[rows.reshape(-1), off : off + 32 * H] = (
            v.permute(0, 2, 1, 3).reshape(-1, 32 * H))

    def _scores(self, a, d, rows):
        H = d["heads"]
        C = 32 * H
        q, k, v = (self._heads(a[0], rows, H, i * C, 3 * C) for i in range(3))
        return q, k, v, q @ k.transpose(-1, -2) / math.sqrt(32)

    def _mask(self, d, s0, seqs):
        H, n = d["heads"], d["n"]
        m = dropout_mask(d, seqs * H * n * n, s0 * H * n * n)
        return None if m is None else m.view(seqs, H, n, n)

    def _attn_fwd(self, a, d):
        H = d["heads"]
        for s0, rows in self._blocks(d):
            q, k, v, s = self._scores(a, d, rows)
            lse = torch.logsumexp(s, -1)
            P = torch.exp(s - lse[..., None])
            m = self._mask(d, s0, rows.shape[0])
            self._put(a[1], rows, H, 0, 32 * H, (P if m is None else P * m) @ v)
            n_tok = int(rows.max()) + 1
            a[2][: n_tok * H].view(n_tok, H)[rows.reshape(-1)] = lse.permute(0, 2, 1).reshape(-1, H)

    def _attn_bwd(self, a, d, dq):
        H = d["heads"]
        C = 32 * H
        for s0, rows in self._blocks(d):
            q, k, v, s = self._scores(a, d, rows)
            n_tok = int(rows.max()) + 1
            per_row = lambda t: t[: n_tok * H].view(n_tok, H)[rows.reshape(-1)].view(*rows.shape, H).permute(0, 2, 1)  # noqa: E731
            P = torch.exp(s - per_row(a[2])[..., None])
            do = self._heads(a[1], rows, H, 0, C)
            m = self._mask(d, s0, rows.shape[0])
            dp = do @ v.transpose(-1, -2)
            if m is not None:
                dp = dp * m
            ds = P * (dp - per_row(a[3])[..., None])
            if dq:
                self._put(a[4], rows, H, 0, 3 * C, ds @ k / math.sqrt(32))
            else:
                self._put(a[4], rows, H, C, 3 * C, ds.transpose(-1, -2) @ q / math.sqrt(32))
                self._put(a[4], rows, H, 2 * C, 3 * C, (P if m is None else P * m).transpose(-1, -2) @ do)

    def _attn_dq(self, a, d):
        self._attn_bwd(a, d, True)

    def _attn_dkv(self, a, d):
        self._attn_bwd(a, d, False)


# ---------------------------------------------------------------------------------------------- float64 on real data
ROWS = 2048          # rows of a row-wise op checked (its first ones) on large inputs
ELEMS = 1 << 22      # elements of an elementwise op checked (a prefix of whole channel rows)
PROBS = 1 << 22      # attention probabilities checked (the first sequences)
INPLACE = {"rope": (0,), "gate_bwd": (0,), "gelu_bwd": (0,), "rms_bwd": (4,), "reduce": (1,), "gemm": (4,)}


def _cpu(t, n=None):
    return (t if n is None else t[:n]).detach().double().cpu()


def _note(ratios, op, got, ref, bound):
    from numerics import worst

    r = worst(got, ref, bound)
    ratios[op] = max(ratios.get(op, 0.0), r)
    return r


def check64(c, a, before, ratios, skipped):
    """The call c, just run on the arrays a (before: copies of the slots it updates in place, taken before it ran),
    against its train_kernels_reference restatement within that op's bound, on its own inputs (large ones sampled:
    the first rows, elements or sequences).  ratios[op] keeps the worst ratio; skipped counts the calls no derived
    bound covers (attention with dropout, the batch-statistics terms of bn_scale).  Returns [(what, ratio)]."""
    import train_kernels_reference as R_K

    d, op = c.desc, c.op
    out = []
    if op == "gemm":
        M, N, K = d["M"], d["N"], d["K"]
        Mc = min(M, ROWS)
        ext = lambda rows, cols, rs, cs: (rows - 1) * rs + (cols - 1) * cs + 1  # noqa: E731
        A = torch.as_strided(_cpu(a[0], ext(M, K, d["a_rs"], d["a_cs"])), (Mc, K), (d["a_rs"], d["a_cs"]))
        B = torch.as_strided(_cpu(a[1], ext(N, K, d["b_rs"], d["b_cs"])), (N, K), (d["b_rs"], d["b_cs"]))
        bias = None if len(a) < 4 or a[3] is None else _cpu(a[3], N)
        resid = None
        if len(a) > 4 and a[4] is not None:
            resid = torch.as_strided(_cpu(before.get(4, a[4]), ext(Mc, N, d["ldr"], 1)), (Mc, N), (d["ldr"], 1))
        gel = len(a) > 5 and a[5] is not None
        eff = d["splits"] or dw_splits(K, M, N)
        m = dropout_mask(c.desc, Mc * N)
        ref, e, g, eg = R_K.gemm_ref(A, B, bias, None if m is not None and not gel else resid, splits=eff)
        if m is not None:
            m = m.view(Mc, N)
            if gel:  # the mask applies to gelu_out alone
                g, eg = g * m, R_K.SAFE * (eg * m + R_K.U * (g * m).abs()) + R_K.TINY
            else:    # to the result before resid is added
                y = ref * m + (resid if resid is not None else 0)
                e = R_K.SAFE * (e * m + R_K.U * ((ref * m).abs() + y.abs())) + R_K.TINY
                ref = y
        got = torch.as_strided(_cpu(a[2], ext(Mc, N, d["ldc"], 1)), (Mc, N), (d["ldc"], 1))
        out.append(("C", _note(ratios, op, got, ref, e)))
        if gel:
            got = torch.as_strided(_cpu(a[5], ext(Mc, N, d["ldc"], 1)), (Mc, N), (d["ldc"], 1))
            out.append(("gelu_out", _note(ratios, op, got, g, eg)))
    elif op == "reduce":
        n, Z = d["M"], d["splits"]
        ref, e = R_K.reduce_ref(_cpu(a[0], Z * n).view(Z, n), d["scale"])
        m = dropout_mask(c.desc, n)
        if m is not None:
            ref, e = ref * m, R_K.SAFE * (e * m + R_K.U * (ref * m).abs()) + R_K.TINY
        if d.get("beta"):
            y = ref + d["beta"] * _cpu(before[1], n)
            e = R_K.SAFE * (e + R_K.U * ((d["beta"] * _cpu(before[1], n)).abs() + y.abs())) + R_K.TINY
            ref = y
        out.append(("out", _note(ratios, op, _cpu(a[1], n), ref, e)))
    elif op == "colsum":
        M, N = d["M"], d["N"]
        A = _cpu(a[0], M * N).view(M, N)
        B = None if a[1] is None else _cpu(a[1], M * N).view(M, N)
        rs = None if a[2] is None else _cpu(a[2], M)
        extra = 0.0
        if len(a) > 5 and a[5] is not None:  # centred: one more rounding, the subtraction, per factor
            A = A - _cpu(a[5], N)
            B = A if B is None else B
            extra = 2 * R_K.U * (A * B).abs().sum(0) * abs(d["scale"])
        ref, e, _, _ = R_K.colsum_ref(A, B, rs, colsum_splits(M, N), d["scale"])
        out.append(("out", _note(ratios, op, _cpu(a[4], N), ref, e + R_K.SAFE * extra)))
    elif op == "rms_fwd":
        M, C = d["M"], d["C"]
        Mc = min(M, ROWS)
        xn, e, inv, ei = R_K.rms_fwd_ref(_cpu(a[0], Mc * C).view(Mc, C), _cpu(a[1], C))
        out += [("xn", _note(ratios, op, _cpu(a[2], Mc * C).view(Mc, C), xn, e)), ("inv", _note(ratios, op, _cpu(a[3], Mc), inv, ei))]
    elif op == "rms_bwd":
        M, C = d["M"], d["C"]
        Mc = min(M, ROWS)
        dres = _cpu(before[4], Mc * C).view(Mc, C) if d.get("flag") else None
        ref, e = R_K.rms_bwd_ref(_cpu(a[0], Mc * C).view(Mc, C), _cpu(a[1], Mc * C).view(Mc, C), _cpu(a[2], Mc),
                                 _cpu(a[3], C), dres)
        out.append(("dx", _note(ratios, op, _cpu(a[4], Mc * C).view(Mc, C), ref, e)))
    elif op in ("bn_gelu_fwd", "bn_gelu_bwd", "bn_scale"):
        C = d["C"]
        n = min(d["M"], ELEMS // C * C)
        if op == "bn_gelu_fwd":
            ref, e = R_K.bn_gelu_fwd_ref(_cpu(a[0], n), [_cpu(t, C) for t in a[1:5]], C)
            out.append(("y", _note(ratios, op, _cpu(a[5], n), ref, e)))
        elif op == "bn_gelu_bwd":
            dbn, e1, dz, e2 = R_K.bn_gelu_bwd_ref(_cpu(a[0], n), _cpu(a[1], n), [_cpu(t, C) for t in a[2:6]], C)
            out += [("dbn", _note(ratios, op, _cpu(a[6], n), dbn, e1)), ("dz", _note(ratios, op, _cpu(a[7], n), dz, e2))]
        elif len(a) > 6 and a[6] is not None:
            skipped[op + " (batch statistics)"] += 1
        else:
            ref, e = R_K.bn_scale_ref(_cpu(a[0], n), [_cpu(t, C) for t in a[1:5]], C)
            out.append(("dx", _note(ratios, op, _cpu(a[5], n), ref, e)))
    elif op == "bn_grads":
        C = d["C"]
        dw, e, db = R_K.bn_grads_ref(_cpu(a[0], C), _cpu(a[1], C), [_cpu(t, C) for t in a[2:6]])
        if a[6] is not None:
            out.append(("dw", _note(ratios, op, _cpu(a[6], C), dw, e)))
        if a[7] is not None:
            out.append(("db", _note(ratios, op, _cpu(a[7], C), db, torch.zeros_like(db))))
    elif op == "gelu_bwd":
        n = min(d["M"], ELEMS)
        ref, e = R_K.gelu_bwd_ref(_cpu(before[0], n), _cpu(a[1], n))
        m = dropout_mask(c.desc, n)
        if m is not None:
            ref, e = ref * m, R_K.SAFE * (e * m + R_K.U * (ref * m).abs()) + R_K.TINY
        out.append(("dh", _note(ratios, op, _cpu(a[2], n), ref, e)))
    elif op in ("im2col", "col2im"):
        g = [d[k] for k in ("B", "F", "S", "L", "C", "sb", "sf", "st", "sc")]
        g[0] = 1  # the first batch item
        B_, Fo, S, L, C, sb, sf, st, sc = g
        n_in = (Fo * S - 1) * sf + (L - 1) * st + (C - 1) * sc + 1
        rows, K = Fo * L, C * S * 3
        if op == "im2col":
            bn = [_cpu(t, Fo * S) for t in a[2:6]] if d.get("flag") else None
            ref, e = R_K.im2col_ref(_cpu(a[0], n_in), tuple(g), bn)
            out.append(("col", _note(ratios, op, _cpu(a[1], rows * K).view(rows, K), ref, e)))
        else:
            ref, e = R_K.col2im_ref(_cpu(a[0], rows * K), tuple(g), n_in)
            ok = ~torch.isnan(ref)
            out.append(("din", _note(ratios, op, _cpu(a[1], n_in)[ok], ref[ok], e[ok])))
    elif op == "concat":
        n = d["B"] * d["F"] * d["L"] * d["C"]
        ref = R_K.concat_ref(_cpu(a[0], n), d["B"], d["F"], d["L"], d["C"], d.get("flag", 0))
        out.append(("dst", _note(ratios, op, _cpu(a[1], n), ref, torch.zeros_like(ref))))
    elif op == "rope":
        C = d["C"]
        M = min(d["M"], max(ROWS, d["L"] * (d["F"] if d["posmode"] else 1)))  # rows reaching every position
        ref, e = R_K.rope_ref(_cpu(before[0], M * 3 * C).view(M, 3 * C), _cpu(a[1], 16), d["L"], d["F"], d["posmode"],
                              d.get("flag", 0))
        out.append(("qkv", _note(ratios, op, _cpu(a[0], M * 3 * C).view(M, 3 * C), ref, e)))
    elif op in ("gate_fwd", "gate_bwd"):
        M, C = d["M"], d["C"]
        Mc, H = min(M, ROWS), C // 32
        if op == "gate_fwd":
            ref, e = R_K.gate_fwd_ref(_cpu(a[0], Mc * C).view(Mc, C), _cpu(a[1], Mc * H).view(Mc, H))
            out.append(("G", _note(ratios, op, _cpu(a[2], Mc * C).view(Mc, C), ref, e)))
        else:
            dO, e0, dg, e1, delta, e2 = R_K.gate_bwd_ref(_cpu(before[0], Mc * C).view(Mc, C),
                                                         _cpu(a[1], Mc * C).view(Mc, C), _cpu(a[2], Mc * H).view(Mc, H))
            out += [("dO", _note(ratios, op, _cpu(a[0], Mc * C).view(Mc, C), dO, e0)),
                    ("dg", _note(ratios, op, _cpu(a[3], Mc * H).view(Mc, H), dg, e1)),
                    ("delta", _note(ratios, op, _cpu(a[4], Mc * H).view(Mc, H), delta, e2))]
    elif op == "head_fwd":
        M = d["M"]
        beat, down = R_K.head_fwd_ref(_cpu(a[0], 2 * M), d.get("flag", 0))
        out += [("beat", _note(ratios, op, _cpu(a[1], M), beat, R_K.U * beat.abs())),
                ("down", _note(ratios, op, _cpu(a[2], M), down, torch.zeros_like(down)))]
    elif op == "head_bwd":
        M = d["M"]
        ref = R_K.head_bwd_ref(_cpu(a[0], M), _cpu(a[1], M), d.get("flag", 0))
        out.append(("dout", _note(ratios, op, _cpu(a[2], 2 * M), ref, R_K.U * ref.abs())))
    elif op.startswith("attn"):
        if d.get("p"):
            skipped[op + " (dropout)"] += 1
            return out
        H, n = d["heads"], d["n"]
        C = 32 * H
        seqs = max(1, min(d["seqs"], PROBS // (H * n * n)))
        rows = R_K.seq_rows(seqs, n, d["seq_in"], d["s_out"], d["s_in"], d["s_pos"])
        tok = int(rows.max()) + 1
        qkv = _cpu(a[0], tok * 3 * C).view(tok, 3 * C)
        if op == "attn_fwd":
            O, eO, lse, el = R_K.attn_fwd_ref(qkv, rows, H)
            gO = R_K._heads(_cpu(a[1], tok * C).view(tok, C), rows, H, 0, C)
            gl = _cpu(a[2], tok * H).view(tok, H)[rows.reshape(-1)].reshape(seqs, n, H).permute(0, 2, 1)
            out += [("O", _note(ratios, op, gO, O, eO)), ("lse", _note(ratios, op, gl.reshape(-1, n), lse, el))]
        else:
            dq, edq, dk, edk, dv, edv = R_K.attn_bwd_ref(qkv, _cpu(a[1], tok * C).view(tok, C), _cpu(a[2], tok * H).view(tok, H),
                                                         _cpu(a[3], tok * H).view(tok, H), rows, H)
            got = _cpu(a[4], tok * 3 * C).view(tok, 3 * C)
            if op == "attn_dq":
                out.append(("dq", _note(ratios, op, R_K._heads(got, rows, H, 0, C), dq, edq)))
            else:
                out += [("dk", _note(ratios, op, R_K._heads(got, rows, H, C, C), dk, edk)),
                        ("dv", _note(ratios, op, R_K._heads(got, rows, H, 2 * C, C), dv, edv))]
    return out
