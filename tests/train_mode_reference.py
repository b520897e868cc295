"""float64 restatement of the reference's BeatThis in train() mode, for tests: the eval-mode oracle
(oracle/beat_this_oracle.py) with batch-statistics BatchNorm and the library's dropout masks (oracle/philox.py) at the
reference's four sites per residual branch (roformer.py: Attend's dropout_p, to_out.1, FeedForward net.3 and net.5).

Masks are numbered as include/beatthis.h states: site 2 s + k of step s of the layer list; element row N + col of the
library's token rows (frontend row ((b F + f) L + t), main row b L + t), or ((seq heads + h) n + i) n + j for an
attention's probabilities."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import beat_this_oracle as O
from oracle import philox

BN_EPS = 1e-5


def site(step: int, k: int) -> int:
    """The dropout site of site k of step `step` (the C library's dropout_site)."""
    return 2 * step + k


def mask(seed: int, site_id: int, p: float, shape) -> torch.Tensor | None:
    """keep / (1 - p) as float64 of the site's first prod(shape) elements, shaped; None at rate 0."""
    if philox.threshold(p) == 0:
        return None
    n = int(np.prod(shape))
    return torch.from_numpy(philox.keep(seed, site_id, p, n).astype(np.float64) * philox.scale(p)).view(*shape)


def batchnorm_train(x, sd, p, dim, stats):
    """BatchNorm in training mode over every axis but `dim`: the batch mean and biased variance normalise; stats[p] =
    (mean, biased variance, positions per channel)."""
    dims = [d for d in range(x.ndim) if d != dim]
    mean = x.mean(dim=dims)
    var = x.var(dim=dims, unbiased=False)
    stats[p] = (mean.detach(), var.detach(), x.numel() // x.shape[dim])
    shape = [1] * x.ndim
    shape[dim] = -1
    xhat = (x - mean.view(shape)) / torch.sqrt(var.view(shape) + BN_EPS)
    return xhat * sd[p + ".weight"].view(shape) + sd[p + ".bias"].view(shape)


def attention_train(x, sd, p, heads, pmask, omask):
    """O.attention with P masked after the softmax and to_out's output masked (masks in x's [S, n, *] layout)."""
    q, k, v, gates = O.pre_attention(x, sd, p, heads)
    S, n, _ = x.shape
    if pmask is None:  # no probabilities materialised: long sequences fit
        out = F.scaled_dot_product_attention(q, k, v)
    else:
        out = (torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1]), dim=-1) * pmask.to(v.dtype)) @ v
    out = out * gates.permute(0, 2, 1).unsqueeze(-1).sigmoid()
    out = out.permute(0, 2, 1, 3).reshape(S, n, -1) @ sd[p + ".to_out.0.weight"].T
    return out if omask is None else out * omask.to(out.dtype)


def feedforward_train(x, sd, p, hmask, omask):
    h = O.rmsnorm(x, sd[p + ".net.0.gamma"])
    h = F.gelu(h @ sd[p + ".net.1.weight"].T + sd[p + ".net.1.bias"])
    if hmask is not None:
        h = h * hmask.to(h.dtype)
    out = h @ sd[p + ".net.4.weight"].T + sd[p + ".net.4.bias"]
    return out if omask is None else out * omask.to(out.dtype)


def forward_train(sd: dict, x: torch.Tensor, seed: int, p_front: float, p_trans: float, sum_head=True):
    """BeatThis.forward after .train() on x [B, L, 128] with the library's masks: (beat, downbeat, stats), stats
    {BatchNorm prefix: (batch mean, biased variance, N)}."""
    B, L, _ = x.shape
    stats = {}
    step = 0

    def rows_to(m, layout, Fq):
        """a [B F L, N] (frontend) mask of token rows into the oracle's sequence layout"""
        if m is None:
            return None
        N = m.shape[-1]
        if layout == "freq":  # sequences (b, t) over f
            return m.view(B, Fq, L, N).permute(0, 2, 1, 3).reshape(B * L, Fq, N)
        return m.view(B * Fq, L, N) if layout == "time" else m.view(B, L, N)

    def attn(z, p, heads, layout, Fq, rate):
        nonlocal step
        S, n, C = z.shape
        pm = mask(seed, site(step, 0), rate, (S, heads, n, n))
        om = rows_to(mask(seed, site(step, 1), rate, (S * n, C)), layout, Fq)
        step += 1
        return attention_train(z, sd, p, heads, pm, om)

    def ffn(z, p, layout, Fq, rate):
        nonlocal step
        S, n, C = z.shape
        H = sd[p + ".net.1.weight"].shape[0]
        hm = rows_to(mask(seed, site(step, 0), rate, (S * n, H)), layout, Fq)
        om = rows_to(mask(seed, site(step, 1), rate, (S * n, C)), layout, Fq)
        step += 1
        return feedforward_train(z, sd, p, hm, om)

    h = batchnorm_train(x.transpose(1, 2), sd, "frontend.stem.bn1d", 1, stats)[:, None]
    h = F.conv2d(h, sd["frontend.stem.conv2d.weight"], stride=(4, 1), padding=(0, 1))
    h = F.gelu(batchnorm_train(h, sd, "frontend.stem.bn2d", 1, stats))
    step += 1
    for i in range(3):
        p = f"frontend.blocks.{i}"
        if (p + ".partial.attnF.to_qkv.weight") in sd:
            C, Fq = h.shape[1], h.shape[2]
            heads = C // 32
            z = h.permute(0, 3, 2, 1).reshape(B * L, Fq, C)
            z = z + attn(z, p + ".partial.attnF", heads, "freq", Fq, p_front)
            z = z + ffn(z, p + ".partial.ffF", "freq", Fq, p_front)
            z = z.view(B, L, Fq, C).permute(0, 2, 1, 3).reshape(B * Fq, L, C)
            z = z + attn(z, p + ".partial.attnT", heads, "time", Fq, p_front)
            z = z + ffn(z, p + ".partial.ffT", "time", Fq, p_front)
            h = z.view(B, Fq, L, C).permute(0, 3, 1, 2)
        h = F.conv2d(h, sd[p + ".conv2d.weight"], stride=(2, 1), padding=(0, 1))
        h = F.gelu(batchnorm_train(h, sd, p + ".norm", 1, stats))
        step += 1
    h = h.permute(0, 3, 1, 2).reshape(B, L, -1)
    h = h @ sd["frontend.linear.weight"].T + sd["frontend.linear.bias"]
    step += 1
    D = h.shape[-1]
    n_layers = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transformer_blocks.layers."))
    for layer in range(n_layers):
        p = f"transformer_blocks.layers.{layer}"
        h = attn(h, p + ".0", D // 32, "main", 1, p_trans) + h
        h = ffn(h, p + ".1", "main", 1, p_trans) + h
    h = O.rmsnorm(h, sd["transformer_blocks.norm.gamma"])
    o = h @ sd["task_heads.beat_downbeat_lin.weight"].T + sd["task_heads.beat_downbeat_lin.bias"]
    beat = o[..., 0] + o[..., 1] if sum_head else o[..., 0]
    return beat, o[..., 1], stats


def activation_floats(hp: dict, B: int, L: int) -> int:
    """Floats of the training-mode activation store, counted independently of the library: the eval-mode store (each
    step's saved tensors, as tests/test_gpu_train.py counts them, every allocation rounded up to 4 floats) and, per
    BatchNorm of ch channels, its batch mean and variance of ch rounded up to 4 floats each."""
    def r4(n):
        return (n + 3) // 4 * 4

    BL, D = B * L, hp["transformer_dim"]

    def attn(C, M):
        return r4(M * C) * 2 + r4(M) + r4(3 * M * C) + 2 * r4(M * C // 32) + r4(M * C)

    def ffn(C, M, mult):
        return 2 * r4(M * C) + r4(M) + 2 * r4(M * mult * C)

    n = r4(BL * hp["spect_dim"]) + r4(BL * hp["stem_dim"] * hp["spect_dim"] // 4)
    C, F_ = hp["stem_dim"], hp["spect_dim"] // 4
    bn = 2 * r4(hp["spect_dim"]) + 2 * r4(C)
    for _ in range(3):
        if hp["partial_transformers"]:
            n += 2 * (attn(C, BL * F_) + ffn(C, BL * F_, 4))
        n += r4(BL * F_ * C) + r4(BL * F_ // 2 * 2 * C)
        bn += 2 * r4(2 * C)
        C, F_ = 2 * C, F_ // 2
    n += 2 * r4(BL * C * F_)
    n += hp["n_layers"] * (attn(D, BL) + ffn(D, BL, hp["ff_mult"])) + 2 * r4(BL * D) + r4(BL)
    return n + bn
