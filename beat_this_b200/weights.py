"""Checkpoint tensors -> packed parameters of libbeatthis_sm100.so.

Input is the reference's state_dict layout (reference
beat_this/inference.py:56-87 strips the ``model.`` prefix).  Output is a dict
``name -> contiguous float32 numpy array`` uploaded with ``bt_set_param``.  Folds done here
(all exact re-associations of the reference math):

* eval-mode BatchNorm2d after a bias-free conv (beat_tracker.py:115-123,155-165) -> conv
  weight scale + bias.  BatchNorm1d of the stem (``:113``) is kept as an explicit
  scale/shift because the conv zero-pads in time *after* it.
* RMSNorm ``x/max(|x|,1e-12) * sqrt(dim) * gamma`` (roformer.py:22-32): the
  ``sqrt(dim)*gamma`` factor is folded into the columns of the consuming Linear weights
  (to_qkv, to_gates, FeedForward.net.1, and the head after the final norm).
* Conv2d C->2C k(2,3) weights [2C, C, 2, 3] -> GEMM operand [2C, (df, dt, c)].
* frontend.linear over ``b c f t -> b t (c f)`` (beat_tracker.py:76-77): columns permuted
  from (c, f) to (f, c) so that each frequency plane is one contiguous K slab.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .preprocessing import mel_constants

BN_EPS = 1e-5
ROPE_POSITIONS = 1500  # default maximum chunk length: the reference's inference chunk (inference.py:247)

# BeatThis constructor signature (reference beat_tracker.py:39-49); load_model filters the
# checkpoint's hyper_parameters to these names (inference.py:72-78).
MODEL_HPARAM_DEFAULTS = dict(
    spect_dim=128,
    transformer_dim=512,
    ff_mult=4,
    n_layers=6,
    head_dim=32,
    stem_dim=32,
    dropout={"frontend": 0.1, "transformer": 0.2},
    sum_head=True,
    partial_transformers=True,
)


def filter_hparams(hparams: dict) -> dict:
    hp = dict(MODEL_HPARAM_DEFAULTS)
    hp.update({k: v for k, v in hparams.items() if k in MODEL_HPARAM_DEFAULTS})
    return hp


def strip_prefixes(state_dict: dict) -> dict:
    """replace_state_dict_key(sd, 'model.', '') and the '_orig_mod.' stripping of compiled
    checkpoints (inference.py:83, beat_tracker.py:194-197)."""
    return {k.replace("model.", "").replace("_orig_mod.", ""): v for k, v in state_dict.items()}


def _f64(t):
    return t.detach().to("cpu", torch.float64)


def _bn_fold(sd, prefix):
    scale = _f64(sd[prefix + ".weight"]) / torch.sqrt(_f64(sd[prefix + ".running_var"]) + BN_EPS)
    shift = _f64(sd[prefix + ".bias"]) - _f64(sd[prefix + ".running_mean"]) * scale
    return scale, shift


def _attention(out, sd, src, dst, dim):
    g = _f64(sd[src + ".norm.gamma"]) * math.sqrt(dim)
    out[dst + ".wqkv"] = _f64(sd[src + ".to_qkv.weight"]) * g[None, :]
    # gates run as a GEMM with N padded to 32 (heads <= 32): zero rows / zero bias beyond `heads`
    heads = dim // 32
    wg = torch.zeros(32, dim, dtype=torch.float64)
    wg[:heads] = _f64(sd[src + ".to_gates.weight"]) * g[None, :]
    bg = torch.zeros(32, dtype=torch.float64)
    bg[:heads] = _f64(sd[src + ".to_gates.bias"])
    out[dst + ".wg"], out[dst + ".bg"] = wg, bg
    out[dst + ".wout"] = _f64(sd[src + ".to_out.0.weight"])


def _feedforward(out, sd, src, dst, dim):
    g = _f64(sd[src + ".net.0.gamma"]) * math.sqrt(dim)
    out[dst + ".w1"] = _f64(sd[src + ".net.1.weight"]) * g[None, :]
    out[dst + ".b1"] = _f64(sd[src + ".net.1.bias"])
    out[dst + ".w2"] = _f64(sd[src + ".net.4.weight"])
    out[dst + ".b2"] = _f64(sd[src + ".net.4.bias"])


def rope_tables(freqs: torch.Tensor, positions: int = ROPE_POSITIONS):
    """cos/sin of pos*freqs in fp32, as rotary_embedding_torch computes them (fp32 arange,
    fp32 product, fp32 cos/sin)."""
    pos = torch.arange(positions, dtype=torch.float32)
    ang = pos[:, None] * freqs.detach().to("cpu", torch.float32)[None, :]
    return ang.cos(), ang.sin()


def pack_parameters(state_dict: dict, hparams: dict, rope_positions: int = ROPE_POSITIONS, dtype=np.float32) -> dict:
    """rope_positions: rows of the RoPE tables, the longest chunk the loaded model will run (bt_max_chunk).  Rows
    below 1500 do not depend on it.  dtype: of the arrays; the library takes float32, and float64 keeps the folds
    exact for float64 references of the packed layout (the RoPE tables stay the fp32 values either way)."""
    sd = strip_prefixes(state_dict)
    hp = filter_hparams(hparams)
    out: dict = {}
    # ---- constants of the log-mel frontend and RoPE ---------------------------------------
    out.update(mel_constants())
    freq_keys = [k for k in sd if k.endswith("rotary_embed.freqs")]
    if freq_keys:
        freqs = sd[freq_keys[0]]
    else:  # checkpoints saved without the (constant) RoPE buffer
        d = hp["head_dim"]
        freqs = 1.0 / (10000 ** (torch.arange(0, d, 2).float() / d))
    out["rope.cos"], out["rope.sin"] = rope_tables(freqs, rope_positions)
    # ---- stem ----------------------------------------------------------------------------------
    s1, b1 = _bn_fold(sd, "frontend.stem.bn1d")
    s2, b2 = _bn_fold(sd, "frontend.stem.bn2d")
    out["stem.bn1_scale"], out["stem.bn1_shift"] = s1, b1
    out["stem.w"] = _f64(sd["frontend.stem.conv2d.weight"])[:, 0] * s2[:, None, None]  # [32, 4, 3]
    out["stem.bias"] = b2
    # ---- frontend blocks -------------------------------------------------------------------
    c = hp["stem_dim"]
    for i in range(3):
        src = f"frontend.blocks.{i}"
        if hp["partial_transformers"]:
            _attention(out, sd, src + ".partial.attnF", f"b{i}.attnF", c)
            _feedforward(out, sd, src + ".partial.ffF", f"b{i}.ffF", c)
            _attention(out, sd, src + ".partial.attnT", f"b{i}.attnT", c)
            _feedforward(out, sd, src + ".partial.ffT", f"b{i}.ffT", c)
        s, b = _bn_fold(sd, src + ".norm")
        w = _f64(sd[src + ".conv2d.weight"])  # [2C, C, 2(df), 3(dt)]
        out[f"b{i}.conv.w"] = (w.permute(0, 2, 3, 1) * s[:, None, None, None]).reshape(2 * c, 6 * c)
        out[f"b{i}.conv.bias"] = b
        c *= 2
    f_out = hp["spect_dim"] // 32
    D = hp["transformer_dim"]
    w = _f64(sd["frontend.linear.weight"])  # [D, c*f_out], column = ch*f_out + f
    out["lin.w"] = w.view(D, c, f_out).permute(0, 2, 1).reshape(D, c * f_out)
    out["lin.b"] = _f64(sd["frontend.linear.bias"])
    # ---- transformer -----------------------------------------------------------------------------
    for l in range(hp["n_layers"]):
        _attention(out, sd, f"transformer_blocks.layers.{l}.0", f"l{l}.attn", D)
        _feedforward(out, sd, f"transformer_blocks.layers.{l}.1", f"l{l}.ff", D)
    g = _f64(sd["transformer_blocks.norm.gamma"]) * math.sqrt(D)
    out["head.w"] = _f64(sd["task_heads.beat_downbeat_lin.weight"]) * g[None, :]
    out["head.b"] = _f64(sd["task_heads.beat_downbeat_lin.bias"])
    return {
        k: np.ascontiguousarray((v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v)).astype(dtype).reshape(-1))
        for k, v in out.items()
    }


def blob_from_packed(packed: dict):
    """Flatten packed parameters into one float32 blob + index (for the init-time NCCL
    broadcast of the weights, see beat_this_b200/distributed.py)."""
    names = sorted(packed)
    sizes = [int(packed[n].size) for n in names]
    blob = np.concatenate([packed[n] for n in names]).astype(np.float32)
    return blob, names, sizes


def packed_from_blob(blob: np.ndarray, names, sizes) -> dict:
    out, o = {}, 0
    for n, s in zip(names, sizes):
        out[n] = np.ascontiguousarray(blob[o : o + s])
        o += s
    return out
