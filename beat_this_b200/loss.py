"""The beat tracker's training losses (reference beat_this/model/loss.py) on the GPU: ``bt_beat_loss`` for the value,
``bt_beat_loss_backward`` for the gradient to the predictions.

* ``MaskedBCELoss``, ``ShiftTolerantBCELoss``, ``SplittedShiftTolerantBCELoss``: the reference's modules, with its
  constructor signatures, ``pos_weight`` buffer and quirks, for ``[B, T]`` or ``[B, C, T]`` logits on a CUDA device.
* ``beat_loss_rows``: the same losses over ragged rows (one launch for any number of pieces), per row and overall.
* ``loss_from_hparams``: the (beat, downbeat) pair ``PLBeatThis.__init__`` builds from a checkpoint's hyper-parameters.

There is no CPU path: CPU tensors raise.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .engine import Engine

MASKED_BCE, SHIFT_TOLERANT, SPLIT_SHIFT_TOLERANT = 0, 1, 2  # BT_LOSS_* (include/beatthis.h)


def _flat(t, device):
    return t.to(device, torch.float32).contiguous().view(-1)


def _check_device(preds):
    if not preds.is_cuda:
        raise RuntimeError("beat_this_b200 losses run on a CUDA device; there is no CPU fallback")


def beat_loss_rows(preds, targets, mask, offsets, kind, tolerance=3, pos_weight=1.0):
    """Loss of concatenated rows (preds, targets, mask: 1-D device tensors, mask may be None; offsets: row i is
    [offsets[i], offsets[i+1])) -> (float64 tensor of per-row losses, 0-d fp32 tensor of all rows' terms over all rows'
    scored frames).  No gradient; two launches."""
    _check_device(preds)
    dev = preds.device
    x, y = _flat(preds, dev), _flat(targets, dev)
    m = None if mask is None else _flat(mask, dev)
    n = len(offsets) - 1
    row_loss = torch.empty(max(n, 1), dtype=torch.float64, device=dev)
    mean = torch.empty((), dtype=torch.float32, device=dev)
    params = _lib.bt_loss_params(int(kind), int(tolerance), float(pos_weight))
    Engine.shared(dev).beat_loss(x, y, m, offsets, params, row_loss, mean)
    return row_loss[:n], mean


class _BeatLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, preds, targets, mask, offsets, kind, tolerance, pos_weight):
        _, mean = beat_loss_rows(preds, targets, mask, offsets, kind, tolerance, pos_weight)
        ctx.save_for_backward(preds, targets, mask)
        ctx.args = (offsets, _lib.bt_loss_params(int(kind), int(tolerance), float(pos_weight)))
        return mean

    @staticmethod
    def backward(ctx, grad_mean):
        preds, targets, mask = ctx.saved_tensors
        offsets, params = ctx.args
        grad = torch.empty_like(preds)
        g = grad_mean.to(preds.device, torch.float32).contiguous()
        Engine.shared(preds.device).beat_loss_backward(preds, targets, mask, offsets, params, g, grad)
        return grad, None, None, None, None, None, None


def _apply(preds, targets, mask, kind, tolerance, pos_weight):
    """[..., T] logits, targets of the same shape and a mask broadcastable to it -> 0-d fp32 loss (the mean over every
    row of T frames), differentiable in preds."""
    _check_device(preds)
    if targets.shape != preds.shape:
        raise ValueError(f"targets {tuple(targets.shape)} and preds {tuple(preds.shape)} differ in shape")
    T = preds.shape[-1]
    rows = preds.numel() // T if T else 0
    dev = preds.device
    x = preds.float().contiguous().view(-1)
    y = _flat(targets.detach(), dev)
    m = None if mask is None else _flat(torch.broadcast_to(mask.detach().to(dev, torch.float32), preds.shape), dev)
    offsets = (np.arange(rows + 1, dtype=np.int64) * T).tolist()
    return _BeatLoss.apply(x, y, m, offsets, kind, tolerance, pos_weight)


def _pos_weight(pos_weight):
    return torch.tensor(pos_weight, dtype=torch.get_default_dtype())


class MaskedBCELoss(torch.nn.Module):
    """Plain binary cross-entropy on logits with an optional mask of weights (reference loss.py:9-35)."""

    def __init__(self, pos_weight: float = 1):
        super().__init__()
        self.register_buffer("pos_weight", _pos_weight(pos_weight), persistent=False)

    def forward(self, preds: torch.Tensor, targets: torch.Tensor, mask: torch.Tensor | None = None):
        return _apply(preds, targets, mask, MASKED_BCE, 0, float(self.pos_weight))


class ShiftTolerantBCELoss(torch.nn.Module):
    """BCE that tolerates shifts of up to `tolerance` frames between predictions and targets: predictions max-pooled
    over 2 tolerance + 1 frames, frames near a positive target ignored, the 2 tolerance frames at each end unscored
    (reference loss.py:38-92)."""

    def __init__(self, pos_weight: float = 1, tolerance: int = 3):
        super().__init__()
        self.register_buffer("pos_weight", _pos_weight(pos_weight), persistent=False)
        self.tolerance = tolerance

    def forward(self, preds: torch.Tensor, targets: torch.Tensor, mask: torch.Tensor | None = None):
        return _apply(preds, targets, mask, SHIFT_TOLERANT, self.tolerance, float(self.pos_weight))


class SplittedShiftTolerantBCELoss(torch.nn.Module):
    """ShiftTolerantBCELoss split into a positive and a negative part (reference loss.py:95-160): the paper's equation
    (Section 3.3), equal to ShiftTolerantBCELoss for binary targets.  As in the reference, ``tolerance`` is always 3
    and the predictions are spread by the constructor argument, the targets by twice it."""

    def __init__(self, pos_weight: float = 1, tolerance: int = 3):
        super().__init__()
        self.tolerance = 3
        self.spread_preds = tolerance
        self.spread_targets = 2 * tolerance
        self.register_buffer("pos_weight", _pos_weight(pos_weight), persistent=False)

    def forward(self, preds: torch.Tensor, targets: torch.Tensor, mask: torch.Tensor | None = None):
        if mask is None:
            raise ValueError("SplittedShiftTolerantBCELoss needs a mask")
        return _apply(preds, targets, mask, SPLIT_SHIFT_TOLERANT, self.spread_preds, float(self.pos_weight))


LOSS_TYPES = ("shift_tolerant_weighted_bce", "weighted_bce", "bce", "splitted_shift_tolerant_weighted_bce")


def loss_from_hparams(hp: dict):
    """(beat_loss, downbeat_loss) as PLBeatThis.__init__ builds them (reference pl_module.py:62-91) from a checkpoint's
    hyper_parameters; missing keys take PLBeatThis's defaults.  ValueError for an unknown loss_type."""
    loss_type = hp.get("loss_type", "shift_tolerant_weighted_bce")
    pw = hp.get("pos_weights", {"beat": 1, "downbeat": 1})
    if loss_type == "shift_tolerant_weighted_bce":
        return ShiftTolerantBCELoss(pos_weight=pw["beat"]), ShiftTolerantBCELoss(pos_weight=pw["downbeat"])
    if loss_type == "weighted_bce":
        return MaskedBCELoss(pos_weight=pw["beat"]), MaskedBCELoss(pos_weight=pw["downbeat"])
    if loss_type == "bce":
        return MaskedBCELoss(), MaskedBCELoss()
    if loss_type == "splitted_shift_tolerant_weighted_bce":
        return (SplittedShiftTolerantBCELoss(pos_weight=pw["beat"]),
                SplittedShiftTolerantBCELoss(pos_weight=pw["downbeat"]))
    raise ValueError(f"loss_type must be one of {', '.join(map(repr, LOSS_TYPES))}, got {loss_type!r}")


def loss_spec(module) -> tuple:
    """(kind, tolerance, pos_weight) of one of the three modules, the arguments of beat_loss_rows."""
    if isinstance(module, SplittedShiftTolerantBCELoss):
        return SPLIT_SHIFT_TOLERANT, module.spread_preds, float(module.pos_weight)
    if isinstance(module, ShiftTolerantBCELoss):
        return SHIFT_TOLERANT, module.tolerance, float(module.pos_weight)
    if isinstance(module, MaskedBCELoss):
        return MASKED_BCE, 0, float(module.pos_weight)
    raise TypeError(f"not a beat_this_b200 loss: {type(module).__name__}")
