"""The reference's optimizer setup (PLBeatThis.configure_optimizers, pl_module.py:279-306) on the GPU.

* ``AdamW``: ``torch.optim.AdamW``'s update (amsgrad and maximize off) as one ``bt_adamw_step`` launch for every
  parameter of every group, with torch's per-parameter state, so ``state_dict()`` / ``load_state_dict()`` exchange
  state with ``torch.optim.AdamW`` and with the ``optimizer_states`` of a Lightning checkpoint in both directions.
* ``CosineWarmupScheduler``: the reference's schedule (pl_module.py:342-369): a linear warm-up over ``warmup`` steps
  times a cosine decay over ``max_iters``, then a rise towards half the base rate.
* ``param_groups``: the reference's two groups: trainable tensors of two or more dimensions decay, the rest do not.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .engine import Engine


def param_groups(module: torch.nn.Module, weight_decay: float) -> list:
    """The reference's parameter groups, in ``module.parameters()`` order: trainable tensors with ndim >= 2 take
    `weight_decay`, the other trainable ones 0."""
    params = [p for p in module.parameters() if p.requires_grad]
    return [{"params": [p for p in params if p.ndim >= 2], "weight_decay": weight_decay},
            {"params": [p for p in params if p.ndim <= 1], "weight_decay": 0}]


class AdamW(torch.optim.Optimizer):
    """``torch.optim.AdamW(params, lr, betas, eps, weight_decay)`` with ``amsgrad=False`` and ``maximize=False``, its
    step one ``bt_adamw_step`` launch (include/beatthis.h: torch's foreach arithmetic, op by op in fp32) on the current
    stream of the parameters' device.  Parameters must be contiguous fp32 CUDA tensors on one device, gradients dense;
    anything else is refused before a launch.  A parameter without a gradient is skipped, as torch skips it."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2):
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f"Invalid beta parameters: {betas}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        # torch.optim.AdamW's group keys, so that state dicts pass between the two unchanged
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                        foreach=None, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=True)
        super().__init__(params, defaults)

    @staticmethod
    def _check(what, t, device):
        if t.is_sparse:
            raise RuntimeError(f"AdamW does not support sparse gradients ({what})")
        if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError(f"AdamW updates contiguous float32 CUDA tensors; {what} is {t.dtype} on {t.device}"
                               f"{'' if t.is_contiguous() else ', not contiguous'}; there is no CPU fallback")
        if device is not None and t.device != device:
            raise RuntimeError(f"AdamW updates the tensors of one device; {what} is on {t.device}, not {device}")

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        work, device = [], None
        for gi, group in enumerate(self.param_groups):
            if group.get("amsgrad") or group.get("maximize"):
                raise ValueError(f"param group {gi}: amsgrad and maximize are not supported")
            for p in group["params"]:
                if p.grad is None:
                    continue
                self._check(f"group {gi} parameter {tuple(p.shape)}", p, device)
                device = p.device
                self._check("its gradient", p.grad, device)
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                for k in ("exp_avg", "exp_avg_sq"):
                    self._check(f"its {k}", state[k], device)
                    if state[k].shape != p.shape:
                        raise RuntimeError(f"{k} of shape {tuple(state[k].shape)} for a parameter {tuple(p.shape)}")
                work.append((group, p, state))
        entries = []
        for group, p, state in work:
            state["step"] += 1  # torch's float32 CPU step, incremented before the update
            beta1, beta2 = group["betas"]
            entries.append(_lib.bt_adamw_entry(
                p.data_ptr(), p.grad.data_ptr(), state["exp_avg"].data_ptr(), state["exp_avg_sq"].data_ptr(),
                p.numel(), float(group["lr"]), float(beta1), float(beta2), float(group["eps"]),
                float(group["weight_decay"]), int(state["step"].item())))
        if entries:
            Engine.shared(device).adamw_step(entries)
        return loss


class CosineWarmupScheduler(torch.optim.lr_scheduler.LRScheduler):
    """The reference's learning-rate schedule, stepped once per optimizer step: at step s the factor of every base
    rate is, in numpy float64 as the reference computes it,

    * s < max_iters: 0.5 (1 + cos(pi s / max_iters)), times s / warmup while s <= warmup (0 at step 0, so the first
      optimizer step runs at rate 0);
    * s >= max_iters: raise_to min((s - max_iters) / warmup, 1), raise_to = 0.5.

    ``warmup`` below 1 is a ValueError (the reference divides by it)."""

    def __init__(self, optimizer, warmup, max_iters):
        if warmup < 1:
            raise ValueError(f"warmup must be at least 1 step, got {warmup}")
        self.warmup = warmup
        self.max_num_iters = int(max_iters)
        self.raise_to = 0.5  # the factor after max_iters; a state attribute, as in the reference's state_dict
        super().__init__(optimizer)

    def get_lr(self):
        # Python floats of the reference's float64 products, so that a state_dict holds no numpy scalars
        factor = self.get_lr_factor(self.last_epoch)
        return [float(base_lr * factor) for base_lr in self.base_lrs]

    def get_lr_factor(self, step):
        if step >= self.max_num_iters:
            return self.raise_to * min((step - self.max_num_iters) / self.warmup, 1)
        factor = 0.5 * (1 + np.cos(np.pi * (step / self.max_num_iters)))
        if step <= self.warmup:
            factor *= step / self.warmup
        return factor
