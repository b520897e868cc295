"""The reference's ``BeatThis`` as a trainable module on the GPU: parameters named and shaped as its ``state_dict``,
forward and backward through ``bt_train_forward_ex`` / ``bt_train_backward_ex`` (fp32 CUDA cores).

By default the gradient is that of the eval-mode function the inference path computes: BatchNorm on its running
statistics and no dropout, and ``.train(True)`` raises rather than train with other semantics than asked for.  A module
made with ``train_mode=True`` also runs the reference's training-mode function after ``.train()``: dropout at the
rates of ``hparams["dropout"]`` and batch-statistics BatchNorm that updates the running statistics.  There is no CPU
path.
"""
from __future__ import annotations

import math

import torch

from . import _lib
from .engine import Engine
from .inference import load_checkpoint
from .weights import filter_hparams, strip_prefixes


class _BeatThisFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, mode, spect, *params):
        # mode: None (eval mode) or (seed, dropout_frontend, dropout_transformer); the running statistics in params
        # are updated in place by a training-mode pass and never read by its backward
        B, L, _ = spect.shape
        eng = module.engine
        act = torch.empty(eng.train_activation_bytes(B, L, mode), dtype=torch.uint8, device=spect.device)
        beat = torch.empty(B, L, device=spect.device)
        down = torch.empty(B, L, device=spect.device)
        eng.train_forward(params, spect, act, beat, down, mode=mode)
        ctx.module, ctx.act, ctx.shape, ctx.mode = module, act, (B, L), mode
        # autograd tracks the trainable entries; the buffers (running statistics, num_batches_tracked) and freqs are
        # held as they are, so a second training-mode forward before this backward may update them in place, as with
        # torch's BatchNorm (a training-mode backward never reads the running statistics)
        ctx.save_for_backward(*[p for p, t in zip(params, module._trainable) if t])
        ctx.fixed = [None if t else p for p, t in zip(params, module._trainable)]
        return beat, down

    @staticmethod
    def backward(ctx, dbeat, ddown):
        saved = iter(ctx.saved_tensors)
        params = [next(saved) if p is None else p for p in ctx.fixed]
        B, L = ctx.shape
        dev = ctx.act.device
        dbeat = torch.zeros(B, L, device=dev) if dbeat is None else dbeat.to(torch.float32).contiguous()
        ddown = torch.zeros(B, L, device=dev) if ddown is None else ddown.to(torch.float32).contiguous()
        grads = [torch.empty_like(p) if trainable and ctx.needs_input_grad[3 + i] else None
                 for i, (p, trainable) in enumerate(zip(params, ctx.module._trainable))]
        dspect = torch.empty(B, L, 128, device=dev) if ctx.needs_input_grad[2] else None
        ctx.module.engine.train_backward(params, ctx.act, B, L, dbeat, ddown, grads, dspect, mode=ctx.mode)
        return (None, None, dspect, *grads)


class BeatThisModule(torch.nn.Module):
    """Parameters and buffers named and shaped as the reference's ``BeatThis`` (``state_dict()`` keys match), on one
    CUDA device.  ``forward(spect [B, L, 128])`` returns ``{"beat", "downbeat"}`` logits [B, L] with gradients to every
    trainable parameter and to ``spect``.

    A default module is always in eval mode.  With ``train_mode=True``, ``.train()`` selects the reference's
    training-mode function: each forward draws a 64-bit dropout seed from torch's default generator (so
    ``torch.manual_seed`` makes runs repeatable), uses batch statistics in every BatchNorm and updates its running
    statistics and ``num_batches_tracked``, also under ``torch.no_grad()``."""

    def __init__(self, hparams: dict, device="cuda", *, train_mode: bool = False):
        super().__init__()
        self.train_mode = bool(train_mode)
        self.hparams = filter_hparams(hparams)
        self.checkpoint_hparams = dict(hparams)
        self.engine = Engine(None, self.hparams, device)  # a weight-less fp32 context of the model's shape
        dev = self.engine.device
        self._names, self._trainable = [], []
        for name, shape, trainable in _lib.train_param_table(self.hparams):
            *path, leaf = name.split(".")
            parent = self
            for part in path:
                if not hasattr(parent, part):
                    parent.add_module(part, torch.nn.Module())
                parent = getattr(parent, part)
            if leaf == "num_batches_tracked":
                parent.register_buffer(leaf, torch.zeros((), dtype=torch.int64, device=dev))
            elif trainable or leaf == "freqs":  # rotary_embed.freqs: a parameter without gradient in the reference
                parent.register_parameter(leaf, torch.nn.Parameter(torch.zeros(shape, device=dev),
                                                                   requires_grad=trainable))
            else:
                parent.register_buffer(leaf, torch.zeros(shape, device=dev))
            self._names.append(name)
            self._trainable.append(trainable)
        super().train(False)

    def train(self, mode: bool = True):
        if mode and not self.train_mode:
            raise NotImplementedError("this BeatThisModule runs the eval-mode function only; make it with "
                                      "train_mode=True for dropout and batch-statistics BatchNorm")
        return super().train(mode)

    @torch.no_grad()
    def reset_parameters(self, generator: torch.Generator | None = None) -> "BeatThisModule":
        """The reference's initialisation (BeatThis._init_weights and the modules' own defaults), for training from
        scratch: linear weights N(0, 0.02) and biases 0, conv2d weights kaiming_normal_(fan_out, relu), BatchNorm
        weight 1, bias 0, running mean 0, running variance 1 and no batches tracked, RMSNorm gamma 1, and the rotary
        frequencies 1 / 10000^(2i / 32).  Random entries are drawn on the host from `generator` (None: torch's
        default generator), in table order."""
        for name, t in zip(self._names, self._tables()):
            leaf = name.rsplit(".", 1)[1]
            bn = name.rsplit(".", 1)[0] + ".running_mean" in self._names
            if leaf == "freqs":
                val = 1.0 / (10000 ** (torch.arange(0, 32, 2, dtype=torch.float32) / 32))
            elif bn and leaf in ("weight", "running_var") or leaf == "gamma":
                val = torch.ones(t.shape)
            elif leaf == "weight" and t.ndim == 4:
                fan_out = t.shape[0] * t.shape[2] * t.shape[3]
                val = torch.randn(t.shape, generator=generator) * (math.sqrt(2.0) / math.sqrt(fan_out))
            elif leaf == "weight":
                val = torch.randn(t.shape, generator=generator) * 0.02
            else:  # biases, running means, num_batches_tracked
                val = torch.zeros(t.shape, dtype=t.dtype)
            t.copy_(val.to(t.dtype))
        return self

    def _tables(self):
        named = dict(self.named_parameters())
        named.update(self.named_buffers())
        return [named[n] for n in self._names]

    def forward(self, spect: torch.Tensor) -> dict:
        if not spect.is_cuda:
            raise RuntimeError("BeatThisModule runs on a CUDA device; there is no CPU fallback")
        if spect.ndim != 3 or spect.shape[2] != 128:
            raise ValueError(f"expected spectrograms [B, L, 128], got {tuple(spect.shape)}")
        spect = spect.to(self.engine.device, torch.float32).contiguous()
        mode = None
        if self.training:
            seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64).item()) & (2 ** 64 - 1)
            rates = self.hparams["dropout"]
            mode = (seed, float(rates["frontend"]), float(rates["transformer"]))
            # before the function saves its inputs: an in-place bump after would fail autograd's version check
            with torch.no_grad():
                for name, t in zip(self._names, self._tables()):
                    if name.endswith(".num_batches_tracked"):
                        t.add_(1)
        beat, down = _BeatThisFunction.apply(self, mode, spect, *self._tables())
        return {"beat": beat, "downbeat": down}

    @classmethod
    def from_checkpoint(cls, checkpoint_path, device="cuda", *, train_mode: bool = False) -> "BeatThisModule":
        """A module with the weights of a reference ``.ckpt`` (a file, a short name or an already loaded dict)."""
        ckpt = checkpoint_path if isinstance(checkpoint_path, dict) else load_checkpoint(checkpoint_path, "cpu")
        state_dict = strip_prefixes(ckpt["state_dict"])
        module = cls(ckpt["hyper_parameters"], device, train_mode=train_mode)
        module.load_state_dict(state_dict)
        return module

    def save_checkpoint(self, path: str, hparams: dict | None = None) -> str:
        """Write the weights in the reference ``.ckpt`` layout (``model.``-prefixed ``state_dict`` and
        ``hyper_parameters``: `hparams`, by default those the module was made with)."""
        torch.save({
            "state_dict": {"model." + k: v.detach().cpu() for k, v in self.state_dict().items()},
            "hyper_parameters": dict(hparams if hparams is not None else self.checkpoint_hparams),
        }, path)
        return path
