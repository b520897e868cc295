"""The reference's ``BeatThis`` as a trainable module on the GPU: parameters named and shaped as its ``state_dict``,
forward and backward through ``bt_train_forward`` / ``bt_train_backward`` (fp32 CUDA cores).

The gradient is that of the eval-mode function the inference path computes: BatchNorm on its running statistics and
no dropout.  ``.train(True)`` raises rather than train with other semantics than asked for.  There is no CPU path.
"""
from __future__ import annotations

import torch

from . import _lib
from .engine import Engine
from .inference import load_checkpoint
from .weights import filter_hparams, strip_prefixes


class _BeatThisFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, spect, *params):
        B, L, _ = spect.shape
        eng = module.engine
        act = torch.empty(eng.train_activation_bytes(B, L), dtype=torch.uint8, device=spect.device)
        beat = torch.empty(B, L, device=spect.device)
        down = torch.empty(B, L, device=spect.device)
        eng.train_forward(params, spect, act, beat, down)
        ctx.module, ctx.act, ctx.shape = module, act, (B, L)
        ctx.save_for_backward(*params)
        return beat, down

    @staticmethod
    def backward(ctx, dbeat, ddown):
        params = ctx.saved_tensors
        B, L = ctx.shape
        dev = ctx.act.device
        dbeat = torch.zeros(B, L, device=dev) if dbeat is None else dbeat.to(torch.float32).contiguous()
        ddown = torch.zeros(B, L, device=dev) if ddown is None else ddown.to(torch.float32).contiguous()
        grads = [torch.empty_like(p) if trainable and ctx.needs_input_grad[2 + i] else None
                 for i, (p, trainable) in enumerate(zip(params, ctx.module._trainable))]
        dspect = torch.empty(B, L, 128, device=dev) if ctx.needs_input_grad[1] else None
        ctx.module.engine.train_backward(params, ctx.act, B, L, dbeat, ddown, grads, dspect)
        return (None, dspect, *grads)


class BeatThisModule(torch.nn.Module):
    """Parameters and buffers named and shaped as the reference's ``BeatThis`` (``state_dict()`` keys match), on one
    CUDA device.  ``forward(spect [B, L, 128])`` returns ``{"beat", "downbeat"}`` logits [B, L] with gradients to every
    trainable parameter and to ``spect``.  Always in eval mode."""

    def __init__(self, hparams: dict, device="cuda"):
        super().__init__()
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
        if mode:
            raise NotImplementedError("BeatThisModule runs the eval-mode function only: dropout and batch-statistics "
                                      "BatchNorm are not implemented")
        return super().train(False)

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
        beat, down = _BeatThisFunction.apply(self, spect, *self._tables())
        return {"beat": beat, "downbeat": down}

    @classmethod
    def from_checkpoint(cls, checkpoint_path, device="cuda") -> "BeatThisModule":
        """A module with the weights of a reference ``.ckpt`` (a file, a short name or an already loaded dict)."""
        ckpt = checkpoint_path if isinstance(checkpoint_path, dict) else load_checkpoint(checkpoint_path, "cpu")
        state_dict = strip_prefixes(ckpt["state_dict"])
        module = cls(ckpt["hyper_parameters"], device)
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
