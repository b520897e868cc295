"""The reference's ``BeatThis`` as a trainable module on the GPU: parameters named and shaped as its ``state_dict``,
forward and backward through ``bt_train_forward_ex`` / ``bt_train_backward_ex`` (fp32 CUDA cores); and ``fit`` /
``python -m beat_this_b200.train``, the reference's training run (launch_scripts/train.py with PLBeatThis) without
Lightning, on one GPU or data-parallel on several (``torchrun --nproc-per-node N -m beat_this_b200.train``).

By default the gradient is that of the eval-mode function the inference path computes: BatchNorm on its running
statistics and no dropout, and ``.train(True)`` raises rather than train with other semantics than asked for.  A module
made with ``train_mode=True`` also runs the reference's training-mode function after ``.train()``: dropout at the
rates of ``hparams["dropout"]`` and batch-statistics BatchNorm that updates the running statistics.  There is no CPU
path.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import math
import os
import random
import sys
from datetime import timedelta

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .engine import Engine
from .inference import load_checkpoint
from .weights import filter_hparams, strip_prefixes


class _BeatThisFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, mode, capture, spect, *params):
        # mode: None (eval mode) or (seed, dropout_frontend, dropout_transformer); the running statistics in params
        # are updated in place by a training-mode pass and never read by its backward.  capture: None, or (running,
        # batch_stats): the pass updates the running table `running` instead and its batch statistics are copied into
        # batch_stats
        B, L, _ = spect.shape
        eng = module.engine
        act = torch.empty(eng.train_activation_bytes(B, L, mode), dtype=torch.uint8, device=spect.device)
        beat = torch.empty(B, L, device=spect.device)
        down = torch.empty(B, L, device=spect.device)
        eng.train_forward(params, spect, act, beat, down, mode=mode, running=None if capture is None else capture[0])
        if capture is not None:  # the store keeps them after the eval-mode layout
            stats = capture[1]
            stats.copy_(act.view(torch.float32)[act.numel() // 4 - stats.numel():])
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
        grads = [torch.empty_like(p) if trainable and ctx.needs_input_grad[4 + i] else None
                 for i, (p, trainable) in enumerate(zip(params, ctx.module._trainable))]
        dspect = torch.empty(B, L, 128, device=dev) if ctx.needs_input_grad[3] else None
        ctx.module.engine.train_backward(params, ctx.act, B, L, dbeat, ddown, grads, dspect, mode=ctx.mode)
        return (None, None, None, dspect, *grads)


class BeatThisModule(torch.nn.Module):
    """Parameters and buffers named and shaped as the reference's ``BeatThis`` (``state_dict()`` keys match), on one
    CUDA device.  ``forward(spect [B, L, 128])`` returns ``{"beat", "downbeat"}`` logits [B, L] with gradients to every
    trainable parameter and to ``spect``.

    A default module is always in eval mode.  With ``train_mode=True``, ``.train()`` selects the reference's
    training-mode function: each forward draws a 64-bit dropout seed from torch's default generator (so
    ``torch.manual_seed`` makes runs repeatable), uses batch statistics in every BatchNorm and updates its running
    statistics and ``num_batches_tracked``, also under ``torch.no_grad()``.  A training-mode forward given
    ``batch_stats`` leaves the running statistics and counters as they are and writes its batch statistics there
    instead; ``replay_batch_stats`` applies them later, bitwise as the forward passes would have."""

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

    def dropout_mode(self) -> tuple:
        """The mode of one training-mode forward pass, (seed, dropout_frontend, dropout_transformer): a 64-bit seed drawn
        from torch's default generator and the model's rates.  Each training-mode forward calls it once; a rank of a
        data-parallel run calls it for every micro-batch another rank runs, so that all ranks draw the same seeds."""
        seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64).item()) & (2 ** 64 - 1)
        rates = self.hparams["dropout"]
        return (seed, float(rates["frontend"]), float(rates["transformer"]))

    def batch_stat_floats(self, B: int, L: int) -> int:
        """The length of the ``batch_stats`` tensor a training-mode forward over [B, L, 128] fills."""
        return self.engine.train_batch_stat_floats(B, L)

    def _counters(self):
        return [t for name, t in zip(self._names, self._tables()) if name.endswith(".num_batches_tracked")]

    def _running(self, scratch: bool = False):
        """The running-statistics table parallel to the parameter table: this module's running statistics, or scratch
        tensors of their shapes (allocated once) that a forward with batch_stats updates instead."""
        if not scratch:
            return self._tables()
        if getattr(self, "_scratch_running", None) is None:
            self._scratch_running = [torch.empty_like(t) if name.endswith((".running_mean", ".running_var")) else None
                                     for name, t in zip(self._names, self._tables())]
        return self._scratch_running

    def forward(self, spect: torch.Tensor, batch_stats: torch.Tensor | None = None) -> dict:
        """batch_stats (training mode only): a contiguous fp32 tensor of batch_stat_floats(B, L) elements on the
        module's device that receives the pass's BatchNorm batch statistics; the running statistics and
        ``num_batches_tracked`` are then left as they are."""
        if not spect.is_cuda:
            raise RuntimeError("BeatThisModule runs on a CUDA device; there is no CPU fallback")
        if spect.ndim != 3 or spect.shape[2] != 128:
            raise ValueError(f"expected spectrograms [B, L, 128], got {tuple(spect.shape)}")
        spect = spect.to(self.engine.device, torch.float32).contiguous()
        mode, capture = None, None
        if self.training:
            mode = self.dropout_mode()
            if batch_stats is not None:
                need = self.batch_stat_floats(*spect.shape[:2])
                if (batch_stats.device != self.engine.device or batch_stats.dtype != torch.float32
                        or not batch_stats.is_contiguous() or batch_stats.numel() != need):
                    raise ValueError(f"batch_stats: need a contiguous float32 tensor of {need} elements on "
                                     f"{self.engine.device}")
                capture = (self._running(scratch=True), batch_stats)
            else:
                # before the function saves its inputs: an in-place bump after would fail autograd's version check
                with torch.no_grad():
                    for t in self._counters():
                        t.add_(1)
        elif batch_stats is not None:
            raise ValueError("batch_stats is for training-mode forward passes")
        beat, down = _BeatThisFunction.apply(self, mode, capture, spect, *self._tables())
        return {"beat": beat, "downbeat": down}

    @torch.no_grad()
    def replay_batch_stats(self, stats, B: int, L: int) -> None:
        """Applies the batch statistics of training-mode forward passes over [B, L, 128] (``batch_stats`` tensors, in
        the order of the passes) to the running statistics and adds their number to ``num_batches_tracked``: bitwise
        what the passes would have done without ``batch_stats``."""
        self.engine.train_running_replay(self._running(), list(stats), B, L)
        for t in self._counters():
            t.add_(len(stats))

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


# ---- the training run (reference launch_scripts/train.py, PLBeatThis) ---------------------------------------------
# The loop follows Lightning's rules as the reference's Trainer applies them, in fp32 without a GradScaler (the
# reference trains at precision="16-mixed"), so no step is ever skipped:
# * every micro-batch runs backward() on (beat_loss + downbeat_loss) / accumulate_grad_batches;
# * the optimizer steps after every accumulate-th micro-batch and after the last one of an epoch, then the scheduler
#   steps and the gradients are set to None; global_step counts optimizer steps;
# * estimated_stepping_batches = ceil(batches per epoch / accumulate) * max_epochs sets the schedule's length.
# Lightning's one-batch sanity validation before training is left out: it changes no training state.

def step_plan(n_batches: int, accumulate: int) -> list:
    """Indices of the micro-batches of an epoch of `n_batches` after which the optimizer steps."""
    return [i for i in range(n_batches) if (i + 1) % accumulate == 0 or i + 1 == n_batches]


def micro_batch_owners(n_batches: int, accumulate: int, world: int) -> list:
    """Who runs what in a data-parallel epoch of `n_batches` micro-batches on `world` ranks: per optimizer-step group of
    step_plan (the consecutive micro-batches up to each step point; the last group may be short), the (rank, slot) of
    each of its micro-batches.  Micro-batch j of a group (0-based) belongs to rank j mod world, in slot j div world, so
    a short group leaves the last ranks idle.  world > accumulate raises ValueError: a rank would never train."""
    if world < 1:
        raise ValueError(f"need at least one rank, got {world}")
    if world > accumulate:
        raise ValueError(f"{world} ranks for {accumulate} micro-batches per optimizer step (accumulate_grad_batches): "
                         f"ranks {accumulate} and up would never train")
    groups, start = [], 0
    for end in step_plan(n_batches, accumulate):
        groups.append([(j % world, j // world) for j in range(end + 1 - start)])
        start = end + 1
    return groups


def estimated_stepping_batches(n_batches: int, accumulate: int, max_epochs: int) -> int:
    return math.ceil(n_batches / accumulate) * max_epochs


def augmentations(tempo: bool, pitch: bool, mask: bool) -> dict:
    """The reference's augmentation settings for --tempo/pitch/mask-augmentation."""
    aug = {}
    if tempo:
        aug["tempo"] = {"min": -20, "max": 20, "stride": 4}
    if pitch:
        aug["pitch"] = {"min": -5, "max": 6}
    if mask:
        aug["mask"] = {"kind": "permute", "min_count": 1, "max_count": 6, "min_len": 0.1, "max_len": 2,
                       "min_parts": 5, "max_parts": 9}
    return aug


def params_str(val=True, hung_data=False, fold=None, loss="shift_tolerant_weighted_bce", transformer_dim=512,
               tempo_augmentation=True, pitch_augmentation=True, mask_augmentation=True, sum_head=True,
               partial_transformers=True, **_) -> str:
    """The run description the reference puts into its checkpoint's file name."""
    head = ("" if val else "noval ") + ("hung " if hung_data else "") + ("" if fold is None else f"fold{fold} ")
    tail = ("" if sum_head else " nosumH ") + ("" if partial_transformers else " nopartialT ")
    return (f"{head}{loss}-h{transformer_dim}-aug{tempo_augmentation}{pitch_augmentation}{mask_augmentation}"
            f"{tail}")


def checkpoint_path(checkpoint_dir, name="", seed=0, **run) -> str:
    """<checkpoint_dir>/<name> S<seed> <params_str>.ckpt, the reference's ModelCheckpoint file name."""
    return os.path.join(str(checkpoint_dir), f"{name} S{seed} {params_str(**run)}".strip() + ".ckpt")


def _rng_state(batches) -> dict:
    """The random states the next epoch draws from, in types torch.load(weights_only=True) reads."""
    version, mt, gauss = random.getstate()
    kind, keys, pos, has_gauss, cached = np.random.get_state()
    return {"python": [version, list(mt), gauss], "numpy": [kind, torch.from_numpy(keys.astype(np.int64)), int(pos),
                                                            int(has_gauss), float(cached)],
            "torch": torch.get_rng_state(), "batches": batches.generator.get_state()}


def _set_rng_state(state: dict, batches) -> None:
    version, mt, gauss = state["python"]
    random.setstate((version, tuple(mt), gauss))
    kind, keys, pos, has_gauss, cached = state["numpy"]
    np.random.set_state((kind, keys.numpy().astype(np.uint32), pos, has_gauss, cached))
    torch.set_rng_state(state["torch"])
    batches.generator.set_state(state["batches"])


def _losses(loss_pair, out, batch):
    """PLBeatThis._compute_loss: the beat loss under the padding mask, the downbeat loss under the padding mask times
    each item's downbeat mask."""
    beat_loss, downbeat_loss = loss_pair
    mask = batch["padding_mask"]
    down_mask = mask.float() * batch["downbeat_mask"].to(mask.device).float()[:, None]
    lb = beat_loss(out["beat"], batch["truth_beat"].float(), mask)
    ld = downbeat_loss(out["downbeat"], batch["truth_downbeat"].float(), down_mask)
    return lb, ld


def _validate(module, batches, loss_pair, post, eval_trim_beats, world: int = 1) -> dict:
    """validation_step over every batch: the loss pair (means over batches weighted by batch size), then the
    post-processed beats under the padding mask scored against truth_orig_* (F-measure and Cemgil, means over
    pieces).  With world > 1, `batches` yields None for the batches other ranks run, and the ranks' results are
    gathered and combined in batch order."""
    from .evaluate import beat_metrics

    module.eval()
    device = module.engine.device
    local = []  # per batch run here: (batch index, fp32 loss pair, size, beats, downbeats, truth beats, truth downbeats)
    with torch.no_grad():
        for b, batch in enumerate(batches):
            if batch is None:
                continue
            out = module(batch["spect"])
            lb, ld = _losses(loss_pair, out, batch)
            beats, downs = post(out["beat"], out["downbeat"], batch["padding_mask"])
            local.append((b, torch.stack([lb, ld]), len(batch["spect"]), list(beats), list(downs),
                          *[[np.frombuffer(t, dtype=np.float64) for t in batch[f"truth_orig_{k}"]]
                            for k in ("beat", "downbeat")]))
    module.train()
    if world > 1:
        parts = [None] * world
        dist.all_gather_object(parts, [(r[0], r[1].cpu(), *r[2:]) for r in local])
        local = sorted((r for part in parts for r in part), key=lambda r: r[0])
    sums, n = torch.zeros(2, dtype=torch.float64, device=device), 0
    est, ref = {"beat": [], "downbeat": []}, {"beat": [], "downbeat": []}
    for _, pair, B, beats, downs, ref_beats, ref_downs in local:
        sums += pair.to(device).double() * B
        n += B
        est["beat"] += beats
        est["downbeat"] += downs
        ref["beat"] += ref_beats
        ref["downbeat"] += ref_downs
    lb, ld = (sums / max(n, 1)).tolist()
    rec = {"val_loss_beat": lb, "val_loss_downbeat": ld, "val_loss": lb + ld}
    for target in ("beat", "downbeat"):
        rows = beat_metrics(est[target], ref[target], min_beat_time=eval_trim_beats, device=module.engine.device)
        rec[f"val_F-measure_{target}"] = float(np.mean(rows[:, 5])) if len(rows) else float("nan")
        rec[f"val_Cemgil_{target}"] = float(np.mean((rows[:, 6] + rows[:, 7]) / 2)) if len(rows) else float("nan")
    return rec


def fit(data="data", checkpoint_dir="checkpoints", *, name="", gpu=0, n_layers=6, transformer_dim=512,
        frontend_dropout=0.1, transformer_dropout=0.2, lr=0.0008, weight_decay=0.01, fps=50,
        loss="shift_tolerant_weighted_bce", warmup_steps=1000, max_epochs=100, batch_size=8,
        accumulate_grad_batches=8, train_length=1500, dbn=False, eval_trim_beats=5, val_frequency=5,
        tempo_augmentation=True, pitch_augmentation=True, mask_augmentation=True, sum_head=True,
        partial_transformers=True, length_based_oversampling_factor=0.65, val=True, hung_data=False, fold=None,
        seed=0, resume_checkpoint=None, test=True, epochs=None) -> list:
    """Train a BeatThis model from scratch (or resume) as the reference's train.py does, on CUDA device `gpu`; the
    keyword arguments are the reference's command-line flags.  Returns one record per epoch run (each also printed
    as a JSON line): epoch, global_step, lr (after the epoch), step_lr (the rate of each optimizer step, as
    LearningRateMonitor logs it), the train losses' means over micro-batches weighted by batch size and, after a
    validation, the val losses, F-measure and Cemgil.  The checkpoint <checkpoint_dir>/<name> S<seed>
    <params_str>.ckpt is written at the end of every epoch (through a temporary file, so an interrupted save leaves
    the last one).  After the last epoch, unless `test` is off, the checkpoint is scored on the test split by
    ``evaluate`` (the reference's trainer.test); its summary goes into the last record under "test".
    epochs: run at most this many epochs in this call (None: up to max_epochs); the schedule still spans max_epochs,
    and `resume_checkpoint` continues the run later.

    Data-parallel: when the default process group is initialised with more than one rank, every rank calls fit with
    the same flags (`gpu` aside: each rank's own device) and the micro-batches of each optimizer step are spread over
    the ranks (micro_batch_owners).  Every rank draws every random number a one-process run draws, in its order, the
    gradients are summed in micro-batch order and the BatchNorm running statistics replayed in it, so the run writes the
    checkpoint and returns the records of the one-process run with the same flags, bitwise; checkpoints pass between
    world sizes.  Rank 0 writes the checkpoint and runs the final test; every rank returns the records."""
    flags = {k: v for k, v in locals().items() if k != "gpu"}
    from . import dataset as D
    from .loss import loss_from_hparams
    from .optim import AdamW, CosineWarmupScheduler, param_groups
    from .postprocessor import Postprocessor

    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    device = torch.device("cuda", gpu)
    torch.cuda.set_device(device)
    if world > 1:
        # the digests first: every rank then refuses what follows alike, whatever flags it was given
        digest = hashlib.sha256(repr(sorted(flags.items())).encode()).hexdigest()
        digests = [None] * world
        dist.all_gather_object(digests, digest)
        if len(set(digests)) > 1:
            raise ValueError(f"the ranks of a data-parallel run were given different flags (digests {digests})")
        micro_batch_owners(0, accumulate_grad_batches, world)  # refuses more ranks than micro-batches per step
    random.seed(seed)  # seed_everything
    np.random.seed(seed)
    torch.manual_seed(seed)

    run = dict(val=val, hung_data=hung_data, fold=fold, loss=loss, transformer_dim=transformer_dim,
               tempo_augmentation=tempo_augmentation, pitch_augmentation=pitch_augmentation,
               mask_augmentation=mask_augmentation, sum_head=sum_head, partial_transformers=partial_transformers)
    aug = augmentations(tempo_augmentation, pitch_augmentation, mask_augmentation)
    dm_hparams = dict(data_dir=str(data), batch_size=batch_size, train_length=train_length, num_workers=0,
                      augmentations=aug, test_dataset="gtzan", hung_data=hung_data, no_val=not val, spect_fps=fps,
                      length_based_oversampling_factor=length_based_oversampling_factor, fold=fold,
                      predict_datasplit="test")
    train_items, val_items = D.train_val_items(data, "gtzan", fold, hung_data, not val)
    train_set = D.BeatTrackingDataset(train_items, data, fps, train_length, deterministic=False, augmentations=aug,
                                      length_based_oversampling_factor=length_based_oversampling_factor)
    val_set = D.BeatTrackingDataset(val_items, data, fps, train_length, deterministic=True, augmentations={})
    train_batches = D.TrainingBatches(train_set, batch_size, shuffle=True, drop_last=True, device=device)
    val_batches = D.TrainingBatches(val_set, batch_size, shuffle=False, drop_last=False, seed=0, device=device)
    if len(train_batches) == 0:
        raise ValueError(f"{len(train_set)} training items make no batch of {batch_size}")
    groups = micro_batch_owners(len(train_batches), accumulate_grad_batches, world)
    if world > 1:
        owners = [r for group in groups for r, _ in group]
        train_batches.shard = lambda k: owners[k] == rank
        val_batches.shard = lambda k: k % world == rank
    pos_weights = train_set.positive_weights(widen_target_mask=3)
    if rank == 0:
        print("Using positive weights: ", pos_weights)

    hparams = dict(spect_dim=128, fps=50, transformer_dim=transformer_dim, ff_mult=4, n_layers=n_layers, stem_dim=32,
                   dropout={"frontend": frontend_dropout, "transformer": transformer_dropout}, lr=lr,
                   weight_decay=weight_decay, pos_weights=pos_weights, head_dim=32, loss_type=loss,
                   warmup_steps=warmup_steps, max_epochs=max_epochs, use_dbn=dbn, eval_trim_beats=eval_trim_beats,
                   sum_head=sum_head, partial_transformers=partial_transformers)
    if loss == "fast_shift_tolerant_weighted_bce":
        raise ValueError("loss_type must be one of 'shift_tolerant_weighted_bce', 'weighted_bce', 'bce'")
    loss_pair = loss_from_hparams(hparams)
    module = BeatThisModule(hparams, device, train_mode=True).reset_parameters()
    opt = AdamW(param_groups(module, weight_decay), lr=lr)
    total_steps = estimated_stepping_batches(len(train_batches), accumulate_grad_batches, max_epochs)
    sched = CosineWarmupScheduler(opt, warmup_steps, total_steps)
    post = Postprocessor("dbn" if dbn else "minimal", 50, engine=module.engine)

    first_epoch, global_step = 0, 0
    if resume_checkpoint is not None:
        # a checkpoint the user names: a Lightning one holds numpy scalars, so it is unpickled in full
        ckpt = torch.load(resume_checkpoint, map_location="cpu", weights_only=False)
        module.load_state_dict(strip_prefixes(ckpt["state_dict"]))
        opt.load_state_dict(ckpt["optimizer_states"][0])
        sched.load_state_dict(ckpt["lr_schedulers"][0])
        first_epoch, global_step = int(ckpt["epoch"]) + 1, int(ckpt["global_step"])
        if "beat_this_b200" in ckpt:
            _set_rng_state(ckpt["beat_this_b200"], train_batches)
        else:
            print(f"{resume_checkpoint} holds no random states: the data order and dropout masks of the resumed "
                  f"epochs differ from those of an uninterrupted run")

    path = checkpoint_path(checkpoint_dir, name, seed, **run)
    os.makedirs(str(checkpoint_dir), exist_ok=True)
    last_epoch = max_epochs if epochs is None else min(max_epochs, first_epoch + epochs)
    plan = set(step_plan(len(train_batches), accumulate_grad_batches))
    exchange = _GradientExchange(module, opt, world, accumulate_grad_batches) if world > 1 else None
    records = []
    module.train()
    for epoch in range(first_epoch, last_epoch):
        sums, n, step_lr = torch.zeros(2, dtype=torch.float64, device=device), 0, []
        if exchange is None:
            for i, batch in enumerate(train_batches):
                out = module(batch["spect"])
                lb, ld = _losses(loss_pair, out, batch)
                ((lb + ld) / accumulate_grad_batches).backward()
                B = len(batch["spect"])
                sums += torch.stack([lb.detach(), ld.detach()]).double() * B
                n += B
                if i in plan:
                    step_lr.append(opt.param_groups[0]["lr"])
                    opt.step()
                    sched.step()
                    opt.zero_grad(set_to_none=True)
                    global_step += 1
        else:
            batches = iter(train_batches)
            for group in groups:
                for owner, slot in group:
                    batch = next(batches)
                    if owner != rank:
                        module.dropout_mode()  # the seed of a micro-batch another rank runs
                        continue
                    out = module(batch["spect"], batch_stats=exchange.stats(slot))
                    lb, ld = _losses(loss_pair, out, batch)
                    ((lb + ld) / accumulate_grad_batches).backward()
                    exchange.pack(slot, lb, ld, batch["spect"].shape)
                for lb_ld, B in exchange.reduce(len(group)):
                    sums += lb_ld.double() * B
                    n += B
                step_lr.append(opt.param_groups[0]["lr"])
                opt.step()
                sched.step()
                opt.zero_grad(set_to_none=True)
                global_step += 1
        lb, ld = (sums / n).tolist()
        rec = {"epoch": epoch, "global_step": global_step, "lr": opt.param_groups[0]["lr"], "step_lr": step_lr,
               "train_loss_beat": lb, "train_loss_downbeat": ld, "train_loss": lb + ld}
        if (epoch + 1) % val_frequency == 0:
            rec.update(_validate(module, val_batches, loss_pair, post, eval_trim_beats, world))
        if rank == 0:
            ckpt = {"epoch": epoch, "global_step": global_step,
                    "state_dict": {"model." + k: v.detach().cpu() for k, v in module.state_dict().items()},
                    "hyper_parameters": hparams, "datamodule_hyper_parameters": dm_hparams,
                    "optimizer_states": [opt.state_dict()], "lr_schedulers": [sched.state_dict()],
                    "beat_this_b200": _rng_state(train_batches)}
            torch.save(ckpt, path + ".tmp")
            os.replace(path + ".tmp", path)
            print(json.dumps(rec), flush=True)
        records.append(rec)
    if test and last_epoch == max_epochs and first_epoch < max_epochs:
        from .evaluate import evaluate

        summary = [None]
        # the others wait for rank 0's test on the host, over gloo with a deadline of days: the test split's length
        # (and the DBN) set how long the test takes, and the default group's watchdog could abort a device wait
        waiting = dist.new_group(backend="gloo", timeout=timedelta(days=7)) if world > 1 else None
        if rank == 0:
            summary[0] = evaluate(path, data=data, datasplit="test", min_beat_time=eval_trim_beats, device=device,
                                  dbn=dbn, losses=True).summary
            print(json.dumps({"test": summary[0]}), flush=True)
        if world > 1:  # the others wait here for rank 0's test
            dist.broadcast_object_list(summary, src=0, group=waiting)
            dist.destroy_process_group(waiting)
        records[-1]["test"] = summary[0]
    if world > 1:
        dist.barrier()  # the checkpoint is written when fit returns on any rank
    return records


class _GradientExchange:
    """The gradient exchange of a data-parallel optimizer step of up to `accumulate` micro-batches on `world` ranks.

    Each rank keeps a send buffer of S = ceil(accumulate / world) slots, one per micro-batch it runs in a step.  A
    slot is a row [P | Q | 4]: the P gradient elements of every trainable parameter in the optimizer's order
    (bt_grad_pack), the Q floats of the micro-batch's BatchNorm batch statistics (captured by its forward pass), and
    its fp32 beat and downbeat losses, batch size and frame length; rows are rounded up to 4 floats.  At the step, one
    all_gather brings every rank's slots to every rank ([world, S, row]), and micro-batch j of the step is read from
    rank j mod world, slot j div world: bt_grad_ordered_sum writes each .grad as the fp32 sum over the micro-batches in
    index order, and bt_train_running_replay applies their batch statistics in that order."""

    def __init__(self, module, opt, world: int, accumulate: int):
        self.module, self.world = module, world
        self.params = [p for group in opt.param_groups for p in group["params"]]
        self.P = sum(p.numel() for p in self.params)
        self.Q = module.batch_stat_floats(1, 1)  # one mean and variance per BatchNorm channel, whatever B and L
        row = (self.P + self.Q + 4 + 3) // 4 * 4
        S = -(-accumulate // world)
        self.send = torch.zeros(S, row, device=module.engine.device)
        self.recv = torch.empty(world, S, row, device=module.engine.device)
        self.grads = [torch.empty_like(p) for p in self.params]  # every step's .grad tensors, allocated once

    def stats(self, slot: int) -> torch.Tensor:
        """Where the forward pass of the micro-batch in `slot` writes its batch statistics."""
        return self.send[slot, self.P : self.P + self.Q]

    def pack(self, slot: int, lb, ld, shape) -> None:
        """After the backward pass of the micro-batch in `slot`: its gradients and losses into the slot, and the
        gradients set to None for the next micro-batch."""
        B, L = shape[0], shape[1]
        self.send[slot, self.P + self.Q : self.P + self.Q + 4] = torch.stack(
            [lb.detach(), ld.detach(), lb.new_tensor(float(B)), lb.new_tensor(float(L))])
        self.module.engine.grad_pack([p.grad for p in self.params], self.send[slot])
        for p in self.params:
            p.grad = None

    def reduce(self, k: int) -> list:
        """At the step of a group of k micro-batches: the gather, every .grad as the ordered sum, the running
        statistics replayed; returns each micro-batch's fp32 (beat, downbeat) losses and batch size, in order."""
        dist.all_gather(list(self.recv.unbind(0)), self.send)
        rows = [self.recv[j % self.world, j // self.world] for j in range(k)]
        for p, g in zip(self.params, self.grads):
            p.grad = g
        self.module.engine.grad_ordered_sum(self.grads, rows)
        tails = [row[self.P + self.Q : self.P + self.Q + 4] for row in rows]
        shapes = [tuple(int(v) for v in t[2:].tolist()) for t in tails]
        start = 0  # one replay per run of micro-batches of one shape
        for j in range(1, k + 1):
            if j == k or shapes[j] != shapes[start]:
                self.module.replay_batch_stats([row[self.P : self.P + self.Q] for row in rows[start:j]],
                                               *shapes[start])
                start = j
        return [(t[:2], B) for t, (B, _) in zip(tails, shapes)]


def build_parser() -> argparse.ArgumentParser:
    """The reference's train.py flags, names and defaults; --data and --checkpoint-dir stand for its fixed paths."""
    ap = argparse.ArgumentParser(prog="python -m beat_this_b200.train",
                                 description="Train a BeatThis model on a prepared dataset on one GPU, or "
                                             "data-parallel on several under torchrun.")
    add = ap.add_argument
    flag = argparse.BooleanOptionalAction
    add("--data", default="data", help="prepared dataset directory (annotations/ and audio/spectrograms/) [%(default)s]")
    add("--checkpoint-dir", default="checkpoints", help="where the checkpoint goes [%(default)s]")
    add("--name", type=str, default="")
    add("--gpu", type=int, default=int(os.environ.get("LOCAL_RANK", "0")),
        help="CUDA device (default: LOCAL_RANK under torchrun, else 0)")
    add("--force-flash-attention", default=False, action=flag, help="accepted, no effect")
    add("--compile", action="store", nargs="*", type=str, default=["frontend", "transformer_blocks", "task_heads"],
        help="accepted, no effect")
    add("--n-layers", type=int, default=6)
    add("--transformer-dim", type=int, default=512)
    add("--frontend-dropout", type=float, default=0.1, help="dropout rate to apply in the frontend")
    add("--transformer-dropout", type=float, default=0.2, help="dropout rate to apply in the main transformer blocks")
    add("--lr", type=float, default=0.0008)
    add("--weight-decay", type=float, default=0.01)
    add("--logger", type=str, choices=["wandb", "none"], default="none", help="only none: there is no wandb")
    add("--num-workers", type=int, default=8, help="accepted, no effect")
    add("--n-heads", type=int, default=16, help="accepted, no effect (the reference does not use it either)")
    add("--fps", type=int, default=50, help="The spectrograms fps.")
    add("--loss", type=str, default="shift_tolerant_weighted_bce",
        choices=["shift_tolerant_weighted_bce", "fast_shift_tolerant_weighted_bce", "weighted_bce", "bce"])
    add("--warmup-steps", type=int, default=1000, help="warmup steps for optimizer")
    add("--max-epochs", type=int, default=100, help="max epochs for training")
    add("--batch-size", type=int, default=8, help="batch size for training")
    add("--accumulate-grad-batches", type=int, default=8)
    add("--train-length", type=int, default=1500, help="maximum seq length for training in frames")
    add("--dbn", default=False, action=flag, help="use the DBN post-processor in validation")
    add("--eval-trim-beats", metavar="SECONDS", type=float, default=5,
        help="Skip the first given seconds per piece in evaluating (default: %(default)s)")
    add("--val-frequency", metavar="N", type=int, default=5, help="validate every N epochs (default: %(default)s)")
    add("--tempo-augmentation", default=True, action=flag, help="Use precomputed tempo augmentation")
    add("--pitch-augmentation", default=True, action=flag, help="Use precomputed pitch augmentation")
    add("--mask-augmentation", default=True, action=flag, help="Use online mask augmentation")
    add("--sum-head", default=True, action=flag, help="Use SumHead instead of two separate Linear heads")
    add("--partial-transformers", default=True, action=flag, help="Use Partial transformers in the frontend")
    add("--length-based-oversampling-factor", type=float, default=0.65,
        help="The factor to oversample the long pieces in the dataset. Set to 0 to only take one excerpt for each "
             "piece.")
    add("--val", default=True, action=flag, help="Train on all data, including validation data, excluding test data "
                                                 "(--no-val); the validation metrics are still computed.")
    add("--hung-data", default=False, action=flag, help="Limit the training to Hung et al. data.")
    add("--fold", type=int, default=None, help="If given, the CV fold number to *not* train on (0-based).")
    add("--seed", type=int, default=0, help="Seed for the random number generators.")
    add("--resume-checkpoint", type=str, default=None, help="Resume training from a local checkpoint.")
    add("--resume-id", type=str, default=None, help="refused: a wandb run id, and there is no wandb")
    add("--test", default=True, action=flag, help="score the final checkpoint on the test split (--no-test: skip)")
    return ap


def parse_args(argv=None) -> dict:
    """fit's keyword arguments from a command line; --logger wandb and --resume-id are refused."""
    ap = build_parser()
    args = ap.parse_args(argv)
    if args.logger == "wandb" or args.resume_id is not None:
        ap.error("--logger wandb and --resume-id need wandb, which this command does not use")
    kw = vars(args)
    for k in ("force_flash_attention", "compile", "logger", "num_workers", "n_heads", "resume_id"):
        del kw[k]
    return kw


def main(argv=None) -> int:
    from .distributed import init_from_env

    rank, world, _ = init_from_env()  # NCCL under torchrun with more than one process
    kw = parse_args(argv)
    if rank == 0:
        print("Starting a new run with the following parameters:")
        print(kw)
    try:
        fit(**kw)
    finally:
        if world > 1 and dist.is_initialized():
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
