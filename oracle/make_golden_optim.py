"""Generate tests/golden/optim.npz by running the UNMODIFIED reference's optimizer setup
(PLBeatThis.configure_optimizers and CosineWarmupScheduler, beat_this/model/pl_module.py:279-369) on the CPU.

    python oracle/make_golden_optim.py <beat_this source tree>      (or BEAT_THIS_REFERENCE=<tree>)

pytorch_lightning and mir_eval are stubs in sys.modules: pytorch_lightning's LightningModule is an nn.Module whose
save_hyperparameters() keeps the constructor's arguments (all PLBeatThis needs of it), LightningDataModule the shim's
of oracle/shims, and mir_eval is empty (Metrics calls it only when used).  A namespace stands in for the trainer,
carrying estimated_stepping_batches.  The model is tiny (transformer_dim 64, one layer).  The fixture holds:

* groups: JSON list of the two parameter groups, each {"names": state_dict names in order, "hparams": the group's
  other keys, initial_lr included};
* lr{k}: param_groups[0]["lr"] after construction and after every scheduler.step(), float64, for the (warmup,
  max_iters) pair sched[k], run to max_iters + warmup + 3 steps;
* after K AdamW and scheduler steps (warmup STEP_WARMUP, max_iters K, lr STEP_LR, weight_decay STEP_WD) on parameters
  and gradients drawn from torch.Generator().manual_seed(SEED), in state_dict order of the trainable entries
  (trainable: their names), first every parameter (randn * PARAM_SCALE), then per step every gradient
  (randn * GRAD_SCALE): fp_param, fp_exp_avg, fp_exp_avg_sq, one fingerprint row per entry
  (oracle/train_fingerprint.py, probes seeded by the entry's position in `trainable`), and final_lr;
* opt_skeleton / sched_skeleton: JSON state_dict skeletons of the optimizer and the scheduler after those steps
  (oracle/state_skeleton.py).
"""
from __future__ import annotations

import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("BEAT_THIS_REFERENCE")
if not REF:
    sys.exit("usage: python oracle/make_golden_optim.py <beat_this source tree>")
sys.path.insert(0, os.path.join(HERE, "shims"))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)
sys.modules["mir_eval"] = types.ModuleType("mir_eval")

import inspect  # noqa: E402

import numpy as np  # noqa: E402
import pytorch_lightning as _pl_shim  # noqa: E402  (oracle/shims: LightningDataModule only)
import torch  # noqa: E402


class LightningModule(torch.nn.Module):
    """An nn.Module whose save_hyperparameters() keeps the caller's constructor arguments in ``hparams``."""

    def save_hyperparameters(self, *args, **kwargs):
        names, _, _, values = inspect.getargvalues(inspect.currentframe().f_back)
        self.hparams = {n: values[n] for n in names if n != "self"}


_pl = types.ModuleType("pytorch_lightning")
_pl.LightningDataModule, _pl.LightningModule = _pl_shim.LightningDataModule, LightningModule
sys.modules["pytorch_lightning"] = _pl

from beat_this.model.pl_module import PLBeatThis  # noqa: E402  (the reference)
from oracle.state_skeleton import skeleton  # noqa: E402
from oracle.train_fingerprint import fingerprint  # noqa: E402

MODEL = dict(transformer_dim=64, n_layers=1)  # the narrowest width the library runs
SCHEDULES = [(5, 20), (1, 7), (10, 10), (12, 4), (3, 40)]
K, STEP_WARMUP, STEP_LR, STEP_WD = 20, 5, 1e-2, 0.05
SEED, PARAM_SCALE, GRAD_SCALE = 1234, 0.5, 0.1


def configured(estimated_stepping_batches, **kw):
    pl = PLBeatThis(**MODEL, **kw)
    pl.trainer = types.SimpleNamespace(estimated_stepping_batches=estimated_stepping_batches)
    conf = pl.configure_optimizers()
    assert conf["lr_scheduler"]["interval"] == "step"
    return pl, conf["optimizer"], conf["lr_scheduler"]["scheduler"]


def main():
    out = {}
    pl, opt, _ = configured(100)
    name_of = {id(p): n for n, p in pl.named_parameters()}
    groups = [{"names": [name_of[id(p)] for p in g["params"]],
               "hparams": {k: v for k, v in g.items() if k != "params"}} for g in opt.param_groups]
    out["groups"] = np.array(json.dumps(groups, default=float))
    print("groups:", [len(g["names"]) for g in groups])

    for k, (warmup, max_iters) in enumerate(SCHEDULES):
        _, opt, sched = configured(max_iters, warmup_steps=warmup)
        lrs = [opt.param_groups[0]["lr"]]
        for _ in range(max_iters + warmup + 3):
            opt.step()  # no gradients: updates nothing
            sched.step()
            lrs.append(opt.param_groups[0]["lr"])
            assert opt.param_groups[1]["lr"] == lrs[-1]
        out[f"lr{k}"] = np.asarray(lrs, dtype=np.float64)
    out["sched"] = np.asarray(SCHEDULES, dtype=np.int64)

    pl, opt, sched = configured(K, warmup_steps=STEP_WARMUP, lr=STEP_LR, weight_decay=STEP_WD)
    named = dict(pl.named_parameters())
    trainable = [n for n in pl.state_dict() if n in named and named[n].requires_grad]
    g = torch.Generator().manual_seed(SEED)
    with torch.no_grad():
        for n in trainable:
            named[n].copy_(torch.randn(named[n].shape, generator=g) * PARAM_SCALE)
    for _ in range(K):
        for n in trainable:
            named[n].grad = torch.randn(named[n].shape, generator=g) * GRAD_SCALE
        opt.step()
        sched.step()
    for key in ("param", "exp_avg", "exp_avg_sq"):
        rows = [fingerprint((named[n] if key == "param" else opt.state[named[n]][key]).detach().numpy(), i)
                for i, n in enumerate(trainable)]
        out[f"fp_{key}"] = np.stack(rows)
    out["trainable"] = np.array(trainable)
    out["final_lr"] = np.array(opt.param_groups[0]["lr"], dtype=np.float64)
    out["steps"] = np.array([K, STEP_WARMUP], dtype=np.int64)
    out["step_hparams"] = np.array([STEP_LR, STEP_WD, PARAM_SCALE, GRAD_SCALE], dtype=np.float64)
    out["seed"] = np.array(SEED)
    out["opt_skeleton"] = np.array(json.dumps(skeleton(opt.state_dict())))
    out["sched_skeleton"] = np.array(json.dumps(skeleton(sched.state_dict())))
    path = os.path.join(ROOT, "tests", "golden", "optim.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
