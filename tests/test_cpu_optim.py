"""CPU tests (no GPU) of the training run's host side: the learning-rate schedule and the parameter groups against
the reference's (tests/golden/optim.npz, oracle/make_golden_optim.py), Lightning's step plan, the command line, and
the AdamW kernel's machine code in the built library."""
import json
import os
import re

import numpy as np
import pytest
import torch

from beat_this_b200 import _lib
from beat_this_b200 import train as T
from beat_this_b200.optim import CosineWarmupScheduler
from conftest import GOLDEN
from support import sass


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "optim.npz"))


def test_schedule_equals_the_reference_bitwise(gold):
    for k, (warmup, max_iters) in enumerate(gold["sched"]):
        opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.0008)
        sched = CosineWarmupScheduler(opt, int(warmup), int(max_iters))
        lrs = [opt.param_groups[0]["lr"]]
        for _ in range(len(gold[f"lr{k}"]) - 1):
            opt.step()
            sched.step()
            lrs.append(opt.param_groups[0]["lr"])
        want = gold[f"lr{k}"]
        assert want[0] == 0.0 and len(want) > max_iters + warmup  # step 0 and both branches are covered
        assert np.array_equal(np.asarray(lrs, dtype=np.float64).view(np.int64), want.view(np.int64)), (warmup, max_iters)


def test_warmup_below_one_is_refused():
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.1)
    with pytest.raises(ValueError):
        CosineWarmupScheduler(opt, 0, 10)


def test_groups_of_the_parameter_table_equal_the_reference(gold, lib_built):
    groups = json.loads(str(gold["groups"]))
    table = _lib.train_param_table({"transformer_dim": 64, "n_layers": 1})
    decay = [n for n, shape, trainable in table if trainable and len(shape) >= 2]
    rest = [n for n, shape, trainable in table if trainable and len(shape) <= 1]
    assert [decay, rest] == [[n.removeprefix("model.") for n in g["names"]] for g in groups]
    assert [g["hparams"]["weight_decay"] for g in groups] == [0.01, 0]


@pytest.mark.parametrize("batches, accumulate", [(1, 1), (8, 8), (10, 4), (7, 3), (5, 8), (16, 2), (9, 1)])
def test_step_plan_follows_lightning(batches, accumulate):
    # Lightning steps when (batch_idx + 1) % accumulate == 0 or on the epoch's last batch
    want = [i for i in range(batches) if (i + 1) % accumulate == 0 or i == batches - 1]
    assert T.step_plan(batches, accumulate) == want
    for epochs in (1, 3):
        assert T.estimated_stepping_batches(batches, accumulate, epochs) == len(want) * epochs


def test_command_line_takes_the_reference_flags():
    kw = T.parse_args([])
    assert kw["lr"] == 0.0008 and kw["max_epochs"] == 100 and kw["accumulate_grad_batches"] == 8
    assert kw["val_frequency"] == 5 and kw["length_based_oversampling_factor"] == 0.65 and kw["warmup_steps"] == 1000
    kw = T.parse_args(["--name", "run", "--no-val", "--hung-data", "--fold", "3", "--loss", "bce", "--no-sum-head",
                       "--no-partial-transformers", "--no-tempo-augmentation", "--compile", "--n-heads", "4",
                       "--num-workers", "2", "--force-flash-attention", "--seed", "7", "--gpu", "0", "--dbn",
                       "--eval-trim-beats", "2.5", "--data", "d", "--checkpoint-dir", "c", "--no-test"])
    assert not kw["val"] and kw["hung_data"] and kw["fold"] == 3 and kw["dbn"] and not kw["test"]
    assert T.checkpoint_path(**kw) == os.path.join(
        "c", "run S7 noval hung fold3 bce-h512-augFalseTrueTrue nosumH  nopartialT.ckpt")
    assert T.checkpoint_path(**T.parse_args([])) == os.path.join(
        "checkpoints", "S0 shift_tolerant_weighted_bce-h512-augTrueTrueTrue.ckpt")
    assert T.augmentations(True, True, True)["tempo"] == {"min": -20, "max": 20, "stride": 4}
    for refused in (["--logger", "wandb"], ["--resume-id", "abc"]):
        with pytest.raises(SystemExit):
            T.parse_args(refused)


def test_adamw_kernel_has_no_local_memory(lib_built):
    fn, found, local = None, set(), []
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
            if "adamw" in fn:
                found.add(fn)
        elif fn and "adamw" in fn and re.search(r"\b(STL|LDL)(\.\w+)*\b", line):
            local.append(line.strip())
    assert len(found) == 1 and "12adamw_kernel" in next(iter(found)), found
    assert not re.search(r"tr_\w+?_kernel", next(iter(found)))
    assert not local, local
