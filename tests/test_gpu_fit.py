"""beat_this_b200.train.fit and ``python -m beat_this_b200.train`` on a prepared dataset generated here: two training
datasets and gtzan, spectrograms brighter on beat frames (so the task is learnable), small0 at B 4, L 200,
accumulate 2, validating every epoch.  Checks Lightning's step rule, the schedule at every step, BatchNorm's batch
counts, the loss going down, the validation records, the checkpoint (inference, evaluate --datasplit test, the
reference's file name), and resume: 2 epochs in one run equal 1 epoch plus a resumed one bitwise, and a checkpoint
without this project's random states (the reference's layout) resumes."""
import json
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from beat_this_b200 import train as T
from beat_this_b200.prepare import BundleWriter
from conftest import ROOT

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = "cuda:0"
SMALL0 = dict(transformer_dim=128, n_layers=6)
RUN = dict(**SMALL0, batch_size=4, train_length=200, accumulate_grad_batches=2, val_frequency=1, warmup_steps=3,
           lr=2e-3, tempo_augmentation=False, pitch_augmentation=False, gpu=0)


def _write_tree(root, seed=0):
    rng = np.random.default_rng(seed)
    for ds, n_train, n_val in (("alpha", 12, 3), ("beta", 10, 3), ("gtzan", 4, 0)):
        ann = root / "annotations" / ds
        (ann / "annotations" / "beats").mkdir(parents=True)
        (ann / "info.json").write_text(json.dumps({"has_downbeats": True}))
        rows = []
        with BundleWriter(root / "audio" / "spectrograms" / f"{ds}.npz") as w:
            for i in range(n_train + n_val):
                stem = f"{ds}{i:02d}"
                T_ = int(rng.integers(300, 600))
                period = int(rng.integers(20, 30))
                beats = np.arange(int(rng.integers(0, period)), T_ - 2, period)
                spect = rng.standard_normal((T_, 128)).astype(np.float32) * 0.3
                spect[beats] += 2.0
                spect[beats[::4]] += 1.0
                w.add(stem, {"track": spect.astype(np.float16)})
                numbers = (np.arange(len(beats)) % 4) + 1
                (ann / "annotations" / "beats" / f"{stem}.beats").write_text(
                    "".join(f"{b / 50:.4f}\t{k}\n" for b, k in zip(beats, numbers)))
                rows.append(f"{stem}\t{'val' if i >= n_train else 'train'}\n")
        if ds != "gtzan":
            (ann / "single.split").write_text("".join(rows))
    return root


@pytest.fixture(scope="module")
def data(tmp_path_factory, lib_built):
    return _write_tree(tmp_path_factory.mktemp("fitdata"))


@pytest.fixture(scope="module")
def three_epochs(data, tmp_path_factory):
    ckdir = tmp_path_factory.mktemp("ck3")
    records = T.fit(str(data), str(ckdir), max_epochs=3, **RUN)
    return records, T.checkpoint_path(ckdir, **RUN), ckdir


def test_steps_schedule_and_losses(three_epochs, data):
    from beat_this_b200 import dataset as D

    records, path, _ = three_epochs
    tr, _ = D.train_val_items(data)
    n_items = len(D.BeatTrackingDataset(tr, data, 50, 200, length_based_oversampling_factor=0.65))
    batches = n_items // RUN["batch_size"]
    per_epoch = math.ceil(batches / RUN["accumulate_grad_batches"])
    assert [r["global_step"] for r in records] == [per_epoch * (e + 1) for e in range(3)]
    total = T.estimated_stepping_batches(batches, RUN["accumulate_grad_batches"], 3)
    lrs = [lr for r in records for lr in r["step_lr"]]
    want = []
    for s in range(total):  # the reference's factor, restated
        f = 0.5 * (1 + np.cos(np.pi * (s / total)))
        if s <= RUN["warmup_steps"]:
            f *= s / RUN["warmup_steps"]
        want.append(float(RUN["lr"] * f))
    assert lrs == want
    ckpt = torch.load(path, map_location="cpu", weights_only=True)
    assert ckpt["epoch"] == 2 and ckpt["global_step"] == total
    assert int(ckpt["state_dict"]["model.frontend.stem.bn1d.num_batches_tracked"]) == 3 * batches
    assert records[-1]["train_loss"] < records[0]["train_loss"], [r["train_loss"] for r in records]
    for r in records:
        for k in ("val_loss", "val_F-measure_beat", "val_Cemgil_beat", "val_F-measure_downbeat", "val_Cemgil_downbeat"):
            assert np.isfinite(r[k]), (k, r)
    assert set(records[-1]["test"]) >= {"F-measure_beat", "Cemgil_beat", "test_loss"}
    for k in ("hyper_parameters", "datamodule_hyper_parameters", "optimizer_states", "lr_schedulers", "beat_this_b200"):
        assert k in ckpt
    assert ckpt["hyper_parameters"]["fps"] == 50 and len(ckpt["hyper_parameters"]) == 18
    assert not any(k in ckpt for k in ("pytorch-lightning_version", "loops", "callbacks"))


def test_checkpoint_loads_for_inference_and_evaluation(three_epochs, data):
    from beat_this_b200 import evaluate as E
    from beat_this_b200.inference import load_model

    _, path, _ = three_epochs
    module = T.BeatThisModule.from_checkpoint(path, DEV)
    x = (torch.rand(2, 200, 128, generator=torch.Generator().manual_seed(3)) * 2).to(DEV)
    with torch.no_grad():
        want = module(x)
    got = load_model(path, DEV, float16=False)(x)
    for k in ("beat", "downbeat"):
        assert (got[k] - want[k]).abs().max().item() < 1e-3
    assert E.main(["--models", path, "--data", str(data), "--datasplit", "test", "--no-float16"]) == 0


def test_resume_is_bitwise(data, tmp_path):
    run = dict(RUN, max_epochs=2, test=False)
    whole = T.fit(str(data), str(tmp_path / "a"), **run)
    first = T.fit(str(data), str(tmp_path / "b"), epochs=1, **run)
    path_b = T.checkpoint_path(tmp_path / "b", **run)
    shutil.copy(path_b, tmp_path / "after_epoch0.ckpt")
    rest = T.fit(str(data), str(tmp_path / "b"), resume_checkpoint=path_b, **run)
    assert first + rest == whole
    a = torch.load(T.checkpoint_path(tmp_path / "a", **run), map_location="cpu", weights_only=True)
    b = torch.load(path_b, map_location="cpu", weights_only=True)
    for k in a["state_dict"]:
        assert torch.equal(a["state_dict"][k], b["state_dict"][k]), k
    sa, sb = a["optimizer_states"][0], b["optimizer_states"][0]
    assert sa["param_groups"] == sb["param_groups"]
    for i in sa["state"]:
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(sa["state"][i][k].cpu(), sb["state"][i][k].cpu()), (i, k)
    assert a["lr_schedulers"] == b["lr_schedulers"]

    # the reference's Lightning layout: no random states of this project, numpy scalars in the scheduler state
    ck = torch.load(tmp_path / "after_epoch0.ckpt", map_location="cpu", weights_only=True)
    del ck["beat_this_b200"]
    ck["lr_schedulers"][0]["_last_lr"] = [np.float64(v) for v in ck["lr_schedulers"][0]["_last_lr"]]
    ck.update({"pytorch-lightning_version": "2.4.0", "loops": {}, "callbacks": {}})
    torch.save(ck, tmp_path / "lightning.ckpt")
    resumed = T.fit(str(data), str(tmp_path / "c"), resume_checkpoint=str(tmp_path / "lightning.ckpt"), **run)
    assert [r["epoch"] for r in resumed] == [1] and resumed[0]["global_step"] == whole[1]["global_step"]


def test_command_writes_the_reference_checkpoint_name(data, tmp_path):
    cmd = [sys.executable, "-m", "beat_this_b200.train", "--max-epochs", "1", "--data", str(data), "--checkpoint-dir",
           str(tmp_path), "--transformer-dim", "128", "--batch-size", "4", "--train-length", "200",
           "--accumulate-grad-batches", "2", "--warmup-steps", "3", "--no-tempo-augmentation",
           "--no-pitch-augmentation", "--val-frequency", "1", "--no-test", "--name", "cli"]
    res = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-3000:]
    assert os.listdir(tmp_path) == ["cli S0 shift_tolerant_weighted_bce-h128-augFalseFalseTrue.ckpt"]
    rec = json.loads([ln for ln in res.stdout.splitlines() if ln.startswith('{"epoch"')][-1])
    assert rec["epoch"] == 0 and "val_F-measure_beat" in rec
