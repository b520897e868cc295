"""Data-parallel training on the GPU: the gradient-exchange kernels (bt_grad_pack, bt_grad_ordered_sum) against
torch's in-place adds bit for bit, bt_train_running_replay against sequential training-mode forward passes, and
``fit`` on several ranks against the one-process run with the same flags: the same checkpoint bytes and records.

Ranks run as processes spawned here on a free port, over gloo on one GPU (NCCL refuses two ranks on one device); the
NCCL and torchrun runs need two GPUs and are skipped on a machine with one."""
import ctypes
import hashlib
import json
import os
import socket
import subprocess
import sys
import traceback

import numpy as np
import pytest
import torch

from beat_this_b200 import _lib, synthetic
from beat_this_b200 import train as T
from beat_this_b200.engine import Engine
from beat_this_b200.prepare import BundleWriter
from conftest import ROOT
from support import DEV, _spect, bits, dev  # noqa: F401 (dev: a fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(3600)]
SMALL0 = dict(transformer_dim=128, n_layers=6)
RUN = dict(**SMALL0, batch_size=4, train_length=200, val_frequency=1, warmup_steps=3, lr=2e-3,
           tempo_augmentation=False, pitch_augmentation=False, length_based_oversampling_factor=0, max_epochs=2)
JOIN_TIMEOUT = 1200  # seconds a spawned run may take before its processes are killed
TWO_GPUS = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (NCCL refuses two ranks on one)")


# ---- the kernels alone -----------------------------------------------------------------------------------------------
SIZES = [0, 1, 3, 4, 5, 17, 255, 256, 257, 2047, 2048, 2049, 4097, 12000, 7, 0, 11999, 1, 8]
SENTINEL = -12345.678


def _values(n, g):
    """n fp32 values: normal ones of several magnitudes, with +-0, +-inf, NaN and subnormals sprinkled in."""
    x = torch.randn(n, generator=g) * torch.tensor([1e-3, 1.0, 1e3, 1e30])[torch.randint(0, 4, (n,), generator=g)]
    special = torch.tensor([0.0, -0.0, float("inf"), -float("inf"), float("nan"), 1e-40, -3e-42, 1.4e-45, -1e-38,
                            3e38, -3e38])
    pick = torch.rand(n, generator=g) < 0.1
    x[pick] = special[torch.randint(0, len(special), (int(pick.sum()),), generator=g)]
    return x.float()


def _tensors(g, shift):
    """One tensor per SIZES entry, each a view `shift` floats into a buffer whose other elements hold SENTINEL."""
    bufs, views = [], []
    for i, n in enumerate(SIZES):
        buf = torch.full((n + 2,), SENTINEL, device=DEV)
        s = shift if i % 2 else 0  # alternate 16-byte aligned entries and entries one float off
        buf[s : s + n] = _values(n, g).to(DEV)
        bufs.append((buf, s, n))
        views.append(buf[s : s + n])
    return bufs, views


def _sentinels_intact(bufs):
    for buf, s, n in bufs:
        rest = torch.cat([buf[:s], buf[s + n :]])
        assert bool((rest == SENTINEL).all()), "an element outside the table was written"


def _row(total, g, shift, fill=None):
    base = torch.full((total + 3,), SENTINEL, device=DEV)
    if fill is not None:
        base[shift : shift + total] = fill
    else:
        base[shift : shift + total] = _values(total, g).to(DEV)
    return base, base[shift : shift + total]


def _train_module():
    return T.BeatThisModule.from_checkpoint(synthetic.make_checkpoint("small0", 0), DEV, train_mode=True)


def test_pack_round_trips_bitwise(dev):
    eng = Engine.shared(DEV)
    g = torch.Generator().manual_seed(0)
    for shift in (0, 1):
        bufs, grads = _tensors(g, shift)
        total = sum(SIZES)
        base, row = _row(total, g, shift, fill=0.0)
        n0 = eng.launches
        eng.grad_pack(grads, row)
        assert eng.launches == n0 + 1
        torch.cuda.synchronize()
        assert torch.equal(bits(row), bits(torch.cat(grads)))
        assert bool((base[:shift] == SENTINEL).all()) and bool((base[shift + total :] == SENTINEL).all())
        _sentinels_intact(bufs)
        back_bufs, back = _tensors(g, 1 - shift)
        n0 = eng.launches
        eng.grad_ordered_sum(back, [row])
        assert eng.launches == n0 + 1
        torch.cuda.synchronize()
        for a, b in zip(back, grads):
            assert torch.equal(bits(a), bits(b))
        _sentinels_intact(back_bufs)


@pytest.mark.parametrize("k", range(1, 9))
def test_ordered_sum_equals_sequential_in_place_adds(dev, k):
    eng = Engine.shared(DEV)
    g = torch.Generator().manual_seed(100 + k)
    total = sum(SIZES)
    for shift in (0, 1):
        rows = [_row(total, g, (shift + j) % 2)[1] for j in range(k)]
        copies = [bits(r).clone() for r in rows]
        bufs, grads = _tensors(g, shift)
        n0 = eng.launches
        eng.grad_ordered_sum(grads, rows)
        assert eng.launches == n0 + 1
        off = 0
        for n, got in zip(SIZES, grads):
            want = rows[0][off : off + n].clone()  # AccumulateGrad: the first gradient as it is, then in-place adds
            for r in rows[1:]:
                want.add_(r[off : off + n])
            assert torch.equal(bits(got), bits(want)), (k, shift, n)
            off += n
        _sentinels_intact(bufs)
        for r, c in zip(rows, copies):  # the rows are only read
            assert torch.equal(bits(r), c)


def test_refusals_launch_nothing(dev):
    module = _train_module()
    eng = module.engine
    lib, ctx = eng.lib, eng.ctx
    stream = eng._stream()
    x = torch.zeros(64, device=DEV)
    E = _lib.bt_grad_entry
    ok = (E * 1)(E(x.data_ptr(), 64))
    null_grad = (E * 1)(E(None, 4))
    neg = (E * 1)(E(x.data_ptr(), -1))
    ptrs = ctypes.c_void_p * 2
    rows = ptrs(x.data_ptr(), x.data_ptr())
    null_rows = ptrs(x.data_ptr(), None)
    n0 = eng.launches
    refused = [
        lib.bt_grad_pack(ctx, ok, -1, x.data_ptr(), stream),
        lib.bt_grad_pack(ctx, None, 1, x.data_ptr(), stream),
        lib.bt_grad_pack(ctx, neg, 1, x.data_ptr(), stream),
        lib.bt_grad_pack(ctx, null_grad, 1, x.data_ptr(), stream),
        lib.bt_grad_pack(ctx, ok, 1, None, stream),
        lib.bt_grad_ordered_sum(ctx, ok, -1, rows, 2, stream),
        lib.bt_grad_ordered_sum(ctx, None, 1, rows, 2, stream),
        lib.bt_grad_ordered_sum(ctx, neg, 1, rows, 2, stream),
        lib.bt_grad_ordered_sum(ctx, null_grad, 1, rows, 2, stream),
        lib.bt_grad_ordered_sum(ctx, ok, 1, rows, 0, stream),
        lib.bt_grad_ordered_sum(ctx, ok, 1, None, 2, stream),
        lib.bt_grad_ordered_sum(ctx, ok, 1, null_rows, 2, stream),
    ]
    running = module._running()
    n_params = len(running)
    table = eng._table_ptrs(running, "running statistic")
    stats = torch.zeros(module.batch_stat_floats(2, 64), device=DEV)
    sp = ptrs(stats.data_ptr(), stats.data_ptr())
    sp_null = ptrs(stats.data_ptr(), None)
    holed = list(table)
    holed[[i for i, name in enumerate(module._names) if name.endswith(".running_var")][0]] = None
    holed = (ctypes.c_void_p * n_params)(*holed)
    refused += [
        lib.bt_train_running_replay(ctx, table, n_params, sp, 2, 0, 64, stream),
        lib.bt_train_running_replay(ctx, table, n_params, sp, 2, 1, 1, stream),
        lib.bt_train_running_replay(ctx, table, n_params - 1, sp, 2, 2, 64, stream),
        lib.bt_train_running_replay(ctx, None, n_params, sp, 2, 2, 64, stream),
        lib.bt_train_running_replay(ctx, holed, n_params, sp, 2, 2, 64, stream),
        lib.bt_train_running_replay(ctx, table, n_params, sp, -1, 2, 64, stream),
        lib.bt_train_running_replay(ctx, table, n_params, None, 2, 2, 64, stream),
        lib.bt_train_running_replay(ctx, table, n_params, sp_null, 2, 2, 64, stream),
    ]
    assert refused == [-1] * len(refused), refused
    assert eng.launches == n0
    # nothing to do launches nothing
    empty = (E * 2)(E(x.data_ptr(), 0), E(None, 0))
    assert lib.bt_grad_pack(ctx, empty, 2, x.data_ptr(), stream) == 0
    assert lib.bt_grad_ordered_sum(ctx, empty, 2, rows, 2, stream) == 0
    assert lib.bt_train_running_replay(ctx, table, n_params, None, 0, 2, 64, stream) == 0
    assert eng.launches == n0


@pytest.mark.parametrize("k", [1, 3])
def test_running_replay_equals_sequential_training_forwards(dev, k):
    B, L = 2, 64
    plain, captured = _train_module(), _train_module()
    plain.train(), captured.train()
    spects = [_spect(B, L, seed=10 + j).to(DEV) for j in range(k)]
    start = {n: t.clone() for n, t in captured.state_dict().items()}
    torch.manual_seed(5)
    want = [plain(x) for x in spects]
    torch.manual_seed(5)
    stats = [torch.full((captured.batch_stat_floats(B, L),), float("nan"), device=DEV) for _ in range(k)]
    got = [captured(x, batch_stats=s) for x, s in zip(spects, stats)]
    for a, b in zip(want, got):  # the same function: the capture only redirects the running statistics
        assert torch.equal(bits(a["beat"]), bits(b["beat"])) and torch.equal(bits(a["downbeat"]), bits(b["downbeat"]))
    for name, t in captured.state_dict().items():  # untouched until the replay
        assert torch.equal(t, start[name]), name
    for s in stats:
        assert not bool(torch.isnan(s).any())
    n0 = captured.engine.launches
    captured.replay_batch_stats(stats, B, L)
    n_bn = sum(name.endswith(".running_mean") for name in captured._names)
    assert captured.engine.launches == n0 + 2 * n_bn * k
    ps, cs = plain.state_dict(), captured.state_dict()
    for name in ps:
        if "running" in name or name.endswith("num_batches_tracked"):
            assert torch.equal(bits(ps[name]) if ps[name].is_floating_point() else ps[name],
                               bits(cs[name]) if cs[name].is_floating_point() else cs[name]), name
    counter = "frontend.stem.bn1d.num_batches_tracked"
    assert int(cs[counter]) == int(start[counter]) + k


# ---- fit on several ranks ------------------------------------------------------------------------------------------
def _write_tree(root, seed=1):
    """Two training datasets of 11 and 10 pieces with 3 validation pieces each, and gtzan for the test: 21 training
    excerpts of 200 frames make 5 batches of 4."""
    rng = np.random.default_rng(seed)
    for ds, n_train, n_val in (("alpha", 11, 3), ("beta", 10, 3), ("gtzan", 3, 0)):
        ann = root / "annotations" / ds
        (ann / "annotations" / "beats").mkdir(parents=True)
        (ann / "info.json").write_text(json.dumps({"has_downbeats": True}))
        rows = []
        with BundleWriter(root / "audio" / "spectrograms" / f"{ds}.npz") as w:
            for i in range(n_train + n_val):
                stem = f"{ds}{i:02d}"
                frames = int(rng.integers(250, 450))
                period = int(rng.integers(18, 32))
                beats = np.arange(int(rng.integers(0, period)), frames - 2, period)
                spect = rng.standard_normal((frames, 128)).astype(np.float32) * 0.3
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


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(rank, world, port, backend, devices, kw, out):
    """One rank of a spawned run: fit, with a digest of the parameters after every optimizer step."""
    import torch.distributed as dist

    from beat_this_b200 import optim
    from beat_this_b200 import train as T

    try:
        dist.init_process_group(backend, init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
        digests, step = [], optim.AdamW.step

        def hooked(self, closure=None):
            loss = step(self, closure)
            flat = torch.cat([p.detach().reshape(-1) for group in self.param_groups for p in group["params"]])
            digests.append(hashlib.sha256(flat.cpu().numpy().tobytes()).hexdigest())
            return loss

        optim.AdamW.step = hooked
        records = T.fit(**kw, gpu=devices[rank])
        out.put((rank, "ok", records, digests))
    except BaseException as e:  # noqa: BLE001 (reported to the test)
        out.put((rank, "error", f"{type(e).__name__}: {e}", traceback.format_exc()))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _spawn(world, kw, backend="gloo", devices=None):
    """fit on `world` spawned ranks; returns each rank's (status, records or error, digests or traceback).  Every
    process is joined, or killed after JOIN_TIMEOUT."""
    ctx = torch.multiprocessing.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    devices = devices or [0] * world
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, backend, devices, kw, out)) for r in range(world)]
    for p in procs:
        p.start()
    results = {}
    try:
        for _ in range(world):
            rank, *res = out.get(timeout=JOIN_TIMEOUT)
            results[rank] = res
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    assert len(results) == world, f"only ranks {sorted(results)} reported"
    return [results[r] for r in range(world)]


def _same(a, b, where="checkpoint"):
    """Bitwise equality of two loaded checkpoints' contents."""
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape, where
        a, b = a.cpu(), b.cpu()
        if a.is_floating_point():
            a, b = a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)
        assert torch.equal(a, b), where
    elif isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b), (where, list(a), list(b))
        for k in a:
            _same(a[k], b[k], f"{where}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{where}[{i}]")
    elif isinstance(a, float):
        assert isinstance(b, float) and np.float64(a).view(np.int64) == np.float64(b).view(np.int64), (where, a, b)
    else:
        assert a == b, (where, a, b)


def _check_equal_runs(path_a, path_b, records_a, records_b, same_bytes=True):
    """Equal records and checkpoint contents; same_bytes: equal files too.  A resumed run's checkpoint holds the same
    values but pickles fewer shared objects than an uninterrupted run's, at any world size, so its bytes differ."""
    assert json.dumps(records_a) == json.dumps(records_b)
    a = torch.load(path_a, map_location="cpu", weights_only=True)
    b = torch.load(path_b, map_location="cpu", weights_only=True)
    _same(a, b)
    if same_bytes:
        with open(path_a, "rb") as fa, open(path_b, "rb") as fb:
            assert fa.read() == fb.read(), "the checkpoint files differ"


def _ranks_ok(results):
    for status, what, detail in results:
        assert status == "ok", f"{what}\n{detail}"
    records, digests = results[0][1], results[0][2]
    for _, r, d in results[1:]:
        assert json.dumps(r) == json.dumps(records), "the ranks returned different records"
        assert d == digests, "the ranks' parameters differ after an optimizer step"
    return records


@pytest.fixture(scope="module")
def data(tmp_path_factory, lib_built):
    from beat_this_b200 import dataset as D

    root = _write_tree(tmp_path_factory.mktemp("dpdata"))
    tr, _ = D.train_val_items(root)
    assert len(D.BeatTrackingDataset(tr, root, 50, 200)) // 4 == 5  # five micro-batches per epoch
    return root


@pytest.fixture(scope="module")
def one_process(data, tmp_path_factory):
    """The one-process runs the data-parallel ones must equal: accumulate 2 (with the final test) and 3."""
    out = {}
    for acc, test in ((2, True), (3, False)):
        ckdir = tmp_path_factory.mktemp(f"one{acc}")
        kw = dict(RUN, data=str(data), checkpoint_dir=str(ckdir), accumulate_grad_batches=acc, test=test)
        out[acc] = (kw, T.fit(**kw, gpu=0), T.checkpoint_path(**kw))
    return out


@pytest.mark.parametrize("acc", [2, 3])
def test_two_ranks_equal_one_process_bitwise(one_process, tmp_path, acc):
    # accumulate 2: the epoch's last step has one micro-batch and rank 1 sits it out; accumulate 3: rank 0 runs two
    # micro-batches of the first step and rank 1 one
    kw, records, path = one_process[acc]
    kw = dict(kw, checkpoint_dir=str(tmp_path))
    got = _ranks_ok(_spawn(2, kw))
    assert len(got) == 2 and all("val_loss" in r for r in got) and ("test" in got[-1]) == (acc == 2)
    _check_equal_runs(path, T.checkpoint_path(**kw), records, got)


def test_checkpoints_pass_between_world_sizes(one_process, tmp_path):
    kw, records, path = one_process[3]
    kw = dict(kw, checkpoint_dir=str(tmp_path))
    first = _ranks_ok(_spawn(2, dict(kw, epochs=1)))
    rest = T.fit(**kw, gpu=0, resume_checkpoint=T.checkpoint_path(**kw))
    _check_equal_runs(path, T.checkpoint_path(**kw), records, first + rest, same_bytes=False)


def test_more_ranks_than_micro_batches_are_refused_on_every_rank(data, tmp_path):
    kw = dict(RUN, data=str(data), checkpoint_dir=str(tmp_path / "never"), accumulate_grad_batches=2, test=False)
    results = _spawn(3, kw)
    for status, what, _ in results:
        assert status == "error" and what.startswith("ValueError") and "would never train" in what, what
    assert not os.path.exists(tmp_path / "never")


@TWO_GPUS
def test_two_gpus_over_nccl_equal_one_process_bitwise(one_process, tmp_path):
    kw, records, path = one_process[2]
    kw = dict(kw, checkpoint_dir=str(tmp_path))
    got = _ranks_ok(_spawn(2, kw, backend="nccl", devices=[0, 1]))
    _check_equal_runs(path, T.checkpoint_path(**kw), records, got)


@TWO_GPUS
def test_torchrun_command_equals_one_process(data, tmp_path):
    argv = ["--max-epochs", "1", "--data", str(data), "--transformer-dim", "128", "--batch-size", "4",
            "--train-length", "200", "--accumulate-grad-batches", "3", "--warmup-steps", "3",
            "--no-tempo-augmentation", "--no-pitch-augmentation", "--val-frequency", "1", "--no-test",
            "--length-based-oversampling-factor", "0", "--name", "dp"]
    kw = T.parse_args(argv + ["--checkpoint-dir", str(tmp_path / "one"), "--gpu", "0"])
    T.fit(**kw)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), "-m", "beat_this_b200.train", *argv, "--checkpoint-dir",
           str(tmp_path / "two")]
    res = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=JOIN_TIMEOUT)
    assert res.returncode == 0, res.stderr[-3000:]
    name = os.listdir(tmp_path / "one")
    assert os.listdir(tmp_path / "two") == name
    with open(tmp_path / "one" / name[0], "rb") as a, open(tmp_path / "two" / name[0], "rb") as b:
        assert a.read() == b.read()
