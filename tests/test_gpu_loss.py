"""bt_beat_loss / bt_beat_loss_backward (csrc/kernels_loss.cu) against the numpy restatement of their contract
(tests/loss_reference.py) and the unmodified reference's outputs (tests/golden/loss.npz), the loss modules' autograd
path, and the test losses of beat_this_b200.evaluate."""
import ctypes

import numpy as np
import pytest
import torch

import loss_reference as R
from loss_reference import CASES, GOLD, GRAD_TOL, fixture_case

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = "cuda:0"
KINDS = (R.MASKED_BCE, R.SHIFT_TOLERANT, R.SPLIT_SHIFT_TOLERANT)


def _rows(rng, kind, t, n):
    """n seeded and edge rows for one (kind, t): minimum lengths, tie-heavy logits, all-zero masks, soft targets, ragged
    lengths up to 100 000 frames."""
    lo = 1 if kind == R.MASKED_BCE else 4 * t + 1
    lens, xs, ys, ms = [], [], [], []
    for i in range(n):
        v = i % 6
        L = lo if v == 0 else int(rng.integers(lo, lo + 600)) if v < 5 else int(rng.integers(20000, 100001))
        x = rng.choice(np.array([-1.5, 0.25, 2.0], np.float32), L) if v in (0, 1) else (rng.standard_normal(L) * 3).astype(np.float32)
        y = (rng.random(L) < 0.1).astype(np.float32)
        if v in (2, 4):
            y = y * 0.9 + 0.05
        m = np.zeros(L, np.float32) if v == 3 else np.where(rng.random(L) < 0.1, 0.0, rng.random(L)).astype(np.float32)
        if v == 1:
            m = (rng.random(L) < 0.9).astype(np.float32)
        lens.append(L)
        xs.append(x)
        ys.append(y)
        ms.append(m)
    return np.concatenate(xs), np.concatenate(ys), np.concatenate(ms), np.concatenate([[0], np.cumsum(lens)]).tolist()


def _kernel(x, y, m, off, kind, t, pw, g=0.7):
    """(row losses, mean, gradient) from the kernels, on host."""
    from beat_this_b200 import loss as L

    xd = torch.from_numpy(x).to(DEV).requires_grad_(True)
    yd, md = torch.from_numpy(y).to(DEV), None if m is None else torch.from_numpy(m).to(DEV)
    rows, mean = L.beat_loss_rows(xd.detach(), yd, md, off, kind, t, pw)
    out = L._BeatLoss.apply(xd, yd, md, off, kind, t, pw)
    (out * g).backward()
    assert torch.equal(out.detach(), mean)
    return rows.cpu().numpy(), float(mean), xd.grad.cpu().numpy()


def _assert_close(rows, mean, grad, want, g=0.7):
    wrows, wmean, wgrad = want
    assert np.all(np.abs(rows - wrows) <= 1e-6 * np.abs(wrows) + 1e-12)
    assert abs(mean - wmean) <= 1e-6 * abs(wmean) + 1e-12
    assert np.max(np.abs(grad - wgrad)) <= GRAD_TOL * np.max(np.abs(wgrad))
    assert np.array_equal(grad != 0, wgrad != 0)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("t", [0, 1, 3, 7])
@pytest.mark.parametrize("pw", [1.0, 4.5])
def test_kernel_equals_restatement(lib_built, kind, t, pw):
    rng = np.random.default_rng(100 * kind + 10 * t + int(pw))
    x, y, m, off = _rows(rng, kind, t, 60)
    got = _kernel(x, y, m, off, kind, t, pw)
    _assert_close(*got, R.loss_rows(x, y, m, off, kind, t, pw, grad_mean=0.7))
    if kind != R.SPLIT_SHIFT_TOLERANT:  # no mask
        got = _kernel(x, y, None, off, kind, t, pw)
        _assert_close(*got, R.loss_rows(x, y, None, off, kind, t, pw, grad_mean=0.7))
    # every row alone gives its row loss bit for bit, and the whole set repeats bit for bit
    from beat_this_b200 import loss as L

    xd, yd, md = (torch.from_numpy(a).to(DEV) for a in (x, y, m))
    rows, mean = L.beat_loss_rows(xd, yd, md, off, kind, t, pw)
    for i in range(0, len(off) - 1, 7):
        one, _ = L.beat_loss_rows(xd[off[i] : off[i + 1]], yd[off[i] : off[i + 1]], md[off[i] : off[i + 1]],
                                  [0, off[i + 1] - off[i]], kind, t, pw)
        assert torch.equal(one[0], rows[i])
    rows2, mean2 = L.beat_loss_rows(xd, yd, md, off, kind, t, pw)
    assert torch.equal(rows, rows2) and torch.equal(mean, mean2)
    assert np.array_equal(_kernel(x, y, m, off, kind, t, pw)[2], _kernel(x, y, m, off, kind, t, pw)[2])


@pytest.mark.parametrize("k", CASES)
def test_modules_against_reference_fixture(lib_built, k):
    from beat_this_b200 import loss as L

    kind, t, pw, has_mask = GOLD[f"spec{k}"]
    kind, t = int(kind), int(t)
    cls = (L.MaskedBCELoss, L.ShiftTolerantBCELoss, L.SplittedShiftTolerantBCELoss)[kind]
    module = cls(pos_weight=float(pw)) if kind == 0 else cls(pos_weight=float(pw), tolerance=t)
    x = torch.tensor(GOLD[f"preds{k}"], device=DEV, requires_grad=True)
    y = torch.tensor(GOLD[f"targets{k}"], device=DEV)
    mask = torch.tensor(GOLD[f"mask{k}"], device=DEV) if has_mask else None  # bool, float or [B, 1] as stored
    loss = module(x, y, mask)
    assert loss.shape == () and loss.dtype == torch.float32 and loss.is_cuda
    loss.backward()
    want, grad = float(GOLD[f"loss{k}"]), GOLD[f"grad{k}"]
    assert abs(loss.item() - want) <= 1e-6 * abs(want)
    g = x.grad.cpu().numpy()
    assert np.max(np.abs(g - grad)) <= GRAD_TOL * np.max(np.abs(grad))
    assert np.array_equal(g != 0, grad != 0)
    *_, rl, rg = fixture_case(k)
    assert rl == want and np.array_equal(rg, grad.ravel())


def test_errors_before_any_launch_and_weightless_ctx(lib_built):
    from beat_this_b200 import _lib
    from beat_this_b200.engine import Engine

    eng = Engine(None, None, DEV)  # no parameters at all
    buf = torch.zeros(64, device=eng.device)
    tgt = torch.zeros(64, device=eng.device)
    grad = torch.zeros(64, device=eng.device)
    rows = torch.zeros(4, dtype=torch.float64, device=eng.device)
    mean = torch.zeros((), device=eng.device)
    one = torch.ones((), device=eng.device)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    N = ctypes.c_void_p(None)

    def fwd(off, kind=1, t=3, pw=1.0, x=P(buf), m=P(buf), out=P(mean)):
        p = _lib.bt_loss_params(kind, t, pw)
        return eng.lib.bt_beat_loss(eng.ctx, x, P(tgt), m, _lib.i64_array(off), len(off) - 1, ctypes.byref(p), P(rows),
                                    out, None)

    def bwd(off, kind=1, t=3, pw=1.0, m=P(buf), g=P(one)):
        p = _lib.bt_loss_params(kind, t, pw)
        return eng.lib.bt_beat_loss_backward(eng.ctx, P(buf), P(tgt), m, _lib.i64_array(off), len(off) - 1,
                                             ctypes.byref(p), g, P(grad), None)

    before = eng.launches
    bad = [dict(off=[0, 13], kind=3), dict(off=[0, 13], kind=-1), dict(off=[0, 13], t=-1),
           dict(off=[0, 300], t=65), dict(off=[0, 13], pw=float("nan")), dict(off=[0, 13], pw=float("inf")),
           dict(off=[0, 12]), dict(off=[0, 13, 20]), dict(off=[0, 13, 12]), dict(off=[1, 14]), dict(off=[0]),
           dict(off=[0, 13], m=N, kind=2), dict(off=[0, 0], kind=0)]
    for kw in bad:
        assert fwd(**kw) == -1, kw
        assert bwd(**kw) == -1, kw
    assert fwd([0, 13], x=N) == -1 and fwd([0, 13], out=N) == -1 and bwd([0, 13], g=N) == -1
    assert eng.launches == before
    assert eng.lib.bt_beat_loss(eng.ctx, P(buf), P(buf), N, None, 1, ctypes.byref(_lib.bt_loss_params(0, 0, 1.0)),
                                P(rows), P(mean), None) == -1
    assert eng.launches == before
    # later calls are unaffected: 2 launches forward, 1 backward
    x = torch.linspace(-3, 3, 64, device=eng.device)
    buf.copy_(x)
    tgt[::9] = 1
    assert fwd([0, 13, 64], kind=1, t=3, pw=2.0, m=N) == 0
    assert eng.launches == before + 2
    assert bwd([0, 13, 64], kind=1, t=3, pw=2.0, m=N) == 0
    assert eng.launches == before + 3
    torch.cuda.synchronize()
    want = R.loss_rows(x.cpu().numpy(), tgt.cpu().numpy(), None, [0, 13, 64], 1, 3, 2.0)
    assert np.allclose(rows[:2].cpu().numpy(), want[0], rtol=1e-6) and abs(mean.item() - want[1]) <= 1e-6 * abs(want[1])


# ---- evaluate(losses=True) -----------------------------------------------------------------------------------------
SECS = (30.0, 14.0, 9.0)


@pytest.fixture(scope="module")
def clips():
    from beat_this_b200 import synthetic

    return [synthetic.synth_clip(700 + i, s) for i, s in enumerate(SECS)]


def _annotate(ann, names, preds):
    """Shifted predictions as annotations; the second piece gets beats only (no downbeat annotations)."""
    from beat_this_b200.utils import save_beat_tsv

    for i, (name, (b, d)) in enumerate(zip(names, preds)):
        if i == 1:
            (ann / f"{name}.beats").write_text("".join(f"{v + 0.03}\n" for v in b))
        else:
            save_beat_tsv(b + 0.03, d + 0.03, ann / f"{name}.beats")


def _want_losses(module_pair, pieces, logits):
    from beat_this_b200 import loss as L
    from beat_this_b200.evaluate import framewise_truth

    out = {}
    for t, (target, module) in enumerate(zip(("beat", "downbeat"), module_pair)):
        kind, tol, pw = L.loss_spec(module)
        vals = []
        for p, lg in zip(pieces, logits):
            x = lg[t].cpu().numpy()
            y = framewise_truth(p.beats if t == 0 else p.downbeats, len(x))
            m = np.full(len(x), 1.0 if t == 0 or p.has_downbeats else 0.0, np.float32)
            vals.append(R.loss_rows(x, y, m, [0, len(x)], kind, tol, pw)[1])
        out[f"test_loss_{target}"] = np.asarray(vals)
    out["test_loss"] = out["test_loss_beat"] + out["test_loss_downbeat"]
    return out


def _check(E, runner, pieces, logits):
    from beat_this_b200.loss import loss_from_hparams

    plain = E.evaluate(runner, pieces, min_beat_time=5.0)
    res = E.evaluate(runner, pieces, min_beat_time=5.0, losses=True)
    for a, b in zip(plain.predictions, res.predictions):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    for k, v in plain.metrics.items():
        assert np.array_equal(res.metrics[k], v), k
    assert list(res.summary)[: len(plain.summary)] == list(plain.summary)
    assert [res.summary[k] for k in plain.summary] == list(plain.summary.values())
    want = _want_losses(loss_from_hparams(runner.model.checkpoint_hparams), pieces, logits)
    for k in E.LOSS_KEYS:
        assert np.all(np.abs(res.metrics[k] - want[k]) <= 1e-6 * np.abs(want[k])), (k, res.metrics[k], want[k])
        assert res.summary[k] == float(np.mean(res.metrics[k]))
    assert res.metrics["test_loss_downbeat"][1] == 0.0  # no downbeat annotations: masked out
    assert np.all(res.metrics["test_loss_beat"] > 0)
    return res


@pytest.mark.parametrize("float16", [False, True])
def test_evaluate_losses(small0_ckpt, clips, tmp_path, capsys, float16):
    from scipy.io import wavfile

    from beat_this_b200 import evaluate as E

    runner = E.make_runner(small0_ckpt, DEV, float16)
    # audio files
    (tmp_path / "wav").mkdir()
    paths = []
    for i, x in enumerate(clips):
        paths.append(tmp_path / "wav" / f"c{i}.wav")
        wavfile.write(paths[-1], 22050, np.round(x * 32767).astype(np.int16))
    ann = tmp_path / "ann"
    ann.mkdir()
    names = [p.stem for p in paths]
    _annotate(ann, names, runner.batch(paths))
    pieces = E.discover_audio([tmp_path / "wav"], ann)
    _check(E, runner, pieces, runner.frames_batch(paths))
    # stored spectrograms
    spects = [runner.signal2spect(x, 22050).cpu().numpy().astype(np.float16) for x in clips]
    sdir = tmp_path / "data" / "audio" / "spectrograms"
    sdir.mkdir(parents=True)
    np.savez(sdir / "ds.npz", **{f"c{i}/track": s for i, s in enumerate(spects)})
    sp_ann = tmp_path / "data" / "annotations" / "ds" / "annotations" / "beats"
    sp_ann.mkdir(parents=True)
    logits = runner.spects2frames([s.astype(np.float32) for s in spects])
    _annotate(sp_ann, names, [runner.frames2beats(b, d) for b, d in logits])
    pieces = E.discover_data(tmp_path / "data")
    res = _check(E, runner, pieces, logits)
    # the command line prints what the API returns
    capsys.readouterr()
    E._print_single(res)
    api = capsys.readouterr().out
    flags = ["--float16" if float16 else "--no-float16", "--no-dbn", "--losses"]
    assert E.main(["--models", small0_ckpt, "--data", str(tmp_path / "data"), "--eval-trim-beats", "5", *flags]) == 0
    cli = capsys.readouterr().out.splitlines()
    assert cli[0] == f"Single model prediction for {small0_ckpt}" and "\n".join(cli[1:]) + "\n" == api
    assert any(line.startswith("test_loss: ") for line in cli)


@pytest.mark.parametrize("loss_type", ["splitted_shift_tolerant_weighted_bce", "weighted_bce"])
def test_evaluate_losses_of_other_loss_types(small0_ckpt, clips, loss_type):
    from beat_this_b200 import evaluate as E
    from beat_this_b200.inference import load_checkpoint

    ckpt = load_checkpoint(small0_ckpt, "cpu")
    ckpt["hyper_parameters"] = dict(ckpt["hyper_parameters"], loss_type=loss_type, pos_weights={"beat": 5, "downbeat": 20})
    runner = E.make_runner(ckpt, DEV, False)
    spects = [runner.signal2spect(x, 22050).cpu().numpy() for x in clips]
    logits = runner.spects2frames(spects)
    preds = [runner.frames2beats(b, d) for b, d in logits]
    pieces = [E.Piece(f"p{i}", b + 0.02, d, i != 1, spect=s) for i, (s, (b, d)) in enumerate(zip(spects, preds))]
    _check(E, runner, pieces, logits)
