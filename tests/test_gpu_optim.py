"""bt_adamw_step (csrc/kernels_optim.cu) and beat_this_b200.optim on the GPU:
* the kernel against its float64 restatement within the derived elementwise bound (tests/optim_reference.py), over
  entries of 0 .. 4097 and more elements, aligned and offset by one float (the scalar path), with and without decay,
  at steps 1, 2, 10^3 and 10^6, in one table; lr 0 leaves the parameters bitwise unchanged; sentinels past every end
  and a NULL-grad entry stay untouched; two calls write the same bytes; one call is one "adamw" launch; every refusal
  launches and profiles nothing;
* optim.AdamW against torch.optim.AdamW(foreach=True) over 100 steps on small0's parameter shapes, with state dicts
  crossing both ways at step 50;
* the reference's fixture (tests/golden/optim.npz): groups, hyperparameters, state after K steps, state_dict
  skeletons."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch

import optim_reference as R
from beat_this_b200 import _lib, synthetic
from beat_this_b200.engine import Engine
from beat_this_b200.optim import AdamW, CosineWarmupScheduler, param_groups
from beat_this_b200.train import BeatThisModule
from conftest import GOLDEN
from oracle.state_skeleton import skeleton
from oracle.train_fingerprint import bounds, fingerprint

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAD = 9
SENTINEL = 4321.0


@pytest.fixture(scope="module")
def eng(lib_built):
    return Engine.shared(DEV)


class Case:
    """One table entry: four device buffers with the entry's n elements at `offset` floats, sentinels around them."""

    def __init__(self, n, offset, seed, null_grad=False, **hp):
        g = torch.Generator().manual_seed(seed)
        self.n, self.offset, self.hp, self.null_grad = n, offset, hp, null_grad
        vals = [torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.1, torch.randn(n, generator=g) * 0.01,
                torch.rand(n, generator=g) * 1e-3]
        self.bufs = []
        for v in vals:
            b = torch.full((offset + n + PAD,), SENTINEL)
            b[offset : offset + n] = v
            self.bufs.append(b.to(DEV))
        self.host = [v.double().numpy() for v in vals]  # p, g, m, v

    def views(self):
        return [b[self.offset : self.offset + self.n] for b in self.bufs]

    def entry(self):
        p, g, m, v = (b.data_ptr() + 4 * self.offset for b in self.bufs)
        h = self.hp
        return _lib.bt_adamw_entry(p, None if self.null_grad else g, m, v, self.n, h["lr"], h["beta1"], h["beta2"],
                                   h["eps"], h["weight_decay"], h["step"])


def _cases():
    cases, seed = [], 0
    for n in (0, 1, 3, 4, 5, 4097, 3 * 4096 + 7):
        for offset in (0, 1):
            for wd, step in ((0.01, 1), (0.0, 2), (0.05, 1000), (0.01, 10 ** 6)):
                seed += 1
                cases.append(Case(n, offset, seed, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=wd,
                                  step=step))
    cases.append(Case(300, 0, 999, lr=0.1, beta1=0.3, beta2=0.5, eps=1e-6, weight_decay=0.1, step=3))  # lerp's 2nd form
    return cases


def _launches(eng):
    return int(eng.lib.bt_launch_count(eng.ctx))


def test_kernel_against_the_restatement(eng):
    cases = _cases() + [Case(64, 0, 5000, null_grad=True, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8,
                             weight_decay=0.01, step=1)]
    before = [[b.clone() for b in c.bufs] for c in cases]
    eng.profile_enable(True)
    eng.profile_reset()
    n0 = _launches(eng)
    eng.adamw_step([c.entry() for c in cases])
    torch.cuda.synchronize()
    assert _launches(eng) == n0 + 1
    prof = eng.profile_results()
    eng.profile_enable(False)
    assert {k: n for k, (_, n) in prof.items() if n} == {"adamw": 1}, prof
    worst = 0.0
    for c, b0 in zip(cases, before):
        for b, old in zip(c.bufs, b0):  # sentinels
            assert torch.equal(b[: c.offset], old[: c.offset]) and torch.equal(b[c.offset + c.n :], old[c.offset + c.n :])
        if c.null_grad or c.n == 0:
            assert all(torch.equal(b, old) for b, old in zip(c.bufs, b0))
            continue
        want, bound = R.adamw(*c.host, **c.hp)
        p, g, m, v = (t.cpu().double().numpy() for t in c.views())
        assert np.array_equal(g, c.host[1])
        for got, w, e in zip((p, m, v), want, bound):
            err = np.abs(got - w)
            assert (err <= e).all(), (c.n, c.offset, c.hp, float((err / e).max()))
            worst = max(worst, float((err / e).max()))
    print(f"\nworst error / bound: {worst:.3f}")

    # the same inputs again: the same bytes
    again = [[b.clone() for b in c.bufs] for c in cases]
    for c, b0 in zip(cases, before):
        for b, old in zip(c.bufs, b0):
            b.copy_(old)
    eng.adamw_step([c.entry() for c in cases])
    torch.cuda.synchronize()
    for c, a in zip(cases, again):
        assert all(torch.equal(b, x) for b, x in zip(c.bufs, a))


def test_zero_learning_rate_keeps_the_parameters(eng):
    cases = [Case(n, off, 77 + n, lr=0.0, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, step=5)
             for n in (5, 4097) for off in (0, 1)]
    p0 = [c.bufs[0].clone() for c in cases]
    eng.adamw_step([c.entry() for c in cases])
    torch.cuda.synchronize()
    for c, p in zip(cases, p0):
        assert torch.equal(c.bufs[0], p)


def test_refusals_launch_nothing(eng):
    lib, ctx = eng.lib, eng.ctx
    ok = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, step=1)
    base = Case(16, 0, 3, **ok)
    bad = {"numel": dict(numel=-1), "nan lr": dict(lr=math.nan), "inf eps": dict(eps=math.inf),
           "nan wd": dict(weight_decay=math.nan), "lr": dict(lr=-1e-3), "eps": dict(eps=-1.0),
           "beta1": dict(beta1=1.0), "beta2": dict(beta2=-0.1), "step": dict(step=0), "param": dict(param=None),
           "exp_avg": dict(exp_avg=None), "exp_avg_sq": dict(exp_avg_sq=None)}
    eng.profile_enable(True)
    eng.profile_reset()
    n0 = _launches(eng)
    b0 = [b.clone() for b in base.bufs]
    for name, change in bad.items():
        good, e = base.entry(), base.entry()
        for k, v in change.items():
            setattr(e, k, v)
        table = (_lib.bt_adamw_entry * 2)(good, e)
        assert lib.bt_adamw_step(ctx, table, 2, None) == -1, name  # BT_ERR_ARG
        assert b"bt_adamw_step" in lib.bt_last_error(ctx), name
    assert lib.bt_adamw_step(ctx, (_lib.bt_adamw_entry * 1)(base.entry()), -1, None) == -1
    assert lib.bt_adamw_step(ctx, None, 1, None) == -1
    torch.cuda.synchronize()
    assert _launches(eng) == n0
    assert all(n == 0 for _, n in eng.profile_results().values())
    assert all(torch.equal(b, x) for b, x in zip(base.bufs, b0))
    assert lib.bt_adamw_step(ctx, (_lib.bt_adamw_entry * 1)(base.entry()), 1, None) == 0
    torch.cuda.synchronize()
    assert _launches(eng) == n0 + 1
    eng.profile_enable(False)


def _ulps(a, b):
    """Worst difference in units of the last place over the elements of b of at least 1 % of its rms: values near
    zero, where a tiny difference is many ulps, are left to the normwise bound."""
    keep = b.abs() >= 0.01 * b.pow(2).mean().sqrt()
    a, b = a[keep], b[keep]
    ia, ib = (t.view(torch.int32).long() for t in (a, b))
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max().item()) if a.numel() else 0


def _shapes():
    return [shape for _, shape, trainable in _lib.train_param_table(synthetic.model_hparams("small0")) if trainable]


def _pair(params, opt_cls, **kw):
    groups = [{"params": [p for p in params if p.ndim >= 2], "weight_decay": 0.01},
              {"params": [p for p in params if p.ndim <= 1], "weight_decay": 0}]
    return opt_cls(groups, lr=1e-3, **kw)


def test_against_torch_foreach(eng):
    g = torch.Generator().manual_seed(5)
    init = [torch.randn(s, generator=g) * 0.1 for s in _shapes()]
    ours = [torch.nn.Parameter(t.to(DEV)) for t in init]
    ref = [torch.nn.Parameter(t.to(DEV)) for t in init]
    opt_a, opt_b = _pair(ours, AdamW), _pair(ref, torch.optim.AdamW, foreach=True)
    worst_ulp, bitwise, worst_rel = 0, True, 0.0
    for step in range(100):
        if step == 50:  # state dicts cross both ways
            sa, sb = opt_a.state_dict(), opt_b.state_dict()
            opt_a, opt_b = _pair(ours, AdamW), _pair(ref, torch.optim.AdamW, foreach=True)
            opt_a.load_state_dict(sb)
            opt_b.load_state_dict(sa)
        for a, b in zip(ours, ref):
            grad = (torch.randn(a.shape, generator=g) * 0.01).to(DEV)
            a.grad, b.grad = grad.clone(), grad.clone()
        opt_a.step()
        opt_b.step()
        for a, b in zip(ours, ref):
            sa, sb = opt_a.state[a], opt_b.state[b]
            assert sa["step"].dtype == torch.float32 and not sa["step"].is_cuda and float(sa["step"]) == step + 1
            for x, y in ((a.detach(), b.detach()), (sa["exp_avg"], sb["exp_avg"]), (sa["exp_avg_sq"], sb["exp_avg_sq"])):
                rel = float((x - y).norm() / max(y.norm(), 1e-30))
                worst_rel = max(worst_rel, rel)
                assert rel <= 1e-6, (step, tuple(a.shape), rel)
                bitwise &= torch.equal(x, y)
            worst_ulp = max(worst_ulp, _ulps(a.detach(), b.detach()))  # the moments cross zero, where ulps mislead
    print(f"\nworst normwise relative difference {worst_rel:.2e}, worst parameter difference {worst_ulp} ulp, "
          f"bitwise: {bitwise}")


def test_refused_in_python_before_a_launch(eng):
    n0 = _launches(eng)
    cpu = torch.nn.Parameter(torch.zeros(4))
    cpu.grad = torch.zeros(4)
    half = torch.nn.Parameter(torch.zeros(4, device=DEV, dtype=torch.float16))
    half.grad = torch.zeros_like(half)
    strided = torch.nn.Parameter(torch.zeros(4, 4, device=DEV).t())
    strided.grad = torch.zeros(4, 4, device=DEV).t()
    sparse = torch.nn.Parameter(torch.zeros(4, device=DEV))
    sparse.grad = torch.zeros(4, device=DEV).to_sparse()
    for p in (cpu, half, strided, sparse):
        with pytest.raises(RuntimeError):
            AdamW([p]).step()
    good = torch.nn.Parameter(torch.zeros(4, device=DEV))
    good.grad = torch.ones(4, device=DEV)
    opt = AdamW([good])
    sd = opt.state_dict()
    sd["param_groups"][0]["amsgrad"] = True
    opt.load_state_dict(sd)
    with pytest.raises(ValueError):
        opt.step()
    assert _launches(eng) == n0


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "optim.npz"))


def test_reference_fixture(eng, gold):
    hp = {"transformer_dim": 64, "n_layers": 1}
    groups = json.loads(str(gold["groups"]))
    module = BeatThisModule(hp, DEV)
    name_of = {id(p): n for n, p in module.named_parameters()}
    opt = AdamW(param_groups(module, 0.01), lr=0.0008)
    CosineWarmupScheduler(opt, 1000, 100)
    for got, want in zip(opt.param_groups, groups):
        assert [name_of[id(p)] for p in got["params"]] == [n.removeprefix("model.") for n in want["names"]]
        assert json.loads(json.dumps({k: v for k, v in got.items() if k != "params"})) == want["hparams"]

    K, warmup = (int(x) for x in gold["steps"])
    lr, wd, pscale, gscale = (float(x) for x in gold["step_hparams"])
    module = BeatThisModule(hp, DEV)
    named = dict(module.named_parameters())
    trainable = [n.removeprefix("model.") for n in gold["trainable"]]
    g = torch.Generator().manual_seed(int(gold["seed"]))
    with torch.no_grad():
        for n in trainable:
            named[n].copy_(torch.randn(named[n].shape, generator=g) * pscale)
    opt = AdamW(param_groups(module, wd), lr=lr)
    sched = CosineWarmupScheduler(opt, warmup, K)
    for _ in range(K):
        for n in trainable:
            named[n].grad = (torch.randn(named[n].shape, generator=g) * gscale).to(DEV)
        opt.step()
        sched.step()
    assert opt.param_groups[0]["lr"] == float(gold["final_lr"])
    for key in ("param", "exp_avg", "exp_avg_sq"):
        for i, n in enumerate(trainable):
            t = named[n] if key == "param" else opt.state[named[n]][key]
            got = fingerprint(t.detach().cpu().numpy(), i)
            want = gold[f"fp_{key}"][i]
            assert (np.abs(got - want) <= bounds(want, t.numel(), i, 1e-5)).all(), (key, n)
    assert json.loads(json.dumps(skeleton(opt.state_dict()))) == json.loads(str(gold["opt_skeleton"]))
    assert json.loads(json.dumps(skeleton(sched.state_dict()))) == json.loads(str(gold["sched_skeleton"]))
