"""bt_train_forward / bt_train_backward and BeatThisModule against float64 autograd through the oracle restatement of
the reference's BeatThis in eval mode."""
import ctypes
import os

import numpy as np
import pytest
import torch

from beat_this_b200 import _lib, synthetic
from beat_this_b200.engine import Engine
from beat_this_b200.loss import ShiftTolerantBCELoss
from beat_this_b200.train import BeatThisModule
from oracle import beat_this_oracle as O
from support import DEV, GRAD_BOUND, LOGIT_TOL, _module, _rel, _spect

pytestmark = pytest.mark.gpu


def _oracle(module, x, dbeat, ddown, sum_head):
    """float64 logits and gradients (spect first, then every trainable entry by name) of the eval-mode reference."""
    sd = {k: (v.detach().cpu().double().requires_grad_(v.requires_grad) if v.is_floating_point() else v.cpu())
          for k, v in module.state_dict(keep_vars=True).items()}
    x64 = x.double().requires_grad_(True)
    beat, down = O.forward(sd, x64, sum_head=sum_head)
    names = [k for k, v in sd.items() if v.is_floating_point() and v.requires_grad]
    grads = torch.autograd.grad((beat, down), [x64] + [sd[k] for k in names], (dbeat.double(), ddown.double()))
    return beat.detach(), down.detach(), grads[0], dict(zip(names, grads[1:]))


CASES = [  # family, B, L, lengths of a zero-padded batch (None: dense), hyper-parameter overrides
    ("small0", 1, 1, None, {}),
    ("small0", 3, 17, None, {}),
    ("small0", 8, 17, None, {}),
    ("small0-nosum", 3, 17, None, {}),
    ("small0-nopartial", 3, 17, None, {}),
    ("64", 1, 1500, None, {}),
    ("1024", 3, 17, None, {"ff_mult": 2}),   # 32 heads, the widest model bt_create takes
    ("1024", 1, 40, None, {}),               # FFN hidden of 4096, the widest scratch row
    ("small0", 2, 1700, None, {}),
    ("small0", 3, 400, (400, 251, 90), {}),
    ("final0", 8, 1500, None, {}),           # the reference's training batch: dW sums 12 000 rows
]


@pytest.mark.parametrize("family,B,L,lengths,overrides", CASES)
def test_gradients_match_float64_autograd(family, B, L, lengths, overrides):
    module, _ = _module(family, **overrides)
    sum_head = synthetic.model_hparams(family)["sum_head"]
    x = _spect(B, L, 1, lengths)
    xs = x.to(DEV).requires_grad_(True)
    out = module(xs)
    if lengths is None:
        g = torch.Generator().manual_seed(2)
        dbeat, ddown = torch.randn(B, L, generator=g), torch.randn(B, L, generator=g)
        (out["beat"] * dbeat.to(DEV)).sum().backward(retain_graph=True)
        (out["downbeat"] * ddown.to(DEV)).sum().backward()
    else:  # the reference's loss pair with its padding mask
        mask = torch.zeros(B, L, device=DEV)
        for b, n in enumerate(lengths):
            mask[b, :n] = 1
        targets = (torch.rand(B, L, generator=torch.Generator().manual_seed(3)) < 0.1).float().to(DEV)
        beat, down = out["beat"], out["downbeat"]
        beat.retain_grad(), down.retain_grad()
        loss = ShiftTolerantBCELoss()(beat, targets, mask) + ShiftTolerantBCELoss()(down, targets * 0.5, mask)
        loss.backward()
        dbeat, ddown = beat.grad.cpu(), down.grad.cpu()
    ob, od, gx, gp = _oracle(module, x, dbeat, ddown, sum_head)
    assert (out["beat"].detach().cpu().double() - ob).abs().max() < LOGIT_TOL
    assert (out["downbeat"].detach().cpu().double() - od).abs().max() < LOGIT_TOL
    errs = {"spect": _rel(xs.grad, gx)}
    params = dict(module.named_parameters())
    for name, ref in gp.items():
        errs[name] = _rel(params[name].grad, ref)
    worst = max(errs, key=errs.get)
    assert errs[worst] <= GRAD_BOUND, f"{worst}: {errs[worst]:.3e}"
    assert set(gp) == {n for n, p in params.items() if p.requires_grad}


def test_activation_store_matches_an_independent_count():
    hp = synthetic.model_hparams("small0")
    eng = Engine(None, hp, DEV)
    B, L = 2, 10  # B L and every per-step count a multiple of 4: no alignment padding
    BL, D = B * L, hp["transformer_dim"]

    def attn(C, M):
        return M * (C + C + 1 + 3 * C + 2 * (C // 32) + C)  # in, xn, inv, qkv, gate logits + lse, out

    def ffn(C, M, mult):
        return M * (2 * C + 1 + 2 * mult * C)  # in, xn, inv, pre-GELU, GELU

    n = BL * 128 + BL * 32 * 32  # stem: spectrogram copy, conv output
    C, F = 32, 32
    for _ in range(3):
        n += 2 * (attn(C, BL * F) + ffn(C, BL * F, 4)) + BL * F * C + BL * F * C  # partial transformer; conv in, out
        C, F = 2 * C, F // 2
    n += 2 * BL * C * F  # frontend.linear: its input tokens and the gathered rows
    n += hp["n_layers"] * (attn(D, BL) + ffn(D, BL, hp["ff_mult"])) + BL * (2 * D + 1)
    assert eng.train_activation_bytes(B, L) == 4 * n


def test_logits_match_the_fp32_inference_path():
    from beat_this_b200.inference import load_model

    module, ckpt = _module("small0", 4)
    x = _spect(3, 1500, 5).to(DEV)
    with torch.no_grad():
        out = module(x)
    ref = load_model(ckpt, DEV, float16=False)(x)
    for k in ("beat", "downbeat"):
        assert (out[k] - ref[k]).abs().max().item() < LOGIT_TOL


def test_backward_is_bitwise_repeatable():
    module, _ = _module("small0", 1)
    x = _spect(2, 300, 6).to(DEV)
    runs = []
    for _ in range(2):
        module.zero_grad(set_to_none=True)
        xs = x.clone().requires_grad_(True)
        out = module(xs)
        (out["beat"].square().sum() + out["downbeat"].sum()).backward()
        runs.append([xs.grad.clone()] + [p.grad.clone() for p in module.parameters() if p.grad is not None])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def test_refusals_before_anything_is_enqueued():
    hp = synthetic.model_hparams("small0")
    module, _ = _module("small0")
    eng = module.engine
    params = module._tables()
    B, L = 2, 10
    spect = torch.zeros(B, L, 128, device=DEV)
    beat, down = torch.zeros(B, L, device=DEV), torch.zeros(B, L, device=DEV)
    act = torch.empty(eng.train_activation_bytes(B, L), dtype=torch.uint8, device=DEV)
    lib = eng.lib
    ptrs = eng._table_ptrs(params, "parameter")
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    before = eng.launches
    # pointer count, a store one byte short, B < 1
    assert lib.bt_train_forward(eng.ctx, ptrs, len(params) - 1, p(spect), B, L, p(act), act.numel(), p(beat), p(down),
                                stream) == -1
    assert lib.bt_train_forward(eng.ctx, ptrs, len(params), p(spect), B, L, p(act), act.numel() - 1, p(beat), p(down),
                                stream) == -1
    assert lib.bt_train_forward(eng.ctx, ptrs, len(params), p(spect), 0, L, p(act), act.numel(), p(beat), p(down),
                                stream) == -1
    grads = eng._table_ptrs([None] * len(params), "gradient")
    assert lib.bt_train_backward(eng.ctx, ptrs, len(params), p(act), act.numel(), B, 2 * L, p(beat), p(down), grads,
                                 None, stream) == -1
    assert eng.launches == before
    # a 16-bit context
    half = Engine(None, hp, DEV, half=True)
    assert half.lib.bt_train_forward(half.ctx, ptrs, len(params), p(spect), B, L, p(act), act.numel(), p(beat),
                                     p(down), stream) == -1
    assert b"BT_DTYPE_F32" in lib.bt_last_error(half.ctx)
    assert _lib.train_param_table(hp) and lib.bt_train_activation_bytes(eng.ctx, 0, L) == -1


def test_adamw_steps_lower_the_loss_and_the_checkpoint_reloads(tmp_path):
    from beat_this_b200.inference import load_model

    module, _ = _module("small0", 7)
    assert not module.training
    with pytest.raises(NotImplementedError, match="dropout"):
        module.train()
    g = torch.Generator().manual_seed(8)
    B, L = 4, 256
    x = (torch.rand(B, L, 128, generator=g) * 4).to(DEV)
    beats = torch.zeros(B, L, device=DEV)
    beats[:, ::25] = 1
    downs = torch.zeros(B, L, device=DEV)
    downs[:, ::100] = 1
    mask = torch.ones(B, L, device=DEV)
    mask[1, 200:] = 0
    loss_b, loss_d = ShiftTolerantBCELoss(), ShiftTolerantBCELoss()
    opt = torch.optim.AdamW([p for p in module.parameters() if p.requires_grad], lr=1e-3)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        out = module(x)
        loss = loss_b(out["beat"], beats, mask) + loss_d(out["downbeat"], downs, mask)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.8 * losses[0], losses
    path = module.save_checkpoint(os.path.join(tmp_path, "trained.ckpt"))
    with torch.no_grad():
        out = module(x[:, :L])
    ref = load_model(path, DEV, float16=False)(x)
    for k in ("beat", "downbeat"):
        assert (out[k] - ref[k]).abs().max().item() < LOGIT_TOL
    again = BeatThisModule.from_checkpoint(path, DEV)
    assert all(torch.equal(a, b) for a, b in zip(module.state_dict().values(), again.state_dict().values()))
    assert np.isfinite(losses).all()


def test_fixture_fingerprints_are_reproduced():
    """Gradients of the unmodified reference's BeatThis (tests/golden/train_grads.npz, oracle/make_golden_train_grads.py)
    under its loss pair: logits, loss, the spectrogram's gradient and every parameter's fingerprint."""
    from oracle.train_fingerprint import bounds, fingerprint

    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "train_grads.npz"))
    k = 0
    while f"family{k}" in z:
        c = {name: z[f"{name}{k}"] for name in ("family", "seed", "spect", "beat", "downbeat", "dbeat", "ddown",
                                                  "dspect", "names", "fp", "loss", "truth_beat", "truth_downbeat",
                                                  "padding_mask", "downbeat_mask")}
        module, _ = _module(str(c["family"]), int(c["seed"]))
        x = torch.tensor(c["spect"], device=DEV, requires_grad=True)
        out = module(x)
        assert np.abs(out["beat"].detach().cpu().numpy() - c["beat"]).max() < LOGIT_TOL
        assert np.abs(out["downbeat"].detach().cpu().numpy() - c["downbeat"]).max() < LOGIT_TOL
        t = lambda a: torch.tensor(a, device=DEV, dtype=torch.float32)  # noqa: E731
        mask = t(c["padding_mask"])
        loss = ShiftTolerantBCELoss()(out["beat"], t(c["truth_beat"]), mask) + \
            ShiftTolerantBCELoss()(out["downbeat"], t(c["truth_downbeat"]), mask * t(c["downbeat_mask"])[:, None])
        assert abs(loss.item() - float(c["loss"])) <= 1e-3 * abs(float(c["loss"]))
        torch.autograd.backward((out["beat"], out["downbeat"]), (t(c["dbeat"]), t(c["ddown"])))
        ref = c["dspect"].astype(np.float64)
        assert np.linalg.norm(x.grad.cpu().numpy() - ref) <= GRAD_BOUND * np.linalg.norm(ref)
        params = dict(module.named_parameters())
        index = {n: i for i, n in enumerate(module.state_dict())}
        for name, fp in zip(c["names"], c["fp"]):
            name = str(name)
            g = params[name].grad.double().cpu().numpy()
            i = index[name]
            assert (np.abs(fingerprint(g, i) - fp) <= bounds(fp, g.size, i, GRAD_BOUND)).all(), name
        k += 1
    assert k == 4


def _attention_backward64(qkv, gates, freqs, dy):
    """float64 autograd of y = softmax(rope(q) rope(k)^T / sqrt 32) v * sigmoid(gates) per head."""
    seqs, n, C3 = qkv.shape
    heads = C3 // 96
    qkv = qkv.double().requires_grad_(True)
    g = gates.double().requires_grad_(True)
    q, k, v = qkv.view(seqs, n, 3, heads, 32).permute(2, 0, 3, 1, 4)
    q, k = O.rope(q, freqs), O.rope(k, freqs)
    p = torch.softmax(q @ k.transpose(-1, -2) / np.sqrt(32), dim=-1)
    y = ((p @ v) * torch.sigmoid(g).permute(0, 2, 1)[..., None]).permute(0, 2, 1, 3).reshape(seqs, n, heads * 32)
    y.backward(dy.double())
    return y.detach(), qkv.grad, g.grad


@pytest.mark.parametrize("n", [1, 7, 33, 1500])
@pytest.mark.parametrize("heads", [1, 16])
def test_attention_backward_hook_matches_float64(n, heads):
    eng = Engine(None, synthetic.model_hparams("small0"), DEV)
    seqs = 2 if n < 1500 else 1
    gen = torch.Generator().manual_seed(n * 100 + heads)
    qkv = torch.randn(seqs, n, 3 * heads * 32, generator=gen) * 0.6
    gates = torch.randn(seqs, n, heads, generator=gen)
    dy = torch.randn(seqs, n, heads * 32, generator=gen)
    freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
    before = eng.launches
    y, dqkv, dg = eng.debug_attention_backward(qkv.to(DEV), gates.to(DEV), freqs.to(DEV), dy.to(DEV))
    assert eng.launches - before == 7
    y64, dqkv64, dg64 = _attention_backward64(qkv, gates, freqs, dy)
    for got, ref in ((y, y64), (dqkv, dqkv64), (dg, dg64)):
        assert _rel(got, ref) <= GRAD_BOUND


def test_host_or_double_parameters_raise_before_any_launch():
    module, _ = _module("small0")
    x = _spect(1, 8, 9).to(DEV)
    before = module.engine.launches
    module.double()
    with pytest.raises(RuntimeError, match="float32"):
        module(x)
    module.float().cpu()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        module(x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        module.to(DEV)(x.cpu())
    assert module.engine.launches == before
    with torch.no_grad():
        module(x)  # back on the device it runs
