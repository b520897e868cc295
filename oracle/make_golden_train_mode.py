"""Generate tests/golden/train_mode.npz by running the UNMODIFIED reference's BeatThis (beat_this/model/beat_tracker.py)
in train() mode and float64 under its training loss pair, as oracle/make_golden_train_grads.py does in eval mode.

    python oracle/make_golden_train_mode.py <beat_this source tree>      (or BEAT_THIS_REFERENCE=<tree>)

torch's own dropout streams are neither specified nor stable, so every nn.Dropout and every Attend of the reference
model is patched to apply the library's counter-based mask for its site (oracle/philox.py and the numbering of
include/beatthis.h), permuted into the reference's tensor layout; the rate of each site is the module's own (the
reference's dropout["frontend"] / dropout["transformer"] placement), and a module applies it only in training mode,
as the reference does.  BatchNorm is the reference's own nn.BatchNorm1d / 2d in training mode.  Per case k the fixture
holds what train_grads.npz holds (inputs, logits, loss, gradients at the logits, dspect, one fingerprint row per
trainable entry) and the dropout seed (mode_seed{k}), the rates (rates{k}), the running statistics after the call
(running{k}, in the order of running_names{k}) and num_batches_tracked (tracked{k}).  The script also checks that
tests/train_mode_reference.py (the float64 restatement the GPU tests use) gives the same logits and gradients.
"""
from __future__ import annotations

import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("BEAT_THIS_REFERENCE")
if not REF:
    sys.exit("usage: python oracle/make_golden_train_mode.py <beat_this source tree>")
sys.path.insert(0, os.path.join(HERE, "shims"))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from beat_this.model import roformer  # noqa: E402  (the reference)
from beat_this.model.beat_tracker import BeatThis  # noqa: E402  (the reference)
from beat_this.model.loss import ShiftTolerantBCELoss  # noqa: E402  (the reference)
from beat_this_b200 import synthetic  # noqa: E402
from oracle import beat_this_oracle as O  # noqa: E402
from oracle import philox  # noqa: E402
from oracle.train_fingerprint import fingerprint  # noqa: E402

# family, checkpoint seed, frames per item (zero-padded to the longest), downbeat annotations per item, dropout seed,
# dropout rates (frontend, transformer)
CASES = [
    ("small0", 0, (40, 31, 20), (1, 1, 0), 0x5EED0001, (0.1, 0.2)),
    ("small0-nosum", 1, (33, 33), (1, 1), 2 ** 63 + 12345, (0.5, 0.9)),
    ("small0-nopartial", 2, (33, 25), (1, 1), 77, (0.1, 0.2)),
    ("final0", 3, (48, 30), (0, 1), 2 ** 40 + 3, (0.1, 0.2)),
]
MODEL_ARGS = ("spect_dim", "transformer_dim", "ff_mult", "n_layers", "head_dim", "stem_dim", "sum_head",
              "partial_transformers")


def steps(hp: dict) -> list[str]:
    """The model's layer list as include/beatthis.h numbers it (dropout site 2 s + k of step s), by module name."""
    out = ["frontend.stem"]
    for i in range(3):
        p = f"frontend.blocks.{i}"
        if hp["partial_transformers"]:
            out += [p + ".partial.attnF", p + ".partial.ffF", p + ".partial.attnT", p + ".partial.ffT"]
        out.append(p)
    out.append("frontend.linear")
    for layer in range(hp["n_layers"]):
        out += [f"transformer_blocks.layers.{layer}.0", f"transformer_blocks.layers.{layer}.1"]
    return out + ["head"]


def patch(model, hp, seed, B, L):
    """Give every nn.Dropout and Attend of `model` the library's mask of its site."""
    index = {name: s for s, name in enumerate(steps(hp))}

    def to_reference(m, name):
        """a mask of the library's token rows [rows, N] into the layout of the tensor the module sees"""
        if ".attnF" in name or ".ffF" in name:  # "(b t) f c": library rows ((b F + f) L + t)
            Fq = m.shape[0] // (B * L)
            return m.view(B, Fq, L, -1).permute(0, 2, 1, 3).reshape(B * L, Fq, -1)
        return m  # "(b f) t c" and the main blocks' "b t d" are the library's row order

    for name, mod in model.named_modules():
        if isinstance(mod, torch.nn.Dropout):
            owner, k = name.rsplit(".", 2)[0], {"to_out.1": 1, "net.3": 0, "net.5": 1}[".".join(name.split(".")[-2:])]
            site = 2 * index[owner] + k

            def drop(x, mod=mod, site=site, name=name):
                if not mod.training or philox.threshold(mod.p) == 0:
                    return x
                keep = philox.keep(seed, site, mod.p, x.numel())
                m = torch.from_numpy(keep.astype(np.float64) * philox.scale(mod.p)).view(-1, x.shape[-1])
                return x * to_reference(m, name).reshape(x.shape).to(x.dtype)

            mod.forward = drop
        elif isinstance(mod, roformer.Attend):
            site = 2 * index[name.rsplit(".", 1)[0]]

            def attend(q, k, v, mod=mod, site=site):
                p = mod.dropout if mod.training else 0.0
                P = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(q.shape[-1]), dim=-1)  # [S, h, n, n]
                if philox.threshold(p):
                    keep = philox.keep(seed, site, p, P.numel())
                    P = P * torch.from_numpy(keep.astype(np.float64) * philox.scale(p)).view(P.shape).to(P.dtype)
                return P @ v

            assert mod.scale is None  # the reference's attentions use the default scale
            mod.forward = attend


def main():
    import train_mode_reference as TM

    out = {}
    for k, (family, seed, lengths, has_down, mode_seed, rates) in enumerate(CASES):
        ckpt = synthetic.make_checkpoint(family, seed)
        hp = dict(ckpt["hyper_parameters"])
        sd = O.strip_prefix(ckpt["state_dict"])
        dropout = {"frontend": rates[0], "transformer": rates[1]}
        model = BeatThis(**{a: hp[a] for a in MODEL_ARGS}, dropout=dropout).double().train()
        model.load_state_dict(sd)
        rng = np.random.default_rng(200 + k)
        B, L = len(lengths), max(lengths)
        patch(model, hp, mode_seed, B, L)
        spect = (rng.random((B, L, 128)) * 4).astype(np.float32)
        pad = np.zeros((B, L), np.float32)
        for b, n in enumerate(lengths):
            spect[b, n:] = 0
            pad[b, :n] = 1
        beat = (rng.random((B, L)) < 0.12).astype(np.float32) * pad
        down = beat * (rng.random((B, L)) < 0.3)
        dmask = np.asarray(has_down, np.float32)

        x = torch.tensor(spect, dtype=torch.float64, requires_grad=True)
        pred = model(x)
        lb, ld = (pred[t].detach().requires_grad_(True) for t in ("beat", "downbeat"))
        pw = hp["pos_weights"]
        mask = torch.tensor(pad, dtype=torch.float64)
        loss = ShiftTolerantBCELoss(pos_weight=pw["beat"])(lb, torch.tensor(beat, dtype=lb.dtype), mask)
        loss = loss + ShiftTolerantBCELoss(pos_weight=pw["downbeat"])(
            ld, torch.tensor(down, dtype=ld.dtype), mask * torch.tensor(dmask, dtype=torch.float64)[:, None])
        loss.backward()
        torch.autograd.backward((pred["beat"], pred["downbeat"]), (lb.grad, ld.grad))

        named = dict(model.named_parameters())
        names = [n for n in model.state_dict() if n in named and named[n].requires_grad]
        grads = {n: named[n].grad for n in names}
        # the restatement the GPU tests use, on the checkpoint's weights and the same gradients at the logits
        sd64 = {n: v.detach().double().requires_grad_(n in grads) if v.is_floating_point() else v
                for n, v in sd.items()}
        x64 = torch.tensor(spect, dtype=torch.float64, requires_grad=True)
        ob, od, _ = TM.forward_train(sd64, x64, mode_seed, *rates, sum_head=hp["sum_head"])
        og = torch.autograd.grad((ob, od), [x64] + [sd64[n] for n in names], (lb.grad.double(), ld.grad.double()))
        # the two differ in the rounding of the fp32 RoPE angles and the sum head's fp32 cast (below 1e-6 in eval
        # mode, make_golden_train_grads.py); a rate of 0.9 scales kept values by 10, so the check allows 1e-5
        worst = 0.0
        for n, g in zip(["spect"] + names, og):
            ref = x.grad if n == "spect" else grads[n]
            err = float((g - ref).norm() / ref.norm())
            worst = max(worst, err)
            assert err < 1e-5, f"{family}: the restatement's gradient of {n} differs by {err:.2e}"
        assert torch.allclose(ob, pred["beat"].detach().double(), atol=1e-5)
        assert torch.allclose(od, pred["downbeat"].detach(), atol=1e-5)

        after = model.state_dict()
        running = [n for n in after if n.endswith((".running_mean", ".running_var"))]
        tracked = [n for n in after if n.endswith(".num_batches_tracked")]
        index = {n: i for i, n in enumerate(sd)}
        out.update({
            f"family{k}": np.array(family), f"seed{k}": np.array(seed), f"spect{k}": spect,
            f"truth_beat{k}": beat, f"truth_downbeat{k}": down, f"padding_mask{k}": pad, f"downbeat_mask{k}": dmask,
            f"mode_seed{k}": np.array(mode_seed, dtype=np.uint64), f"rates{k}": np.array(rates),
            f"beat{k}": pred["beat"].detach().double().numpy(), f"downbeat{k}": pred["downbeat"].detach().numpy(),
            f"loss{k}": np.array(loss.item()), f"dbeat{k}": lb.grad.double().numpy(),
            f"ddown{k}": ld.grad.double().numpy(), f"dspect{k}": x.grad.numpy(), f"names{k}": np.array(names),
            f"fp{k}": np.stack([fingerprint(grads[n].numpy(), index[n]) for n in names]),
            f"running_names{k}": np.array(running),
            f"running{k}": np.concatenate([after[n].numpy().reshape(-1) for n in running]),
            f"tracked{k}": np.array([int(after[n]) for n in tracked]),
        })
        print(f"{family}: B={B} L={L} rates {rates} loss {loss.item():.6f}, {len(names)} gradients, restatement agrees within {worst:.1e}")
    path = os.path.join(ROOT, "tests", "golden", "train_mode.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
