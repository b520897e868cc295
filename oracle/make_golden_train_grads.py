"""Generate tests/golden/train_grads.npz by running the UNMODIFIED reference's BeatThis (beat_this/model/beat_tracker.py)
in eval mode and float64 under its training loss pair (ShiftTolerantBCELoss on beat and downbeat, the padding mask and
the downbeat mask as PLBeatThis._compute_loss applies them, pl_module.py:99-113).

    python oracle/make_golden_train_grads.py <beat_this source tree>      (or BEAT_THIS_REFERENCE=<tree>)

rotary_embedding_torch comes from oracle/shims.  Cases: seeded synthetic checkpoints small0, small0-nosum,
small0-nopartial and final0, each on a zero-padded batch of random spectrograms with random beat targets.  Per case k
the fixture holds the inputs (spect{k}, truth_beat{k}, truth_downbeat{k}, padding_mask{k}, downbeat_mask{k}), the
reference's logits, loss and gradients at the logits (dbeat{k}, ddown{k}), the full gradient at the spectrogram
(dspect{k}) and one fingerprint row per trainable state_dict entry (fp{k}, oracle/train_fingerprint.py; names{k}).
The script also checks that oracle.beat_this_oracle.forward under float64 autograd gives the same gradients.
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("BEAT_THIS_REFERENCE")
if not REF:
    sys.exit("usage: python oracle/make_golden_train_grads.py <beat_this source tree>")
sys.path.insert(0, os.path.join(HERE, "shims"))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from beat_this.model.beat_tracker import BeatThis  # noqa: E402  (the reference)
from beat_this.model.loss import ShiftTolerantBCELoss  # noqa: E402  (the reference)
from beat_this_b200 import synthetic  # noqa: E402
from oracle import beat_this_oracle as O  # noqa: E402
from oracle.train_fingerprint import fingerprint  # noqa: E402

# family, checkpoint seed, frames per item (the batch is zero-padded to the longest), downbeat annotations per item
CASES = [
    ("small0", 0, (40, 31, 20), (1, 1, 0)),
    ("small0-nosum", 1, (33, 33), (1, 1)),
    ("small0-nopartial", 2, (33, 25), (1, 1)),
    ("final0", 3, (48, 30), (0, 1)),
]
MODEL_ARGS = ("spect_dim", "transformer_dim", "ff_mult", "n_layers", "head_dim", "stem_dim", "sum_head",
              "partial_transformers")


def main():
    out = {}
    for k, (family, seed, lengths, has_down) in enumerate(CASES):
        ckpt = synthetic.make_checkpoint(family, seed)
        hp = ckpt["hyper_parameters"]
        sd = O.strip_prefix(ckpt["state_dict"])
        model = BeatThis(**{a: hp[a] for a in MODEL_ARGS}).double().eval()
        model.load_state_dict(sd)
        rng = np.random.default_rng(100 + k)
        B, L = len(lengths), max(lengths)
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
        # the loss's own gradients at its two inputs (pred["downbeat"] also feeds the sum head's beat, so its .grad
        # after a plain backward would hold both paths)
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
        # the restatement under float64 autograd, on the same weights and gradients at the logits
        sd64 = {n: v.detach().double().requires_grad_(n in grads) for n, v in model.state_dict().items()}
        x64 = torch.tensor(spect, dtype=torch.float64, requires_grad=True)
        ob, od = O.forward(sd64, x64, sum_head=hp["sum_head"])
        og = torch.autograd.grad((ob, od), [x64] + [sd64[n] for n in names], (lb.grad.double(), ld.grad.double()))
        for n, g in zip(["spect"] + names, og):
            ref = x.grad if n == "spect" else grads[n]
            err = float((g - ref).norm() / ref.norm())
            assert err < 1e-6, f"{family}: the restatement's gradient of {n} differs by {err:.2e}"
        assert torch.allclose(ob, pred["beat"].detach().double(), atol=1e-5)
        assert torch.allclose(od, pred["downbeat"].detach(), atol=1e-5)

        index = {n: i for i, n in enumerate(sd)}  # fingerprints are seeded by the entry's index in the state_dict
        out.update({
            f"family{k}": np.array(family), f"seed{k}": np.array(seed), f"spect{k}": spect,
            f"truth_beat{k}": beat, f"truth_downbeat{k}": down, f"padding_mask{k}": pad, f"downbeat_mask{k}": dmask,
            f"beat{k}": pred["beat"].detach().double().numpy(), f"downbeat{k}": pred["downbeat"].detach().numpy(),
            f"loss{k}": np.array(loss.item()), f"dbeat{k}": lb.grad.double().numpy(),
            f"ddown{k}": ld.grad.double().numpy(), f"dspect{k}": x.grad.numpy(), f"names{k}": np.array(names),
            f"fp{k}": np.stack([fingerprint(grads[n].numpy(), index[n]) for n in names]),
        })
        print(f"{family}: B={B} L={L} loss {loss.item():.6f}, {len(names)} gradients, restatement agrees")
    path = os.path.join(ROOT, "tests", "golden", "train_grads.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
