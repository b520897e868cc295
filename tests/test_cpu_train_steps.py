"""CPU tests (no GPU) of the step list of tests/train_steps_reference.py, which tests/test_gpu_train_steps.py ties to
the training passes bit for bit: its steps are the reference model's layer stack in order, every table entry is read by
exactly one forward step and every trainable entry gets its gradient from exactly one backward chain, the store layout
is the independently counted one, and the chains evaluated in float64 (Eval64) and composed over whole passes give
float64 autograd of the reference (oracle.forward in eval mode, train_mode_reference.forward_train with the library's
dropout masks and batch statistics in training mode) on the logits, every gradient, dspect and the running statistics.
Each wrong argument of train_steps_reference.mutations moves the composed result far off autograd, except the dW
split count, which only reorders a sum."""
import collections
import math

import pytest
import torch

import train_mode_reference as TM
import train_steps_reference as R
from beat_this_b200 import synthetic
from oracle import beat_this_oracle as O
from support import _spect

COMPOSE_TOL = 1e-11  # float64 round-off of the same operations in another order, relative to 1 + |value|
# Training mode: each batch-statistics BatchNorm's input gradient is a difference of terms that cancel (it sums to zero
# per channel), and a rate of 0.9 scales kept values by 10, so the same round-off reaches 1.6e-11 there (final0, small0
# zero-padded at rates 0.5 / 0.9)
COMPOSE_TOL_TRAIN = 1e-10
RATES = [None, (0.0, 0.0), (0.1, 0.2), (0.5, 0.9)]  # None: eval mode
SEED = 987654321
CONFIGS = [  # family, B, L, lengths of a zero-padded batch, overrides, the rates it runs at
    ("small0", 3, 17, None, {}, RATES),
    ("small0-nosum", 3, 17, None, {}, RATES),
    ("small0-nopartial", 3, 17, None, {}, RATES),
    ("1024", 3, 17, None, {"ff_mult": 2}, RATES),
    # RoPE positions past 1500.  Eval mode and rate 0 only: with dropout, the float64 masks of its 6.9e8 probabilities
    # per pass take the numpy Philox generator some ten minutes (the GPU test runs it at every rate)
    ("small0", 2, 1700, None, {}, RATES[:2]),
    ("small0", 3, 400, (400, 251, 90), {}, RATES),
    ("final0", 2, 300, None, {}, RATES),
]
CASES = [(f, B, L, n, o, r) for f, B, L, n, o, rates in CONFIGS for r in rates]


def _ids(c):
    f, B, L, n, o, r = c
    return f"{f}{'-ff2' if o else ''}-{B}x{L}{'-padded' if n else ''}-{'eval' if r is None else 'p%g-%g' % r}"


def _hp(family, overrides):
    return dict(synthetic.model_hparams(family), **overrides)


class Pass64:
    """One training forward and backward of a model in float64: the chains composed (run), and float64 autograd of
    the reference on the same parameters, batch and logit gradients (reference)."""

    def __init__(self, family, B, L, lengths, overrides, rates):
        self.hp = _hp(family, overrides)
        self.B, self.L = B, L
        self.mode = None if rates is None else (SEED,) + tuple(rates)
        sd = synthetic.make_state_dict(self.hp, 0)
        self.names = [n for names in R.table(self.hp) for n in names]
        assert self.names == list(sd), "the table is not BeatThis.state_dict()'s order"
        self.sd = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
        self.x = _spect(B, L, 1, lengths).double()
        g = torch.Generator().manual_seed(2)
        self.dbeat = torch.randn(B, L, generator=g, dtype=torch.float64)
        self.ddown = torch.randn(B, L, generator=g, dtype=torch.float64)
        self.steps = R.train_steps(self.hp, B, L, self.mode)

    def run(self, replace=None):
        """The chains over the whole pass (replace: {(step index, "fwd" | "bwd"): chain}) -> the Mem after it."""
        replace = replace or {}
        BL = self.B * self.L
        _, total = R.layout(self.hp, self.B, self.L, self.mode is not None)
        nan = lambda n: torch.full((n,), math.nan, dtype=torch.float64)  # noqa: E731
        P = [self.sd[n].reshape(-1) for n in self.names]
        G = [nan(p.numel()) if R.trainable(n) else None for n, p in zip(self.names, P)]
        S = {k: nan(n) for k, n in R.scratch_sizes(BL).items() if k != "part"}
        X = dict(beat=nan(BL), down=nan(BL), dbeat=self.dbeat.reshape(-1), ddown=self.ddown.reshape(-1),
                 dspect=nan(BL * 128))
        mem = R.Mem(nan(total), P, G, [p.clone() for p in P], S, X)
        mem.get(self.steps[0].A("in"))[:] = self.x.reshape(-1)
        ev = R.Eval64(mem)
        for s in self.steps:
            ev.run(replace.get((s.index, "fwd"), s.fwd))
        for s in reversed(self.steps):
            ev.run(replace.get((s.index, "bwd"), s.bwd))
        return mem

    def reference(self):
        """{"beat", "down", "dspect", every trainable entry, every running statistic after the pass}: float64."""
        sd = {k: v.clone().requires_grad_(R.trainable(k)) if v.is_floating_point() else v for k, v in self.sd.items()}
        x = self.x.clone().requires_grad_(True)
        stats = {}
        if self.mode is None:
            beat, down = O.forward(sd, x, sum_head=self.hp["sum_head"])
        else:
            beat, down, stats = TM.forward_train(sd, x, *self.mode, sum_head=self.hp["sum_head"])
        wrt = [n for n in self.names if R.trainable(n)]
        grads = torch.autograd.grad((beat, down), [x] + [sd[n] for n in wrt], (self.dbeat, self.ddown))
        out = {"beat": beat.detach(), "down": down.detach(), "dspect": grads[0]}
        out.update(zip(wrt, grads[1:]))
        for p, (mean, var, N) in stats.items():
            out[p + ".running_mean"] = 0.9 * self.sd[p + ".running_mean"] + 0.1 * mean
            out[p + ".running_var"] = 0.9 * self.sd[p + ".running_var"] + 0.1 * var * N / (N - 1)
        return out

    def errors(self, mem, ref):
        """max |chain - reference| / (1 + |reference|) per output."""
        got = {"beat": mem.X["beat"], "down": mem.X["down"], "dspect": mem.X["dspect"]}
        for i, n in enumerate(self.names):
            if n in ref and n not in got:
                got[n] = mem.G[i] if R.trainable(n) else mem.R[i]
        return {k: ((got[k] - v.reshape(-1)).abs() / (1 + v.reshape(-1).abs())).max().item() for k, v in ref.items()}


# ---------------------------------------------------------------------------------------------- structure
@pytest.mark.parametrize("family", ["small0", "small0-nopartial", "final0", "small0-nosum"])
@pytest.mark.parametrize("train", [False, True])
def test_steps_cover_the_table_once(family, train):
    hp = _hp(family, {})
    B, L = 3, 17
    mode = (1, 0.1, 0.2) if train else None
    steps = R.train_steps(hp, B, L, mode)
    names = [n for t in R.table(hp) for n in t]
    assert names == list(synthetic.make_state_dict(hp, 0))
    # the steps are the reference's layer stack in order: the modules of the table, step by step
    mods = [s.module for s in steps]
    assert mods[0] == "frontend.stem" and mods[-1] == "" and mods[-2].startswith("transformer_blocks.layers.")
    for s, entries in zip(steps, R.table(hp)):
        assert all(n.startswith(s.module) for n in entries if s.module), (s.module, entries)
    assert [names[s.p] for s in steps] == [t[0] for t in R.table(hp)]
    # every entry read by exactly one forward step (the num_batches_tracked counters by none)
    readers = {i: [] for i in range(len(names))}
    for s in steps:
        for i in {r[1] for c in s.fwd for r in c.slots if r is not None and r[0] in "PR"}:
            readers[i].append(s.index)
    for i, n in enumerate(names):
        want = 0 if n.endswith(".num_batches_tracked") else 1
        assert len(readers[i]) == want, (n, readers[i])
        if train and n.endswith((".running_mean", ".running_var")):  # training mode: only the update reads them
            assert all(r[0] == "R" for c in steps[readers[i][0]].fwd for r in c.slots if r and r[1] == i and r[0] in "PR")
    # every trainable entry written by exactly one call of one backward chain, and nothing else written
    writers = {}
    for s in steps:
        for c in s.bwd:
            for r in c.slots:
                if r is not None and r[0] == "G":
                    writers.setdefault(r[1], []).append(s.index)
    assert sorted(writers) == [i for i, n in enumerate(names) if R.trainable(n)]
    assert all(len(v) == 1 for v in writers.values())
    # the layout: the independently counted store, and every region inside it, 4-float aligned, in order
    regs, total = R.layout(hp, B, L, train)
    want = TM.activation_floats(hp, B, L)
    if not train:
        Fs, C = hp["spect_dim"], hp["stem_dim"]
        want -= 2 * R.r4(Fs) + 2 * R.r4(C) + sum(2 * R.r4(2 * C * 2**i) for i in range(3))
    assert total == want
    offs = sorted(v for r in regs for v in r.values())
    assert offs[0][0] == 0 and all(o % 4 == 0 for o, _ in offs)
    assert all(a[0] + R.r4(a[1]) == b[0] for a, b in zip(offs, offs[1:])) and offs[-1][0] + R.r4(offs[-1][1]) == total


# ---------------------------------------------------------------------------------------------- composition
@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_chains_compose_to_float64_autograd(case):
    ps = Pass64(*case)
    errs = ps.errors(ps.run(), ps.reference())
    worst = max(errs, key=errs.get)
    print(f"{_ids(case)}: {len(errs)} outputs, worst {errs[worst]:.2e} ({worst})")
    assert errs[worst] < (COMPOSE_TOL if ps.mode is None else COMPOSE_TOL_TRAIN), \
        f"{worst}: {errs[worst]:.3e} off float64 autograd"


@pytest.mark.parametrize("rates", [None, (0.1, 0.2)], ids=["eval", "p0.1-0.2"])
@pytest.mark.parametrize("family", ["small0", "small0-nosum"])
def test_mutations_leave_autograd(family, rates):
    """Each wrong argument of train_steps_reference.mutations, alone, moves the composed pass off float64 autograd
    by far more than the composition's round-off; another dW split leaves it within the round-off."""
    ps = Pass64(family, 3, 17, None, {}, rates)
    tol = COMPOSE_TOL if ps.mode is None else COMPOSE_TOL_TRAIN
    ref = ps.reference()
    muts = R.mutations(ps.hp, ps.B, ps.L, ps.steps, ps.mode)
    assert len(muts) == (14 if rates else 10)
    margins = []
    for what, i, d, chain, bitwise_only in muts:
        errs = ps.errors(ps.run({(i, d): chain}), ref)
        worst = max(errs, key=errs.get)
        print(f"{family} {'eval' if rates is None else rates} step {i} {d} with {what}: {errs[worst]:.2e} ({worst})")
        if bitwise_only:
            assert errs[worst] < tol, f"{what}: {errs[worst]:.3e}"
        else:
            assert errs[worst] > 1e5 * tol, f"step {i} {d} with {what} stays within {errs[worst]:.3e}"
            margins.append(errs[worst] / tol)
    print(f"{family} {'eval' if rates is None else rates}: mutation margins {min(margins):.2e} .. {max(margins):.2e} "
          f"x the composition tolerance")


@pytest.mark.parametrize("family,rates", [("small0", None), ("small0", (0.1, 0.2)), ("small0-nopartial", (0.0, 0.0)),
                                          ("small0-nosum", (0.5, 0.9))])
def test_eval64_ops_are_the_kernel_restatements(family, rates):
    """Eval64 restates each op in exact float64; the kernels' unit tests hold them to train_kernels_reference's
    restatements.  Every call of a pass, evaluated by Eval64, lies within that restatement's bound on its own inputs
    (train_steps_reference.check64, the same check the GPU test runs on the hooks), so the two agree on every sign,
    flag and layout convention, and the composition's value is the one the kernels are tested against."""
    ps = Pass64(family, 2, 40, None, {}, rates)
    mem = ps.run()  # a pass's data, then every call again on it
    ratios, skipped = {}, collections.Counter()
    bad = []
    ev = R.Eval64(mem)
    for s, chain in [(s, s.fwd) for s in ps.steps] + [(s, s.bwd) for s in reversed(ps.steps)]:
        for c in chain:
            a = [mem.get(r) for r in c.slots]
            before = {i: a[i].clone() for i in R.INPLACE.get(c.op, ()) if i < len(a) and a[i] is not None}
            ev.run([c])
            bad += [(s.index, c.op, what, r) for what, r in R.check64(c, a, before, ratios, skipped) if not r <= 1.0]
    print(f"{family} {rates}: worst ratios " + ", ".join(f"{k} {v:.2g}" for k, v in sorted(ratios.items())) +
          f"; without a bound: {dict(skipped)}")
    assert not bad, bad[:10]
    assert len(ratios) >= (17 if rates else 20)
