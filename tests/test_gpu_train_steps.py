"""GPU tests (pytest -m gpu): every step of the training passes (bt_train_forward_ex, bt_train_backward_ex) is, bit for
bit, the chain of training-kernel test hooks that tests/train_steps_reference.py lists for it.  The hooks are
unit-tested against float64 one kernel at a time (test_gpu_train_kernels.py, test_gpu_train_mode.py), and the chains,
evaluated in float64 and composed over a pass, give float64 autograd of the reference (test_cpu_train_steps.py); so a
wrong weight, dropout site, statistics slot, sequence geometry, RoPE mode, scale, flag or scratch buffer anywhere in
the passes breaks a tie here, however small its effect on the end-to-end gradients.

Per configuration (the CPU test's, plus final0 at the reference's training batch of 8 x 1500):
- two forward + backward calls from the same parameters and running statistics, on a NaN-filled store, give the same
  bits everywhere; every region of the documented layout is written and every alignment pad is left NaN;
- forward tie: each step's chain, run on the step's stored input, gives every activation it stores, its batch
  statistics and the next step's input (the head: the logits); the running statistics the chains move are the pass's;
- backward tie: the chains replayed from the logits' gradients and the pass's store give every gradient and dspect;
  the first step, going backward, that differs is reported; a call with some gradients NULL (the stem's bn1d entries
  and dspect among them: the stem's early return) leaves the others' bits unchanged;
- launch accounting: the chains' calls, named by the pass launch each stands for, are the profile of one call of each
  pass;
- each of train_steps_reference.mutations breaks its step's tie;
- float64 on real data: every call of both replays is held to its train_kernels_reference restatement on its own
  device inputs, within that op's bound (train_steps_reference.check64); the worst ratio per op is printed.
Mismatches are gathered per configuration and reported together."""
import collections
import math

import pytest
import torch

import train_steps_reference as R
from beat_this_b200 import synthetic
from beat_this_b200.engine import Engine
from support import DEV, _spect, bits

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

RATES = [None, (0.0, 0.0), (0.1, 0.2), (0.5, 0.9)]  # None: eval mode
SEED = 987654321
CONFIGS = [  # family, B, L, lengths of a zero-padded batch, overrides, the rates it runs at
    ("small0", 3, 17, None, {}, RATES),
    ("small0-nosum", 3, 17, None, {}, RATES),
    ("small0-nopartial", 3, 17, None, {}, RATES),
    ("1024", 3, 17, None, {"ff_mult": 2}, RATES),
    ("small0", 2, 1700, None, {}, RATES),
    ("small0", 3, 400, (400, 251, 90), {}, RATES),
    ("final0", 2, 300, None, {}, RATES),
    ("final0", 8, 1500, None, {}, RATES[:1] + RATES[2:3]),
]
CASES = [(f, B, L, n, o, r) for f, B, L, n, o, rates in CONFIGS for r in rates]


def _ids(c):
    f, B, L, n, o, r = c
    return f"{f}{'-ff2' if o else ''}-{B}x{L}{'-padded' if n else ''}-{'eval' if r is None else 'p%g-%g' % r}"


def _nan(n):
    return torch.full((n,), math.nan, device=DEV)


def _same(a, b):
    return torch.equal(bits(a.contiguous().view(-1)), bits(b.contiguous().view(-1)))


def _differ(a, b):
    """(elements whose bits differ, max abs difference)."""
    a, b = a.contiguous().view(-1), b.contiguous().view(-1)
    n = int((bits(a) != bits(b)).sum())
    return n, ((a.double() - b.double()).abs().nan_to_num(math.inf).max().item() if n else 0.0)


class Case:
    """One model, batch and mode: the parameters, running statistics and logit gradients on the device, the passes
    and the replay of their chains."""

    def __init__(self, family, B, L, lengths, overrides, rates):
        self.hp = dict(synthetic.model_hparams(family), **overrides)
        self.B, self.L = B, L
        self.mode = None if rates is None else (SEED,) + tuple(rates)
        self.eng = Engine(None, self.hp, DEV)
        sd = synthetic.make_state_dict(self.hp, 0)
        self.names = [n for t in R.table(self.hp) for n in t]
        assert self.names == list(sd)
        self.P = [sd[n].float().contiguous().to(DEV) for n in self.names]
        self.running0 = [p.clone() for p in self.P]
        self.trainable = [R.trainable(n) for n in self.names]
        self.x = _spect(B, L, 1, lengths).to(DEV)
        g = torch.Generator().manual_seed(2)
        self.dbeat, self.ddown = (torch.randn(B, L, generator=g).to(DEV) for _ in range(2))
        self.regions, self.total = R.layout(self.hp, B, L, self.mode is not None)
        self.steps = R.train_steps(self.hp, B, L, self.mode)
        self.ratios, self.skipped = {}, collections.Counter()  # the float64 check of the replayed calls

    def run_pass(self):
        """A forward and a backward call on a NaN store: (store, running statistics after, logits, grads, dspect)."""
        B, L = self.B, self.L
        act = _nan(self.total)
        running = [p.clone() for p in self.running0]
        beat, down = _nan(B * L).view(B, L), _nan(B * L).view(B, L)
        self.eng.train_forward(self.P, self.x, act.view(torch.uint8), beat, down, mode=self.mode, running=running)
        grads = [torch.full_like(p, math.nan) if t else None for p, t in zip(self.P, self.trainable)]
        dspect = _nan(B * L * 128).view(B, L, 128)
        self.eng.train_backward(self.P, act.view(torch.uint8), B, L, self.dbeat, self.ddown, grads, dspect,
                                mode=self.mode)
        torch.cuda.synchronize()
        return act, running, beat, down, grads, dspect

    def mem(self, store, G=None, running=None, X=None):
        flat = lambda ts: None if ts is None else [None if t is None else t.view(-1) for t in ts]  # noqa: E731
        S = {k: _nan(n) for k, n in R.scratch_sizes(self.B * self.L).items()}
        return R.Mem(store, flat(self.P), flat(G), flat(running), S, X or {})

    def run(self, mem, chain, check=False):
        """Runs the calls of a chain; check: each against float64 as it runs -> the calls over their bounds."""
        bad = []
        for c in chain:
            a = [mem.get(r) for r in c.slots]
            before = {i: a[i].clone() for i in R.INPLACE.get(c.op, ()) if check and i < len(a) and a[i] is not None}
            self.eng.debug_train_kernel(c.op, a, **c.desc)
            if check:
                bad += [f"{c.op} {what} ({c.prod[0]}): {r:.3g} x its bound"
                        for what, r in R.check64(c, a, before, self.ratios, self.skipped) if not r <= 1.0]
        return bad


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_training_steps_tie_to_hooks(case):
    cs = Case(*case)
    tag = _ids(case)
    failures = []
    B, L = cs.B, cs.L

    # two calls, bitwise; the layout written everywhere, its pads untouched
    assert cs.eng.train_activation_bytes(B, L, cs.mode) == 4 * cs.total
    act, running, beat, down, grads, dspect = cs.run_pass()
    again = cs.run_pass()
    for what, a, b in [("store", act, again[0]), ("beat", beat, again[2]), ("down", down, again[3]),
                       ("dspect", dspect, again[5])] + \
            [(n, a, b) for n, a, b in zip(cs.names, running, again[1]) if "running" in n] + \
            [(n, a, b) for n, a, b in zip(cs.names, grads, again[4]) if a is not None]:
        if not _same(a, b):
            failures.append(f"two calls differ in {what}")
    for s, regs in zip(cs.steps, cs.regions):
        for k, (off, n) in regs.items():
            if torch.isnan(act[off : off + n]).any():
                failures.append(f"step {s.index} ({s.module or 'head'}) region {k}: not every element written")
            if not torch.isnan(act[off + n : off + R.r4(n)]).all():
                failures.append(f"step {s.index} region {k}: a pad after it was written")
    del again

    # launch accounting: one call of each pass against the chains
    for d, fn in (("fwd", lambda: cs.eng.train_forward(cs.P, cs.x, _nan(cs.total).view(torch.uint8), _nan(B * L),
                                                       _nan(B * L), mode=cs.mode,
                                                       running=[p.clone() for p in cs.running0])),
                  ("bwd", lambda: cs.eng.train_backward(cs.P, act.view(torch.uint8), B, L, cs.dbeat, cs.ddown,
                                                        [torch.empty_like(g) if g is not None else None for g in grads],
                                                        _nan(B * L * 128), mode=cs.mode))):
        cs.eng.profile_enable(True)
        cs.eng.profile_reset()
        fn()
        prof = cs.eng.profile_results()
        cs.eng.profile_enable(False)
        launched = collections.Counter({k: v[1] for k, v in prof.items() if v[1]})
        chained = collections.Counter(p for s in cs.steps for c in getattr(s, d) for p in c.prod)
        if launched != chained:
            failures.append(f"{d} pass: chains {dict(chained - launched)} not launched; launches "
                            f"{dict(launched - chained)} in no chain")

    # forward tie, step by step from each step's stored input
    pass_mem = R.Mem(act, None, [None if g is None else g.view(-1) for g in grads],
                     [t.view(-1) for t in running], {}, dict(beat=beat.view(-1), down=down.view(-1)))
    fwd_outputs = {s.index: R.step_outputs(cs.steps, s, "fwd") for s in cs.steps}

    def forward_replay(s, chain, rep_running, check=False):
        m = cs.mem(_nan(cs.total), running=rep_running, X=dict(beat=_nan(B * L), down=_nan(B * L)))
        off, n = s.regions["in"]
        m.store[off : off + n] = act[off : off + n]
        bad = cs.run(m, chain, check)
        failures.extend(f"forward step {s.index} ({s.kind} {s.module}) float64: {b}" for b in bad)
        return [(r, m.get(r)) for r in fwd_outputs[s.index]]

    rep_running = [p.clone() for p in cs.running0]
    for s in cs.steps:
        for r, got in forward_replay(s, s.fwd, rep_running, check=True):
            n, mx = _differ(got, pass_mem.get(r))
            if n:
                failures.append(f"forward step {s.index} ({s.kind} {s.module}) {r[:2]}: {n} elements differ, max {mx:.3e}")
    for n_, a, b in zip(cs.names, rep_running, running):
        if "running" in n_ and not _same(a, b):
            failures.append(f"running statistics {n_}: the chains' reductions differ from the pass")
    print(f"{tag}: forward tie checked over {len(cs.steps)} steps")

    # backward tie, replayed from the logits' gradients, the first differing step going backward reported
    muts = R.mutations(cs.hp, B, L, cs.steps, cs.mode)
    snap = {i for _, i, d, _, _ in muts if d == "bwd"}
    G = [torch.full_like(g, math.nan) if g is not None else None for g in grads]
    bm = cs.mem(act, G=G, X=dict(dbeat=cs.dbeat.view(-1), ddown=cs.ddown.view(-1), dspect=_nan(B * L * 128)))
    before, after, first = {}, {}, None
    for s in reversed(cs.steps):
        if s.index in snap:
            before[s.index] = bm.S["dcur"].clone()
        failures.extend(f"backward step {s.index} ({s.kind} {s.module or 'head'}) float64: {b}"
                        for b in cs.run(bm, s.bwd, check=True))
        if s.index in snap:
            after[s.index] = bm.S["dcur"].clone()
        for r in R.step_outputs(cs.steps, s, "bwd"):
            if r[0] == "D":
                continue
            want = dspect.view(-1) if r == ("X", "dspect") else pass_mem.get(r)
            n, mx = _differ(bm.get(r), want)
            if n:
                where = cs.names[r[1]] if r[0] == "G" else "dspect"
                if first is None:
                    first = f"backward step {s.index} ({s.kind} {s.module or 'head'}) first differs"
                failures.append(f"backward step {s.index} {where}: {n} elements differ, max {mx:.3e}")
    if first:
        failures.insert(0, first)
    print(f"{tag}: backward tie checked over {len(cs.steps)} steps")
    for op in sorted(cs.ratios):
        print(f"{tag}: float64 worst |err| / bound of {op:12s} {cs.ratios[op]:.3g}")
    for op, n in sorted(cs.skipped.items()):
        print(f"{tag}: {n} calls of {op} without a derived bound")

    # NULL gradients: every other trainable entry, the stem's bn1d pair and dspect left out
    stem = cs.steps[0]
    keep = [g is not None and (i % 2 == 0) and i not in (stem.p, stem.p + 1) for i, g in enumerate(grads)]
    part = [torch.full_like(g, math.nan) if k else None for g, k in zip(grads, keep)]
    cs.eng.train_backward(cs.P, act.view(torch.uint8), B, L, cs.dbeat, cs.ddown, part, None, mode=cs.mode)
    torch.cuda.synchronize()
    for n_, g, k, full in zip(cs.names, part, keep, grads):
        if k and not _same(g, full):
            failures.append(f"with some gradients NULL, {n_} changes")

    # every mutation breaks its step's tie
    for what, i, d, chain, _ in muts:
        s = cs.steps[i]
        if d == "fwd":
            outs = forward_replay(s, chain, [p.clone() for p in cs.running0])
            diff = sum(_differ(got, pass_mem.get(r))[0] for r, got in outs)
        else:
            G2 = [torch.full_like(g, math.nan) if g is not None else None for g in grads]
            m = cs.mem(act, G=G2, X=dict(dbeat=cs.dbeat.view(-1), ddown=cs.ddown.view(-1), dspect=_nan(B * L * 128)))
            m.S["dcur"].copy_(before[i])
            cs.run(m, chain)
            diff = 0
            for r in R.step_outputs(cs.steps, s, "bwd"):
                want = (dspect.view(-1) if r == ("X", "dspect") else after[i][: r[1]] if r[0] == "D"
                        else pass_mem.get(r))
                diff += _differ(m.get(r), want)[0]
        print(f"{tag} step {i} {d} with {what}: {diff} elements differ")
        if diff == 0:
            failures.append(f"step {i} {d} with {what} leaves the tie intact")

    for f in failures:
        print(f"FAILED {tag}: {f}")
    cs.eng.close()
    assert not failures, f"{tag}: {len(failures)} failures:\n" + "\n".join(failures[:40])
