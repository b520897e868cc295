"""CPU tests (no GPU) of the step list of tests/forward_steps_reference.py, which tests/test_gpu_forward_steps.py ties
to the forward pass bit for bit: its taps are the oracle's, every packed parameter is read by exactly one step of a
pass, and its chains evaluated in float64 from the hook contracts (Eval64) compose to oracle.forward in float64 at
every tap, while each wrong argument of forward_steps_reference.mutations moves its step far off the oracle.  So the
chains the pass is tied to are the reference model's, checked independently of the library."""
import numpy as np
import pytest
import torch

import forward_steps_reference as R
from beat_this_b200 import synthetic, weights
from oracle import beat_this_oracle as O

FAMILIES = ["small0", "final0", "small0-nopartial", "final0-nopartial", "small0-nosum", "final0-nosum"]
WAVES = [R.Wave(2, 1500), R.Wave(4, 1500, [1500, 1500, 712, 52]), R.Wave(2, 3000)]


def _packed(name):
    hp = synthetic.model_hparams(name)
    return hp, synthetic.make_state_dict(hp, 0)


@pytest.mark.parametrize("name", FAMILIES)
def test_steps_are_the_oracle_taps(name):
    hp, sd = _packed(name)
    taps = {}
    with torch.inference_mode():
        O.forward(sd, torch.rand(1, 20, 128, generator=torch.Generator().manual_seed(0)) * 7, taps,
                  sum_head=hp["sum_head"])
    assert R.tap_names(hp) == list(taps)
    for half in (False, True):
        for wave in WAVES:
            steps = R.forward_steps(hp, half, wave)
            prod = [s for s in steps if not s.tap_mode]
            assert [s.name for s in prod] == R.production_taps(hp, half) + ["logits"]
            assert sorted(s.name for s in steps if s.name != "logits") == sorted(taps), "a tap has no step"
            assert len({(s.name, s.tap_mode) for s in steps}) == len(steps)
            # each production step reads the production step before it; a tap-mode variant reads what its pair reads
            names = ["spect"] + [s.name for s in prod]
            assert [s.input for s in prod] == names[:-1]
            pair_input = {s.name.replace(".ff", ".attn"): s.input for s in prod if s.kind.startswith("pair_")}
            for s in steps:
                if s.tap_mode:
                    assert half and s.C in R.FUSED_WIDTHS and s.input == pair_input[s.name]
            # fused kernels on the 16-bit path at widths 32 and 64 only; the out-projection inside the FFN exactly
            # where a pair is
            for s in steps:
                ops = [c.op for c in s.chain]
                fused = half and s.C in R.FUSED_WIDTHS and s.kind != "conv"
                assert ("fused_qkv" in ops or "fused_ff" in ops) == fused, (s.name, ops)
                if s.kind.startswith("pair_"):
                    assert ops[-1] == "fused_ff" and s.chain[-1].args["wout"] == s.name.replace(".ff", ".attn") + ".wout"


@pytest.mark.parametrize("name", FAMILIES)
def test_every_parameter_is_read_by_one_step(name):
    hp, sd = _packed(name)
    packed = weights.pack_parameters(sd, hp)
    model = {k for k in packed if not k.startswith(("mel.", "rope."))}
    for half in (False, True):
        steps = [s for s in R.forward_steps(hp, half, WAVES[1]) if not s.tap_mode]
        read = [p for s in steps for p in s.params]
        assert sorted(read) == sorted(model), "parameters read by no step or by two"
        for s in R.forward_steps(hp, half, WAVES[1]):
            named = set()
            for c in s.chain:
                for k, v in c.args.items():
                    if k in ("w", "wg", "bg", "bias", "w1", "b1", "w2", "b2", "wout", "b") and v is not None:
                        named.add(v)
                named.update(c.args.get("params", ()))
            assert named == set(s.params), (s.name, named, s.params)


def _composition(name, half, wave):
    """The float64 chains of a pass over `wave` (each chunk its own clip, starting at frame 0) and oracle.forward per
    chunk in float64: (steps, {step: (error, chain outputs...)}, oracle taps per chunk, registers before each step,
    evaluator factory)."""
    hp = synthetic.model_hparams(name)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in synthetic.make_state_dict(hp, 0).items()}
    packed = weights.pack_parameters(sd, hp, rope_positions=max(1500, wave.L), dtype=np.float64)
    P = {k: torch.from_numpy(v) for k, v in packed.items()}
    lens = wave.lens or [wave.L] * wave.nb
    offs = np.concatenate([[0], np.cumsum(lens)]).tolist()
    chunks = [(o, n, 0, o, 0, n, n) for o, n in zip(offs, lens)]
    spect = torch.rand(offs[-1], 128, generator=torch.Generator().manual_seed(wave.L), dtype=torch.float64) * 7
    oracle = []
    with torch.inference_mode():
        for o, n in zip(offs, lens):
            taps = {}
            b, d = O.forward(sd, spect[o : o + n][None], taps, sum_head=hp["sum_head"])
            taps["logits"] = torch.stack((b[0], d[0]))
            oracle.append(taps)
    steps = R.forward_steps(hp, half, wave)
    return hp, steps, oracle, lambda regs: R.Eval64(P, wave, chunks, spect, regs), offs


def _error(out, name, oracle, wave, offs):
    """max |chain - oracle| / (1 + |oracle|) over the rows each chunk owns (t < its length)."""
    worst = 0.0
    for i, taps in enumerate(oracle):
        ref = taps[name]
        if name == "logits":
            got = out[:, offs[i] : offs[i + 1]]
        elif ref.ndim == 4:  # [1, F, n, C] frontend
            got = out.reshape(wave.nb, ref.shape[1], wave.L, -1)[i : i + 1, :, : ref.shape[2]]
        else:  # [1, n, D]
            got = out.reshape(wave.nb, wave.L, -1)[i : i + 1, : ref.shape[1]]
        worst = max(worst, ((got - ref).abs() / (1 + ref.abs())).max().item())
    return worst


COMPOSE_TOL = 1e-11  # float64 round-off of the same operations in another order, relative to 1 + |value|
COMPOSE_CASES = [(n, h, w) for n in ("small0", "small0-nopartial", "small0-nosum") for h in (False, True)
                 for w in (R.Wave(2, 40), R.Wave(3, 40, [40, 23, 7]))] + [
    ("final0", True, R.Wave(2, 24, [24, 9])), ("small0", True, R.Wave(1, 1600))]


@pytest.mark.parametrize("name,half,wave", COMPOSE_CASES,
                         ids=[f"{n}-{'h16' if h else 'f32'}-{w.nb}x{w.L}{'-varlen' if w.varlen else ''}"
                              for n, h, w in COMPOSE_CASES])
def test_chains_compose_to_the_oracle(name, half, wave):
    """Every chain evaluated in float64 from the hook contracts (forward_steps_reference.Eval64), composed over the
    pass, gives oracle.forward in float64 at every tap and on the logits, chunk by chunk: every weight, F, position
    mode, q scale, key length and zero_tail of the chains is the reference model's.  The tap-mode variants give the
    oracle's attention taps from the same inputs."""
    hp, steps, oracle, ev, offs = _composition(name, half, wave)
    regs, before = {}, {}
    for s in steps:
        if s.tap_mode:
            r = dict(before[s.name.replace(".attn", ".ff")])
            out = ev(r).run(s)
        else:
            before[s.name] = dict(regs)
            out = ev(regs).run(s)
        err = _error(out, s.name, oracle, wave, offs)
        print(f"{name} {'h16' if half else 'f32'} {s.name:9s}{' (tap mode)' if s.tap_mode else ''}: {err:.2e}")
        assert err < COMPOSE_TOL, f"{s.name}: {err:.3e} off the oracle"


@pytest.mark.parametrize("half", [False, True])
def test_mutations_leave_the_oracle(half):
    """Each wrong argument of forward_steps_reference.mutations, alone, moves its step's float64 value off the
    oracle's tap by far more than the composition's round-off: the chains pin each of them."""
    wave = R.Wave(3, 40, [40, 23, 7])
    hp, steps, oracle, ev, offs = _composition("small0", half, wave)
    regs, before = {}, {}
    for s in steps:
        if not s.tap_mode:
            before[s.name] = dict(regs)
            ev(regs).run(s)
    muts = R.mutations(half, wave, steps)
    assert len(muts) == (8 if half else 6)
    for what, s, m in muts:
        err = _error(ev(dict(before[s.name])).run(m), s.name, oracle, wave, offs)
        print(f"{'h16' if half else 'f32'} {s.name} with {what}: {err:.2e} off the oracle")
        assert err > 1e6 * COMPOSE_TOL, f"{s.name} with {what} stays within {err:.3e} of the oracle"
