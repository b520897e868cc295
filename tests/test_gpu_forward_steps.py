"""GPU tests (pytest -m gpu): every step of the forward pass is, bit for bit, the chain of kernel test hooks that
tests/forward_steps_reference.py lists for it, run on the tap in front of the step as the forward pass saw it.  The
hooks are unit-tested against float64 one kernel at a time (test_gpu_kernels.py, test_gpu_attention.py,
test_gpu_fused.py, test_gpu_chunk_kernels.py), so this ties those bounds to every launch of the pass: a wrong weight,
F, position mode, q scale, key length, gate or stale 16-bit copy in the pass would make a step differ from its chain.
The chains themselves are the reference model's: evaluated in float64 from the hook contracts, they compose to
oracle.forward in float64 (tests/test_cpu_forward_steps.py).

Configurations, one wave each (a tap keeps only the last wave's values): small0 and final0 on the fp32 and the 16-bit
context, over a dense wave of full 1500-frame chunks, a wave of chunks of different lengths from bt_spect2frames
(masked keys, zero_tail, one chunk table for F sequences), and a wave of 3000-frame chunks on a context loaded for
them (RoPE rows past 1500, time-attention planes longer than 1500); final0-nopartial (convolutions fed by the
rounded fp32 stream) and small0-nosum (Head instead of SumHead) on the 16-bit context.

Each configuration also checks that two forward calls give the same logits bitwise (the tie assumes run-to-run
determinism) and that the chains account for every launch of a forward call: their calls, named by the launch each
stands for, are the launch profile of the pass.  Then, for one step of each kind, it reruns the chain with one wrong
but valid argument (posmode 0 or F halved for a frequency attention, q scale 1 for a 16-bit time attention, every key
length L in a wave of chunks of different lengths, the next layer's w2, the other attention's out-projection in a
fused pair, the convolution's time shifts reversed, another bias for frontend.linear) and requires the tie to break:
each such argument is live in its hook, so the pass cannot pass it wrongly and still tie.  The same mutations move
the float64 value of their step off the oracle (tests/test_cpu_forward_steps.py).  Mismatches are gathered
per configuration and reported together."""
import collections
import zlib

import numpy as np
import pytest
import torch

import forward_steps_reference as R
from numerics import QSCALE_H16
from support import bits, dev  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

NAN = float("nan")
LONG = 3000  # frames of the long chunks, and the maximum chunk length of their context


def _planner(lib):
    from beat_this_b200._lib import OVERLAP_MODES, bt_chunking, i64_array

    ck = bt_chunking(1500, 6, OVERLAP_MODES["keep_first"])

    def plan(T):
        n = lib.bt_plan_chunking_max(T, ck, 1500, None, None, None, None, 0)
        arrs = [i64_array([0] * n) for _ in range(4)]
        assert lib.bt_plan_chunking_max(T, ck, 1500, *arrs, n) == n
        return [list(a) for a in arrs]

    return plan


class Pass:
    """One model on one context and one wave: the forward call, its taps and its chunk table."""

    def __init__(self, name, half, wave_kind, dev, lib):
        from beat_this_b200 import synthetic, weights
        from beat_this_b200.engine import Engine

        self.hp = synthetic.model_hparams(name)
        self.half, self.dev = half, dev
        rows = LONG if wave_kind == "long" else weights.ROPE_POSITIONS
        packed = weights.pack_parameters(synthetic.make_state_dict(self.hp, 0), self.hp, rope_positions=rows)
        self.eng = Engine(packed, self.hp, dev, half=half, wave_chunks=4)  # a small workspace: every wave here fits
        self.P = {k: torch.from_numpy(v).to(dev) for k, v in packed.items()}
        self.adt = None if not half else (torch.float16 if self.eng.act_dtype == "f16" else torch.bfloat16)
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(f"{name} {wave_kind}".encode()))
        if wave_kind == "varlen":  # bt_spect2frames on three clips: chunks of 1500, 1500, 712 and 52 frames
            clips = [700, 1800, 40]
            self.fo = np.concatenate([[0], np.cumsum(clips)]).tolist()
            self.spect = (torch.rand(self.fo[-1], 128, generator=g, device=dev) * 7).contiguous()
            plan = _planner(lib)
            chunks = []
            for T, o in zip(clips, self.fo):
                chunks += [(o, T, s, o, lo - s, hi - s, ln) for s, ln, lo, hi in zip(*plan(T))]
            chunks.sort(key=lambda c: -c[6])  # run_chunks: stable, longest first
            self.forward = lambda: self.eng.spect2frames_cat(self.spect, self.fo)
            self.tap = lambda n, cap: self.eng.tap(n, self.spect, self.fo, cap)
        else:
            T, nb = (LONG, 2) if wave_kind == "long" else (1500, 2)
            x = (torch.rand(nb, T, 128, generator=g, device=dev) * 7).contiguous()
            self.spect = x.view(nb * T, 128)
            chunks = [(i * T, T, 0, i * T, 0, T, T) for i in range(nb)]
            self.forward = lambda: self.eng.forward_chunks(x)
            self.tap = lambda n, cap: self.eng.tap_chunks(n, x, cap)
        self.chunks = chunks
        L = chunks[0][6]
        lens = [c[6] for c in chunks]
        self.wave = R.Wave(len(chunks), L, lens if any(n != L for n in lens) else None)
        self.out_frames = self.spect.shape[0]


class Chain:
    """Runs the hook calls of one step.  Registers hold fp32 [rows, cols] tensors: x (the fp32 stream, the step's
    input), xn, gates, qkv, o, h and xb (the 16-bit copy, kept from the step before).  Every output starts as NaN with
    one NaN row past its last, which must survive: a store past the last row or a missing store shows."""

    def __init__(self, ps: Pass, regs: dict):
        self.ps, self.eng, self.P, self.regs = ps, ps.eng, ps.P, regs

    def _param(self, name):
        return None if name is None else self.P[name]

    @staticmethod
    def _nan(rows, cols, dev):
        return torch.full((rows + 1, cols), NAN, device=dev)

    @staticmethod
    def _done(buf, what):
        assert torch.isnan(buf[-1]).all(), f"{what}: stored past its last row"
        out = buf[:-1]
        assert not torch.isnan(out).any(), f"{what}: an element was not stored"
        return out

    def _with_sentinel(self, x):
        buf = self._nan(x.shape[0], x.shape[1], x.device)
        buf[:-1] = x
        return buf

    def run(self, call: R.Call, step: R.Step):
        getattr(self, "_" + call.op)(step, **call.args)

    def _stem(self, step, params):
        ps = self.ps
        L, n = ps.wave.L, ps.wave.nb
        out = torch.full((n * 32 * L * 32 + 32,), NAN, device=ps.dev)
        self.eng.debug_stem(ps.spect, ps.chunks, L, *(self.P[p] for p in params), out)
        assert torch.isnan(out[-32:]).all(), "stem: stored past its output"
        self.regs["x"] = out[:-32].view(-1, 32)

    def _norm(self, step, C, heads, wg, bg):
        x = self.regs["x"]
        M = x.shape[0]
        xn = self._nan(M, C, x.device)
        gates = self._nan(M, heads, x.device) if heads else None
        self.eng.debug_norm(x, xn, M, C, self._param(wg), self._param(bg), gates, heads)
        self.regs["xn"] = self._done(xn, "norm xn")
        if heads:
            self.regs["gates"] = self._done(gates, "norm gates")

    def _gemm(self, step, shape, a, w, bias=None, kind=0, gelu=False, resid=False, out_f32=None, out_act=None,
              resid_epilogue=False, C=0, heads=0, posmode=0, F=1, qscale=1.0):
        A = self.regs[a].contiguous()
        M, N = shape["planes_out"] * shape["L"], shape["N"]
        assert A.numel() == shape["planes_in"] * shape["L"] * shape["lda"], f"gemm: operand {a} has {A.numel()} elements"
        dev = A.device
        if kind == 2:
            o32 = torch.full(((M + 1) * heads,), NAN, device=dev)
        elif out_f32:
            o32 = self._with_sentinel(self.regs["x"]) if resid else self._nan(M, N, dev)
        else:
            o32 = None
        oa = self._nan(M, N, dev) if out_act else None
        rope = (self.P["rope.cos"], self.P["rope.sin"]) if kind == 1 else (None, None)
        self.eng.debug_gemm_full(shape, A, self.P[w], bias=self._param(bias), resid=o32 if resid else None,
                                 out_f32=o32, out_act=oa, rope_cos=rope[0], rope_sin=rope[1],
                                 resid_epilogue=resid_epilogue, kind=kind, gelu=gelu, C=C, heads=heads,
                                 posmode=posmode, F=F, qscale=qscale)
        if kind == 2:
            assert torch.isnan(o32[M * heads :]).all(), "gates gemm: stored past its last row"
            self.regs[out_f32] = o32[: M * heads].view(M, heads)
            assert not torch.isnan(self.regs[out_f32]).any(), "gates gemm: an element was not stored"
        elif out_f32:
            self.regs[out_f32] = self._done(o32, f"gemm {w} fp32 out")
        if out_act:
            self.regs[out_act] = self._done(oa, f"gemm {w} 16-bit out")

    def _fused_qkv(self, step, w, wg, bg, C, L, F, posmode, qscale):
        x = self.regs["x"]
        M, heads, dev = x.shape[0], C // 32, x.device
        cos, sin = self.P["rope.cos"], self.P["rope.sin"]
        qkv, gates = torch.empty(M, 3 * C, device=dev), torch.empty(M, heads, device=dev)
        # bt_debug_fused_qkv takes planes of at most 1500 rows; the kernel works row by row (position m % L or plane
        # (m / L) % F), so longer planes run as pieces of 1500 rows with the RoPE tables advanced to the piece's rows
        for t0 in range(0, L, R.HOOK_ROPE_ROWS):
            t1 = min(L, t0 + R.HOOK_ROPE_ROWS)
            xs = x.view(-1, L, C)[:, t0:t1].reshape(-1, C).contiguous()
            m = xs.shape[0]
            q_out, g_out = self._nan(m, 3 * C, dev), self._nan(m, heads, dev)
            r0 = t0 * 16 if posmode == 0 else 0
            self.eng.debug_fused_qkv(xs, self.P[w], self.P[wg], self.P[bg], cos[r0:], sin[r0:], q_out, g_out, m, C,
                                     t1 - t0, F, posmode, qscale)
            qkv.view(-1, L, 3 * C)[:, t0:t1] = self._done(q_out, "fused qkv").view(-1, t1 - t0, 3 * C)
            gates.view(-1, L, heads)[:, t0:t1] = self._done(g_out, "fused qkv gates").view(-1, t1 - t0, heads)
        self.regs["qkv"], self.regs["gates"] = qkv, gates

    def _qkv(self, C):
        qkv = self.regs["qkv"]
        return [qkv[:, i * C : (i + 1) * C].contiguous() for i in range(3)]

    def _attention_freq(self, step, B, F, L, heads):
        C = heads * 32
        q, k, v = self._qkv(C)
        o = self._nan(q.shape[0], C, q.device)
        self.eng.debug_attention_freq(q, k, v, self.regs["gates"].contiguous(), B, F, out=o)
        self.regs["o"] = self._done(o, "attention_freq")

    def _attention(self, step, seqs, L, heads, key_lens, seqs_per_chunk, qscale):
        C = heads * 32
        q, k, v = self._qkv(C)
        # bt_debug_attention takes q unscaled (fp32: the chain's q scale is 1)
        assert qscale == (R.QSCALE_TIME if self.ps.half else 1.0), f"attention: q scale {qscale}"
        if self.ps.half:
            # the 16-bit hook scales q by its own log2(e) / sqrt(32) before rounding it; the chain's q is the fused
            # or GEMM epilogue's 16-bit q, already scaled by `qscale`.  Dividing by the hook's scale in fp32 gives a
            # value whose fp32 product with that scale rounds back to q (2 fp32 roundings, far inside half a 16-bit
            # ulp), which is checked here before it is relied on
            s = torch.tensor(QSCALE_H16, dtype=torch.float32, device=q.device)
            q = (q / s).contiguous()
            assert torch.equal((q * s).to(self.ps.adt).float(), self.regs["qkv"][:, :C]), "q does not survive the hook's scale"
        o = self._nan(q.shape[0], C, q.device)
        self.eng.debug_attention(q.view(seqs, L, C), k.view(seqs, L, C), v.view(seqs, L, C),
                                 self.regs["gates"].contiguous(), key_lens, seqs_per_chunk, out=o)
        self.regs["o"] = self._done(o, "attention")

    def _fused_ff(self, step, w1, b1, w2, b2, C, wout, xb):
        x = self._with_sentinel(self.regs["x"])
        M = x.shape[0] - 1
        xb_out = self._nan(M, C, x.device) if xb else None
        o = self.regs["o"].contiguous() if wout else None
        self.eng.debug_fused_ff(x, self.P[w1], self.P[b1], self.P[w2], self.P[b2], M, C, o=o, wout=self._param(wout),
                                xb_out=xb_out)
        self.regs["x"] = self._done(x, "fused ff")
        if xb:
            self.regs["xb"] = self._done(xb_out, "fused ff xb")

    def _round16(self, step):
        self.regs["xb"] = self.regs["x"].to(self.ps.adt).float()

    def _zero_tail(self, step, buf, elem_bytes, F, C):
        ps = self.ps
        t = self.regs[buf].contiguous()
        t = t.to(ps.adt) if elem_bytes == 2 else t.clone()
        self.eng.debug_zero_tail(t, ps.chunks, F, ps.wave.L, C)
        self.regs[buf] = t.float()

    def _head(self, step, w, b, sum_head):
        ps = self.ps
        x = self.regs["x"].contiguous()
        beat = torch.full((ps.out_frames,), NAN, device=x.device)
        down = torch.full((ps.out_frames,), NAN, device=x.device)
        self.eng.debug_head(x, x.shape[1], self.P[w], self.P[b], ps.chunks, ps.wave.L, sum_head, beat, down)
        self.regs["logits"] = torch.stack((beat, down))


CONFIGS = [(m, h, w) for w in ("dense", "varlen", "long") for m in ("small0", "final0") for h in (False, True)] + [
    ("final0-nopartial", True, "dense"), ("small0-nosum", True, "dense")]


@pytest.mark.parametrize("model,half,wave_kind", CONFIGS,
                         ids=[f"{m}-{'h16' if h else 'f32'}-{w}" for m, h, w in CONFIGS])
def test_steps_tie_to_hooks(dev, lib_built, model, half, wave_kind):
    ps = Pass(model, half, wave_kind, dev, lib_built)
    eng = ps.eng
    steps = R.forward_steps(ps.hp, half, ps.wave)
    tag = f"{model} {'h16' if half else 'f32'} {wave_kind} (nb={ps.wave.nb}, L={ps.wave.L})"
    failures = []

    # run-to-run determinism, which the tie assumes
    b1, d1 = ps.forward()
    b2, d2 = ps.forward()
    torch.cuda.synchronize()
    if not (torch.equal(bits(b1), bits(b2)) and torch.equal(bits(d1), bits(d2))):
        failures.append("two forward calls give different logits")

    # coverage: the production chains, by the launch each call stands for, are the launch profile of one call
    eng.profile_enable(True)
    eng.profile_reset()
    ps.forward()
    prof = eng.profile_results()
    eng.profile_enable(False)
    launched = collections.Counter({k: v[1] for k, v in prof.items()})
    chained = collections.Counter(c.prod for s in steps if not s.tap_mode for c in s.chain)
    if launched != chained:
        failures.append(f"chains {dict(chained - launched)} not launched; launches {dict(launched - chained)} in no chain")
    want = [s.name for s in steps if not s.tap_mode]
    assert want[-1] == "logits" and want[:-1] == [n for n in R.tap_names(ps.hp) if n in set(want)]

    taps = {}

    def tap(name):
        if name not in taps:
            cap = ps.wave.nb * ps.wave.L * 2048
            t, _ = ps.tap(name, cap)
            assert t.numel() > 0, f"tap {name} is empty"
            taps[name] = t.clone()
        return taps[name]

    regs, before, tied = {}, {}, []
    for s in steps:
        try:
            if s.input != "spect":
                regs["x"] = tap(s.input).view(-1, s.C)
            before[s.name, s.tap_mode] = dict(regs)
            got = _run_chain(ps, s, regs)
            want_t = torch.stack((b1, d1)) if s.name == "logits" else tap(s.name)
            assert want_t.numel() == got.numel(), f"tap has {want_t.numel()} elements, the chain {got.numel()}"
            diff, mx = _differ(got, want_t)
            print(f"{tag} {s.name:9s} {s.kind:9s}{' (tap mode)' if s.tap_mode else '':11s} "
                  f"{'bitwise tie OK' if diff == 0 else f'{diff} elements differ, max {mx:.3e}'}")
            assert diff == 0, f"{diff} of {got.numel()} elements differ from the chain (max abs {mx:.3e})"
            tied.append(s.name)
        except AssertionError as e:
            failures.append(f"{s.name}{' (tap mode)' if s.tap_mode else ''}: {str(e).splitlines()[0]}")
    if len(tied) != len(steps) and not failures:
        failures.append("not every step was tied")

    # strength: one wrong but valid argument per kind of step must break its tie
    for what, s, mutated in R.mutations(ps.half, ps.wave, steps):
        try:
            got = _run_chain(ps, mutated, dict(before[s.name, s.tap_mode]))
            diff, mx = _differ(got, torch.stack((b1, d1)) if s.name == "logits" else tap(s.name))
            print(f"{tag} {s.name:9s} with {what}: {diff / got.numel():.1%} of the elements differ, max {mx:.3e}")
            assert diff > 0, f"{what} leaves the step unchanged"
        except AssertionError as e:
            failures.append(f"{s.name} with {what}: {str(e).splitlines()[0]}")
    for f in failures:
        print(f"FAILED {tag}: {f}")
    ps.eng.close()
    assert not failures, f"{tag}: {len(failures)} failures:\n" + "\n".join(failures)


def _run_chain(ps, step, regs):
    chain = Chain(ps, regs)
    for call in step.chain:
        chain.run(call, step)
    return regs[step.out]


def _differ(got, want):
    """(elements whose bits differ, max abs difference) of two fp32 tensors of the same size."""
    got, want = got.contiguous().view(-1), want.contiguous().view(-1)
    return int((bits(got) != bits(want)).sum()), (got.double() - want.double()).abs().max().item()
