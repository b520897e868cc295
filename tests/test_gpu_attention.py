"""GPU unit tests (pytest -m gpu) of the attention kernels against the float64 restatements and bounds of
tests/attention_reference.py: attn_time_kernel (16-bit context) and attn_time_simt_kernel (fp32) through
bt_debug_attention, attn_freq_mma_kernel<F> (16-bit) and attn_freq_kernel<F> (fp32) through bt_debug_attention_freq.

Every case runs each input family that applies to it, in both contexts.  The output buffer starts as NaN and has one
sentinel row past M that the kernel must not write; every row < M must be finite (chunk rows in [len, L) too: the
kernel computes them from real keys) and within its elementwise bound, and a second launch must give the same bits.
Each case prints its worst error as a fraction of its bound, and each (path, family) its worst over all cases; all
cases run, and the failures are listed together at the end.  On the 16-bit paths the stored value may sit on the
other fp16 neighbour wherever the fp32 error can reach a rounding midpoint, so that ratio is close to a count of ulps;
each case also prints the fp32-level ratio |got - o| / (err + half an ulp of got), o and err the value and bound
before the store: the headroom of the fp32 arithmetic under its derived bound."""
import zlib

import pytest
import torch

import attention_reference as R
from numerics import ulp16
from support import act_dtype, dev, launch_twice  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(3000)]

@pytest.fixture(scope="module")
def engines(lib_built, dev):
    """Weight-less contexts: {False: fp32, True: 16-bit}."""
    from beat_this_b200.engine import Engine

    return {half: Engine(None, None, dev, half=half) for half in (False, True)}


class Family:
    """The worst error-to-bound ratio of one (path, input family) over its cases, and its failures."""

    def __init__(self, name):
        self.name, self.worst, self.worst32, self.failures, self.cases = name, 0.0, 0.0, [], 0

    def run(self, case_id, fn, *args):
        self.cases += 1
        try:
            fn(self, case_id, *args)
        except AssertionError as e:
            self.failures.append(f"{self.name} {case_id}: {str(e).splitlines()[0]}")

    def check(self, case_id, got, res, dt):
        """res: (ref, bound, o, err) of attention_reference; dt: the stored 16-bit type (None: fp32)."""
        ref, bound, o, e32 = res
        assert torch.isfinite(got).all(), "non-finite values in rows < M"
        err = (got - ref).abs()
        ratio = torch.where(err == 0, 0.0, err / bound).max().item()  # a bound of 0 asks for the exact value
        half_ulp = 0.0 if dt is None else ulp16(got, dt) / 2
        r32 = ((got - o).abs() / (e32 + half_ulp)).max().item()
        print(f"{self.name} {case_id}: max {err.max().item():.3e} = {ratio:.3f} of its bound; fp32 level {r32:.3f}")
        self.worst, self.worst32 = max(self.worst, ratio), max(self.worst32, r32)
        assert ratio <= 1, f"off by {ratio:.2f} x its bound"


def _finish(families):
    failures = []
    for fam in families.values():
        print(f"{fam.name}: worst error {fam.worst:.3f} of its bound, fp32 level {fam.worst32:.3f}, over {fam.cases} cases")
        failures += fam.failures
    total = sum(f.cases for f in families.values())
    assert not failures, f"{len(failures)} of {total} attention cases failed:\n" + "\n".join(failures)


def _time_case(fam, case_id, eng, case, q, k, v, gates):
    half = eng.half
    M, C = case.seqs * case.L, 32 * case.heads
    got = launch_twice(lambda out: eng.debug_attention(q, k, v, gates, case.key_lens, case.spc, out=out), M, C, q.device)
    lens = torch.tensor(case.lens(), device=q.device)
    dt = act_dtype(eng) if half else None
    res = R.time_ref(q.double(), k.double(), v.double(), gates.double(), lens, "tc" if half else "simt", dt)
    fam.check(case_id, got, [t.reshape(M, C) for t in res], dt)


def _freq_case(fam, case_id, eng, case, q, k, v, gates):
    half = eng.half
    M, C = case.B * case.F * case.L, 32 * case.heads
    got = launch_twice(lambda out: eng.debug_attention_freq(q, k, v, gates, case.B, case.F, out=out), M, C, q.device)
    dt = act_dtype(eng) if half else None
    res = R.freq_ref(q.double(), k.double(), v.double(), gates.double(), case.B, case.F, "tc" if half else "simt", dt)
    fam.check(case_id, got, res, dt)


def _path(half, what):
    return f"{what} {'tensor-core' if half else 'SIMT'}"


@pytest.mark.parametrize("half", [False, True])
def test_time_attention(engines, dev, half):
    eng = engines[half]
    families = {}
    for case in R.time_cases():
        for family in R.time_families(case):
            fam = families.setdefault(family, Family(f"{_path(half, 'time')} {family}"))
            g = torch.Generator(device=dev).manual_seed(zlib.crc32(f"{case.id} {family}".encode()))
            fam.run(case.id, _time_case, eng, case, *R.time_inputs(case, family, g, dev))
    _finish(families)


@pytest.mark.parametrize("half", [False, True])
def test_freq_attention(engines, dev, half):
    eng = engines[half]
    families = {}
    for case in R.freq_cases("tc" if half else "simt"):
        for family in R.freq_families(case):
            fam = families.setdefault(family, Family(f"{_path(half, 'freq')} {family}"))
            g = torch.Generator(device=dev).manual_seed(zlib.crc32(f"{case.id} {family}".encode()))
            fam.run(case.id, _freq_case, eng, case, *R.freq_inputs(case, family, g, dev))
    _finish(families)


@pytest.fixture(scope="module")
def production():
    return R.production_inputs()


@pytest.mark.parametrize("half", [False, True])
def test_production_activations(engines, dev, half, production):
    """final0's b0.attnF, b0.attnT and main layer 0 on the oracle's q, k, v and gates of the stage-parity input."""
    eng = engines[half]
    fam = Family(f"{'16-bit' if half else 'fp32'} production")
    for name, (case, tensors) in production.items():
        q, k, v, gates = (t.to(dev) for t in tensors)
        fn = _freq_case if isinstance(case, R.FreqCase) else _time_case
        fam.run(f"{name} ({case.id})", fn, eng, case, q, k, v, gates)
    _finish({"production": fam})


def test_hooks_reject_a_short_output(engines, dev):
    """o_count below M * C is refused before anything is enqueued, in both contexts."""
    from ctypes import c_void_p

    from beat_this_b200._lib import BTError, check

    for half, eng in engines.items():
        before = eng.lib.bt_launch_count(eng.ctx)
        x = torch.zeros(2 * 13 * 64 + 1, device=dev)
        p = c_void_p(x.data_ptr())
        M, C = 2 * 13, 64
        with pytest.raises(BTError, match="error -1"):
            check(eng.lib, eng.ctx, eng.lib.bt_debug_attention(eng.ctx, p, p, p, p, p, M * C - 1, 2, 13, 2, None, 1, None))
        F, L, H = 16, 3, 2
        with pytest.raises(BTError, match="error -1"):
            check(eng.lib, eng.ctx, eng.lib.bt_debug_attention_freq(eng.ctx, p, p, p, p, p, F * L * 32 * H - 1, 1, F, L, H,
                                                                    None))
        with pytest.raises(AssertionError, match="elements"):  # the wrappers check the sizes the hooks cannot see
            q = torch.zeros(2, 13, 64, device=dev)
            eng.debug_attention(q, q, q, out=torch.zeros(2 * 13 * 64 - 1, device=dev))
        assert eng.lib.bt_launch_count(eng.ctx) == before, "a rejected call launched"


@pytest.mark.parametrize("path", list(R.PATHS))
def test_hooks_launch_the_listed_kernels(engines, dev, path):
    """Each context's hooks launch the kernels attention_reference.PATHS names for it (the CPU test ties that table to
    the instantiations in the library): one time case and one frequency case per F, under the profiler."""
    half, time_k, freq_k = R.PATHS[path]
    eng = engines[half]
    g = torch.Generator(device=dev).manual_seed(0)
    fcases = {c.F: c for c in R.freq_cases(path) if c.L == 5 and c.B == 1}
    tcase = R.TimeCase(2, 70, 2, (70, 13), 1)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.debug_attention(*R.time_inputs(tcase, "random", g, dev), tcase.key_lens, tcase.spc)
        for c in fcases.values():
            eng.debug_attention_freq(*R.freq_inputs(c, "random", g, dev), c.B, c.F)
        torch.cuda.synchronize(dev)
    names = {e.name for e in prof.events() if "attn_" in e.name}
    print(f"{path}: {sorted(names)}")
    want = {f"bt::{time_k}("} | {f"bt::{freq_k}<{F}>(" for F in fcases}
    got = {w for w in want if any(w in n for n in names)}
    assert got == want and len(names) == len(want), f"launched {sorted(names)}, expected {sorted(want)}"
    assert {(freq_k, F) for F in fcases} | {(time_k, 0)} == R.launched_kernels(path)
