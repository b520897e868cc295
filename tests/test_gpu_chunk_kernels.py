"""GPU unit tests (pytest -m gpu) of the kernels that read the chunk table, against the float64 restatements and
bounds of tests/chunk_kernels_reference.py: stem_kernel (bt_debug_stem), zero_tail_kernel (bt_debug_zero_tail) and
head_kernel (bt_debug_head).

Tables: the planner's chunks (bt_plan_chunking_max) of clips at the planner's edge lengths for several chunkings, all
chunks of a call in one mixed-length wave sorted longest first as run_chunks sorts them, and hand-made edges.  Clips
lie back to back with NaN guard frames between them, in the spectrogram and in the outputs, so that a read or write
outside a clip shows.  Outputs start as NaN (a bit pattern for zero_tail); every element must be within its bound, no
other element may change, and a second run must give the same bits.  Each family prints its worst error as a fraction
of its bound; all cases run, and the failures are listed together at the end."""
import math
import zlib
from ctypes import c_void_p

import numpy as np
import pytest
import torch

import chunk_kernels_reference as R
from support import bits, dev  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

NAN = float("nan")
TAIL = 1024  # guard elements after every output


@pytest.fixture(scope="module")
def engines(lib_built, dev):
    """Weight-less contexts: {False: fp32, True: 16-bit}."""
    from beat_this_b200.engine import Engine

    return {half: Engine(None, None, dev, half=half) for half in (False, True)}


class Family:
    """The worst error-to-bound ratio of a family of cases, and its failures."""

    def __init__(self, name):
        self.name, self.worst, self.failures, self.cases = name, 0.0, [], 0

    def run(self, case_id, fn, *args):
        self.cases += 1
        try:
            fn(self, case_id, *args)
        except AssertionError as e:
            self.failures.append(f"{case_id}: {str(e).splitlines()[0]}")

    def check(self, case_id, what, got, ref, bound):
        got = got.double()
        err = (got - ref).abs()
        ratio = torch.where(err == 0, 0.0, err / bound).nan_to_num(nan=math.inf).max().item()
        self.worst = max(self.worst, ratio)
        assert torch.isfinite(got).all(), f"{what}: non-finite values"
        assert ratio <= 1, f"{what} off by {ratio:.3g} x its bound (max error {err.max().item():.3e})"

    def finish(self):
        print(f"{self.name}: worst error {self.worst:.3f} of its bound over {self.cases} cases")
        for f in self.failures:
            print(f"FAILED {self.name} {f}")
        assert not self.failures, f"{len(self.failures)} of {self.cases} {self.name} cases failed:\n" + "\n".join(self.failures)


# ------------------------------------------------------------------------------ tables
PLANS = [(1500, 6, "keep_first"), (64, 6, "keep_last"), (13, 6, "keep_first"), (1000, 0, "keep_first"),
         (1500, 100, "keep_last"), (8000, 6, "keep_first")]


def _planner(lib, chunk, border, mode):
    from beat_this_b200._lib import OVERLAP_MODES, bt_chunking, i64_array

    ck = bt_chunking(chunk, border, OVERLAP_MODES[mode])
    mx = max(chunk, 1500)

    def plan(T):
        n = lib.bt_plan_chunking_max(T, ck, mx, None, None, None, None, 0)
        arrs = [i64_array([0] * n) for _ in range(4)]
        assert lib.bt_plan_chunking_max(T, ck, mx, *arrs, n) == n
        return [list(a) for a in arrs]

    return plan


def _edge_tables():
    """(name, chunks, L, frames): hand-made chunks.  Tuples are (frame_base, T, start, out_base, write_lo, write_hi,
    len); clips start at 3 and are separated by guard frames."""
    return [
        ("start -749", [(3, 600, -749, 3, 749, 1349, 1500), (606, 2000, -749, 606, 749, 1500, 1500)], 1500, 2610),
        ("past the clip's end", [(3, 900, 500, 3, 0, 400, 1500), (906, 50, 20, 906, 0, 30, 129)], 1500, 960),
        ("T = len = L = 1", [(3, 1, 0, 3, 0, 1, 1)], 1, 6),
        ("L = 129", [(3, 300, -3, 3, 3, 126, 129), (306, 200, 150, 306, 0, 50, 64), (509, 5, -1, 509, 1, 6, 7)], 129, 517),
        ("L = 24000", [(3, 30000, -6, 3, 6, 24000, 24000), (30006, 1000, 10, 30006, 0, 990, 990)], 24000, 31010),
        ("empty owned ranges", [(3, 40, -6, 3, 6, 6, 52), (46, 40, 0, 46, 40, 40, 40), (89, 40, 20, 89, 2, 20, 52)], 52, 132),
    ]


def _tables(lib):
    out = []
    for chunk, border, mode in PLANS:
        chunks, L, frames, offs = R.wave(R.sweep_lengths(chunk, border), _planner(lib, chunk, border, mode))
        out.append((f"plan {chunk}/{border}/{mode}", chunks, L, frames, True))
    return out + [(n, c, L, f, False) for n, c, L, f in _edge_tables()]


def _clip_mask(chunks, frames, dev):
    inside = torch.zeros(frames, dtype=torch.bool, device=dev)
    for fb, T, *_ in chunks:
        inside[fb : fb + T] = True
    return inside


def _spect(chunks, frames, g, dev, lo=0.0, hi=7.0):
    x = torch.rand(frames, 128, generator=g, device=dev) * (hi - lo) + lo
    x[~_clip_mask(chunks, frames, dev)] = NAN
    return x.contiguous()


# ------------------------------------------------------------------------------ stem
def _stem_case(fam, case_id, eng, spect, chunks, L, params):
    n = len(chunks)
    size = n * 32 * L * 32
    runs = []
    for _ in range(2):
        out = torch.full((size + TAIL,), NAN, device=spect.device)
        eng.debug_stem(spect, chunks, L, *params, out)
        runs.append(out)
    assert torch.equal(bits(runs[0]), bits(runs[1])), "not deterministic"
    out = runs[0]
    assert torch.isnan(out[size:]).all(), "stored past n_chunks * 32 * L * 32"
    ref, bound = R.stem_ref(spect.double(), chunks, L, *(p.double() for p in params))
    fam.check(case_id, "stem", out[:size].view(n, 32, L, 32), ref, bound)


def _stem_params(g, dev, kind):
    r = lambda *s: torch.randn(*s, generator=g, device=dev)
    if kind == "padding":  # scale 0, large distinct shifts: every output shows which padding each tap took
        return [torch.zeros(128, device=dev), 100 + 10 * torch.arange(128.0, device=dev), r(32, 12) * 0.01, r(32)]
    return [0.5 + torch.rand(128, generator=g, device=dev), r(128) * 2, r(32, 12) * 0.4, r(32) * 0.3]


def test_stem(engines, dev, lib_built):
    eng = engines[False]
    fam = Family("stem")
    for name, chunks, L, frames, _ in _tables(lib_built):
        for kind in ("random", "padding"):
            case_id = f"{name} {kind} (L={L}, {len(chunks)} chunks)"
            g = torch.Generator(device=dev).manual_seed(zlib.crc32(case_id.encode()))
            fam.run(case_id, _stem_case, eng, _spect(chunks, frames, g, dev), chunks, L, _stem_params(g, dev, kind))
    # GELU sweep: identity BN1d, weight 1 on (df = c % 4, dt = 1), bias 0: a is the input, a dense grid over [-12, 12]
    L = 24000
    grid = torch.linspace(-12, 12, L * 128 - 2, device=dev)
    sweep = torch.cat([grid, torch.tensor([0.0, -0.0], device=dev)]).view(L, 128).contiguous()
    w = torch.zeros(32, 4, 3, device=dev)
    w[torch.arange(32), torch.arange(32) % 4, 1] = 1.0
    ident = [torch.ones(128, device=dev), torch.zeros(128, device=dev), w.view(32, 12).contiguous(), torch.zeros(32, device=dev)]
    fam.run("gelu sweep", _stem_case, eng, sweep, [(0, L, 0, 0, 0, L, L)], L, ident)
    # production weights on the log-mel of synthetic clips, chunked 1500 / 6 / keep_first
    from beat_this_b200 import synthetic, weights
    from beat_this_b200.engine import Engine

    mel = Engine.mel_only(dev)
    specs = mel.logmel([synthetic.synth_clip(i, s) for i, s in ((0, 10.0), (1, 35.0))])
    chunks, L, frames, offs = R.wave([s.shape[0] for s in specs], _planner(lib_built, 1500, 6, "keep_first"))
    spect = torch.full((frames, 128), NAN, device=dev)
    for s, o in zip(specs, offs):
        spect[o : o + s.shape[0]] = s
    for name in ("small0", "final0"):
        hp = synthetic.model_hparams(name)
        packed = weights.pack_parameters(synthetic.make_state_dict(hp, 0), hp)
        params = [torch.from_numpy(packed[k]).to(dev) for k in ("stem.bn1_scale", "stem.bn1_shift", "stem.w", "stem.bias")]
        fam.run(f"{name} weights on log-mel", _stem_case, eng, spect, chunks, L, params)
    fam.finish()


# ------------------------------------------------------------------------------ head
def _head_case(fam, case_id, eng, x, w, b, chunks, L, sum_head, frames, planner):
    D = x.shape[-1]
    runs = []
    for _ in range(2):
        beat = torch.full((frames,), NAN, device=x.device)
        down = torch.full((frames,), NAN, device=x.device)
        eng.debug_head(x, D, w, b, chunks, L, sum_head, beat, down)
        runs.append((beat, down))
    (beat, down), (beat2, down2) = runs
    assert torch.equal(bits(beat), bits(beat2)) and torch.equal(bits(down), bits(down2)), "not deterministic"
    rb, rd, eb, ed = R.head_ref(x.double(), w.double(), b.double(), sum_head)
    owned = R.head_scatter(chunks, L, rb, frames)[1]
    if planner:  # the planner's ranges tile every clip
        assert torch.equal(owned > 0, _clip_mask(chunks, frames, x.device)) and owned.max() <= 1, "not owned exactly once"
    nan_bits = bits(torch.full((1,), NAN, device=x.device))
    for name, got, ref, bnd in (("beat", beat, rb, eb), ("down", down, rd, ed)):
        assert (bits(got)[owned == 0] == nan_bits).all(), f"{name}: a frame no chunk owns was written"
        fam.check(case_id, name, got[owned > 0], R.head_scatter(chunks, L, ref, frames)[0][owned > 0],
                  R.head_scatter(chunks, L, bnd, frames)[0][owned > 0])
    zero = x.view(-1, D).abs().amax(-1) == 0  # zero rows: exactly the bias
    if zero.any():
        bias_beat = (b[0] + b[1]) if sum_head else b[0]
        rows_beat = R.head_scatter(chunks, L, torch.where(zero.view(len(chunks), L), 1.0, 0.0).double(), frames)[0]
        sel = (rows_beat == 1) & (owned > 0)
        assert torch.equal(beat[sel], bias_beat.expand(int(sel.sum()))), "beat of a zero row is not the bias"
        assert torch.equal(down[sel], b[1].expand(int(sel.sum()))), "down of a zero row is not the bias"


def _head_rows(n, L, D, g, dev, scale):
    """Random rows, with every 7th row zero, every 7th + 2 below the 1e-12 clamp, every 7th + 4 at 1e3 scale."""
    x = torch.randn(n, L, D, generator=g, device=dev) * scale
    x[:, 0::7] = 0.0
    x[:, 2::7] *= 1e-15
    x[:, 4::7] *= 1e3
    return x.contiguous()


def test_head(engines, dev, lib_built):
    eng = engines[False]
    fam = Family("head")
    for i, (name, chunks, L, frames, planner) in enumerate(_tables(lib_built)):
        combos = [(D, sh) for D in (64, 128, 512, 1024) for sh in (0, 1)] if L <= 129 else [((64, 128, 512, 1024)[i % 4], i % 2)]
        for D, sh in combos:
            case_id = f"{name} D={D} sum_head={sh} (L={L}, {len(chunks)} chunks)"
            g = torch.Generator(device=dev).manual_seed(zlib.crc32(case_id.encode()))
            x = _head_rows(len(chunks), L, D, g, dev, 1.0)
            w = (torch.randn(2, D, generator=g, device=dev) * 0.4 * math.sqrt(D)).contiguous()
            b = torch.tensor([0.75, -1.5], device=dev)
            fam.run(case_id, _head_case, eng, x, w, b, chunks, L, sh, frames, planner)
    # production weights on the oracle's pre-head activations (final0 and its Head variant)
    from beat_this_b200 import synthetic, weights
    from oracle import beat_this_oracle as O

    for name in ("final0", "final0-nosum"):
        hp = synthetic.model_hparams(name)
        sd = synthetic.make_state_dict(hp, 0)
        packed = weights.pack_parameters(sd, hp)
        taps = {}
        with torch.inference_mode():
            O.forward(sd, torch.rand(2, 150, 128, generator=torch.Generator().manual_seed(9)) * 7, taps, sum_head=hp["sum_head"])
        x = taps["l5.ff"].to(dev).float().contiguous()
        D = hp["transformer_dim"]
        chunks = [(3, 150, 0, 3, 0, 150, 150), (156, 140, -6, 156, 6, 146, 150)]
        w, b = (torch.from_numpy(packed[k]).to(dev) for k in ("head.w", "head.b"))
        fam.run(f"{name} weights", _head_case, eng, x, w, b, chunks, 150, hp["sum_head"], 299, False)
    fam.finish()


# ------------------------------------------------------------------------------ zero_tail
def _zero_tail_case(fam, case_id, eng, chunks, F, L, C, dtype, g):
    n = len(chunks)
    size = n * F * L * C
    raw = torch.randint(1, 2**15 - 1, (size + TAIL,), generator=g, device=g.device, dtype=torch.int32)
    base = (raw if dtype == torch.float32 else raw.to(torch.int16)).view(dtype)
    runs = []
    for _ in range(2):
        buf = base.clone()
        eng.debug_zero_tail(buf, chunks, F, L, C)
        runs.append(buf)
    assert torch.equal(bits(runs[0]), bits(runs[1])), "not deterministic"
    buf = runs[0]
    assert torch.equal(bits(buf[size:]), bits(base[size:])), "changed past n_chunks * F * L * C"
    ref = R.zero_tail_ref(base[:size].view(n, F, L, C), chunks, F, L, C)
    bad = int((bits(buf[:size]) != bits(ref.reshape(-1))).sum())
    assert bad == 0, f"{bad} elements differ from the exact result"


def test_zero_tail(engines, dev, lib_built):
    eng = engines[False]
    fam = Family("zero_tail")
    for name, chunks, L, frames, _ in _tables(lib_built):
        for F, C in ((32, 32), (16, 64), (8, 128)):
            for dtype in (torch.float32, torch.float16):
                case_id = f"{name} F={F} C={C} {dtype} (L={L}, {len(chunks)} chunks)"
                g = torch.Generator(device=dev).manual_seed(zlib.crc32(case_id.encode()))
                fam.run(case_id, _zero_tail_case, eng, chunks, F, L, C, dtype, g)
    fam.finish()


# ------------------------------------------------------------------------------ the hooks are the production kernels
@pytest.mark.parametrize("half", [False, True])
def test_hooks_reproduce_the_forward_pass(dev, lib_built, half):
    """One single-wave bt_spect2frames call on three clips (chunks of 1500, 1500, 700 and 40 frames): its stem tap is
    bt_debug_stem on the same spectrogram, packed parameters and chunk table, and its logits are bt_debug_head on its
    last layer's tap, bitwise."""
    from beat_this_b200 import synthetic, weights
    from beat_this_b200.engine import Engine

    hp = synthetic.model_hparams("small0")
    packed = weights.pack_parameters(synthetic.make_state_dict(hp, 0), hp)
    eng = Engine(packed, hp, dev, half=half)
    clips = [700, 1800, 40]
    fo = np.concatenate([[0], np.cumsum(clips)]).tolist()
    spect = (torch.rand(fo[-1], 128, generator=torch.Generator(device=dev).manual_seed(4), device=dev) * 7).contiguous()
    plan = _planner(lib_built, 1500, 6, "keep_first")
    chunks = []
    for T, o in zip(clips, fo):
        chunks += [(o, T, s, o, lo - s, hi - s, ln) for s, ln, lo, hi in zip(*plan(T))]
    chunks.sort(key=lambda c: -c[6])  # run_chunks: stable, longest first
    n, L, D = len(chunks), chunks[0][6], hp["transformer_dim"]
    P = {k: torch.from_numpy(v).to(dev) for k, v in packed.items()}
    stem_tap, (beat, down) = eng.tap("stem", spect, fo, n * 32 * L * 32)
    out = torch.full((n * 32 * L * 32,), NAN, device=dev)
    eng.debug_stem(spect, chunks, L, P["stem.bn1_scale"], P["stem.bn1_shift"], P["stem.w"], P["stem.bias"], out)
    assert stem_tap.numel() == out.numel() and torch.equal(bits(stem_tap), bits(out)), "stem tap != bt_debug_stem"
    x, (beat2, down2) = eng.tap(f"l{hp['n_layers'] - 1}.ff", spect, fo, n * L * D)
    assert torch.equal(bits(beat), bits(beat2)) and torch.equal(bits(down), bits(down2))
    hb, hd = torch.full_like(beat, NAN), torch.full_like(down, NAN)
    eng.debug_head(x.contiguous(), D, P["head.w"], P["head.b"], chunks, L, hp["sum_head"], hb, hd)
    assert torch.equal(bits(hb), bits(beat)) and torch.equal(bits(hd), bits(down)), "logits != bt_debug_head"


# ------------------------------------------------------------------------------ launches and refusals
def test_one_launch_per_call_and_refusals(engines, dev):
    from beat_this_b200._lib import BTError, bt_debug_chunk

    eng = engines[True]
    L, D = 16, 64
    ok = [(3, 10, -2, 3, 2, 12, 14)]
    spect = torch.zeros(16, 128, device=dev)
    p = [torch.ones(128, device=dev), torch.zeros(128, device=dev), torch.zeros(32, 12, device=dev), torch.zeros(32, device=dev)]
    out = torch.zeros(32 * L * 32, device=dev)
    buf = torch.zeros(2 * 4 * L * 32, device=dev)
    x, w, b = torch.zeros(2 * L * D, device=dev), torch.zeros(2 * D, device=dev), torch.zeros(2, device=dev)
    beat, down = torch.zeros(16, device=dev), torch.zeros(16, device=dev)
    big = torch.zeros(1 << 14, device=dev)  # large enough for every head geometry below

    eng.profile_enable(True)
    eng.profile_reset()
    before = eng.launches
    eng.debug_stem(spect, ok, L, *p, out)
    eng.debug_zero_tail(buf, ok + ok, 4, L, 32)
    eng.debug_head(x, D, w, b, ok + [(3, 10, 0, 3, 0, 0, 1)], L, 1, beat, down)
    prof = eng.profile_results()
    eng.profile_enable(False)
    assert eng.launches == before + 3
    assert {k: v[1] for k, v in prof.items()} == {"stem": 1, "zero_tail": 1, "head": 1}, prof

    def chunk(**kw):
        c = dict(zip(R.FIELDS, ok[0]))
        c.update(kw)
        return [tuple(c[f] for f in R.FIELDS)]

    bad = [
        lambda: eng.debug_stem(spect, [], L, *p, out),  # no chunks
        lambda: eng.debug_stem(spect, ok * 65536, L, *p, torch.zeros(1, device=dev)),  # grid.z
        lambda: eng.debug_stem(spect, ok, 0, *p, out),
        lambda: eng.debug_stem(spect, chunk(len=15), 384001, *p, out),
        lambda: eng.debug_stem(spect, chunk(T=0), L, *p, out),
        lambda: eng.debug_stem(spect, chunk(len=0), L, *p, out),
        lambda: eng.debug_stem(spect, chunk(len=L + 1), L, *p, out),
        lambda: eng.debug_stem(spect, chunk(frame_base=7), L, *p, out),  # clip [7, 17) past 16 frames
        lambda: eng.debug_stem(spect, chunk(frame_base=-1), L, *p, out),
        lambda: eng.debug_stem(spect, ok, L, *p, out[1:]),  # out too small and unaligned
        lambda: eng.debug_stem(spect, ok, L, *p, torch.zeros(32 * L * 32 + 4, device=dev)[1:]),  # unaligned out
        lambda: eng.debug_stem(spect.view(-1)[1:2049], ok, L, *p, out),  # spect not 16-byte aligned
        lambda: eng.debug_zero_tail(buf, ok, 4, L, 6),  # C * 4 bytes not a multiple of 16
        lambda: eng.debug_zero_tail(buf, chunk(len=0), 4, L, 32),
        lambda: eng.debug_zero_tail(buf, chunk(len=L + 1), 4, L, 32),
        lambda: eng.debug_zero_tail(buf, ok * 3, 4, L, 32),  # buffer smaller than 3 chunks
        lambda: eng.debug_zero_tail(buf, ok, 0, L, 32),
        lambda: eng.debug_zero_tail(buf[1:], ok, 4, L, 32),  # unaligned
        lambda: eng.debug_head(big, 32, big, b, ok, L, 1, beat, down),
        lambda: eng.debug_head(big, 96, big, b, ok, L, 1, beat, down),
        lambda: eng.debug_head(torch.zeros(2048, device=dev), 2048, torch.zeros(4096, device=dev), b, ok, 1, 1, beat, down),
        lambda: eng.debug_head(x, D, w, b, chunk(write_lo=-1), L, 1, beat, down),
        lambda: eng.debug_head(x, D, w, b, chunk(write_hi=L + 1), L, 1, beat, down),
        lambda: eng.debug_head(x, D, w, b, chunk(write_lo=5, write_hi=4), L, 1, beat, down),
        lambda: eng.debug_head(x, D, w, b, chunk(start=-6, write_lo=2), L, 1, beat, down),  # frame 3 - 6 + 2 < 0
        lambda: eng.debug_head(x, D, w, b, chunk(out_base=8), L, 1, beat, down),  # frames 8 .. 17, 16 outputs
        lambda: eng.debug_head(x, D, w, b, ok, L, 1, beat[:12], down[:12]),  # last owned frame 12 of 12 outputs
    ]
    before = {h: e.launches for h, e in engines.items()}
    for call in bad:
        with pytest.raises(BTError, match="error -1"):
            call()
    code = eng.lib.bt_debug_zero_tail(eng.ctx, c_void_p(buf.data_ptr()), 8, (bt_debug_chunk * 1)(bt_debug_chunk(*ok[0])),
                                      1, 4, L, 32, buf.numel() * 4, eng._stream())
    assert code == -1  # elem_bytes 8
    assert {h: e.launches for h, e in engines.items()} == before, "a refused call launched"
