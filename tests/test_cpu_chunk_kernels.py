"""CPU tests (no GPU) of tests/chunk_kernels_reference.py, the float64 restatements and bounds of stem_kernel,
head_kernel and zero_tail_kernel:
- the restatements are the reference's blocks (oracle.forward's stem, and its final norm + head on its own pre-head
  activations) on the packed parameters of the synthetic checkpoints;
- gelu_fast's erf, emulated with rcp / ex2 off by their stated errors, stays within E_ERF on 10^7 points;
- fp32 emulations of the kernels stay within the bounds on every family of inputs, and each of the mistakes the GPU
  tests are meant to catch takes the emulation outside them on at least one family."""
import math

import numpy as np
import pytest
import torch
from scipy.special import erf

import chunk_kernels_reference as R


def _packed(name):
    from beat_this_b200 import synthetic, weights

    hp = synthetic.model_hparams(name)
    sd = synthetic.make_state_dict(hp, 0)
    return hp, sd, {k: torch.from_numpy(v).double() for k, v in weights.pack_parameters(sd, hp).items()}


def _stem_params(packed):
    return [packed[k] for k in ("stem.bn1_scale", "stem.bn1_shift", "stem.w", "stem.bias")]


@pytest.mark.parametrize("name", ["small0", "final0"])
def test_stem_restatement_is_the_oracle_stem(name):
    """A chunk that starts 5 frames before its clip and runs 4 past its end: the oracle sees the chunk as split_piece
    pads it (zeros before BN1d); the restatement gathers it from the clip.  They differ by the fp32 rounding of the
    folded parameters only: each of s, h, w, bias is u relative off, so a moves by at most
    u (|bias| + 3 sum |w| (|v s| + |h|)), and the output by GELU_SLOPE times that."""
    from oracle import beat_this_oracle as O

    hp, sd, packed = _packed(name)
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    T, L, start = 40, 49, -5
    clip = torch.rand(T, 128, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 7
    chunk = torch.zeros(L, 128, dtype=torch.float64)
    chunk[-start : -start + T] = clip
    taps = {}
    O.forward(sd64, chunk[None], taps)
    s, h, w, bias = _stem_params(packed)
    ref, _ = R.stem_ref(clip, [(0, T, start, 0, 0, L, L)], L, s, h, w, bias)
    xp = torch.nn.functional.pad((chunk * s).abs() + h.abs(), (0, 0, 1, 1))
    cols = torch.stack([xp[dt : dt + L] for dt in range(3)], dim=-1).view(L, 32, 4, 3)
    tol = R.GELU_SLOPE * R.U * (bias.abs() + 3 * torch.einsum("lfdt,cdt->flc", cols, w.view(32, 4, 3).abs())) * 1.01
    err = (ref[0] - taps["stem"][0]).abs()
    print(f"{name}: stem restatement vs oracle {err.max().item():.2e}, {(err / tol).max().item():.3f} of the tolerance")
    assert (err <= tol).all()


@pytest.mark.parametrize("name", ["small0", "final0-nosum"])
def test_head_restatement_is_the_oracle_head(name):
    """On the oracle's pre-head activations (tap l5.ff), the restatement's o_j are the oracle's logits up to the fp32
    rounding of the folded head weight (u relative per weight) and bias: u (sum |x w_j| / ||x|| + |b_j|)."""
    from oracle import beat_this_oracle as O

    hp, sd, packed = _packed(name)
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    x = torch.rand(2, 23, 128, generator=torch.Generator().manual_seed(5), dtype=torch.float64) * 7
    taps = {}
    beat, down = O.forward(sd64, x, taps, sum_head=hp["sum_head"])
    D = hp["transformer_dim"]
    xh = taps[f"l{hp['n_layers'] - 1}.ff"]
    w, b = packed["head.w"].view(2, D), packed["head.b"]
    rb, rd, _, _ = R.head_ref(xh, w, b, hp["sum_head"])
    den = xh.norm(dim=-1)
    tol = [R.U * ((xh.abs() @ w[j].abs()) / den + b[j].abs()) * 1.01 for j in (0, 1)]
    tb = tol[0] + tol[1] if hp["sum_head"] else tol[0]
    assert ((rb - beat).abs() <= tb).all() and ((rd - down).abs() <= tol[1]).all()


def test_gelu_fast_meets_e_erf():
    """10^7 points over [-12, 12] (both zeros included), rcp and ex2 off by their full stated error in either
    direction."""
    worst = 0.0
    for part in np.array_split(np.linspace(-12, 12, 10_000_001), 4):
        x = np.concatenate([part, [0.0, -0.0]]).astype(np.float32)
        z = np.abs(x.astype(np.float64)) / math.sqrt(2.0)
        for sign in (1.0, -1.0):
            _, erf_abs = R.gelu_fast_np(x, sign)
            worst = max(worst, float(np.abs(erf_abs.astype(np.float64) - erf(z)).max()))
    print(f"gelu_fast erf: worst error {worst:.3e} = {worst / R.E_ERF:.3f} of E_ERF = {R.E_ERF:.3e}")
    assert worst <= R.E_ERF


# ------------------------------------------------------------------------------ emulations against the bounds
def _plan(lib, chunk, border, mode):
    from beat_this_b200._lib import bt_chunking, i64_array

    ck = bt_chunking(chunk, border, mode)

    def plan(T):
        n = lib.bt_plan_chunking_max(T, ck, 1500, None, None, None, None, 0)
        arrs = [i64_array([0] * n) for _ in range(4)]
        assert lib.bt_plan_chunking_max(T, ck, 1500, *arrs, n) == n
        return [list(a) for a in arrs]

    return plan


def _tables(lib):
    """(name, chunks, L, frames) of small mixed-length waves: two planner chunkings on their sweep lengths, and
    hand-made edges (a chunk past its clip's end, one of a single frame, empty owned ranges)."""
    out = []
    for chunk, border, mode in ((13, 6, 0), (64, 6, 1)):
        chunks, L, frames, _ = R.wave(R.sweep_lengths(chunk, border), _plan(lib, chunk, border, mode))
        out.append((f"plan {chunk}/{border}/{'keep_last' if mode else 'keep_first'}", chunks, L, frames))
    edges = [(3, 30, -12, 3, 12, 20, 40), (36, 10, 4, 36, 0, 6, 9), (49, 1, 0, 49, 0, 1, 1), (53, 5, -2, 53, 3, 3, 7)]
    out.append(("edges", edges, 40, 60))
    return out


def _spect(frames, chunks, g):
    """Log-mel scale frames (0 to 7) with NaN in every guard frame (those outside the table's clips)."""
    x = (torch.rand(frames, 128, generator=g, dtype=torch.float64) * 7).float().numpy()
    inside = np.zeros(frames, bool)
    for fb, T, *_ in chunks:
        inside[fb : fb + T] = True
    x[~inside] = np.nan
    return x


def _stem_inputs(g, kind):
    """(bn1_scale, bn1_shift, w, bias) fp32: random, or the padding probe (scale 0, large distinct shifts)."""
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    if kind == "padding":
        return [np.zeros(128, np.float32), (100 + 10 * torch.arange(128.0)).float().numpy(),
                (r(32, 12) * 0.01).float().numpy(), r(32).float().numpy()]
    return [(0.5 + torch.rand(128, generator=g, dtype=torch.float64)).float().numpy(), (r(128) * 2).float().numpy(),
            (r(32, 12) * 0.4).float().numpy(), (r(32) * 0.3).float().numpy()]


def _stem_ratio(spect, chunks, L, params, **kw):
    got = R.stem_np(spect, chunks, L, *params, **kw).astype(np.float64)
    ref, bound = R.stem_ref(torch.from_numpy(spect).double(), chunks, L, *(torch.from_numpy(p).double() for p in params))
    err = np.abs(got - ref.numpy())
    return float(np.where(np.isfinite(got), err / np.maximum(bound.numpy(), 1e-300), np.inf).max())


def _head_ratio(chunks, L, D, sum_head, g, scale=1.0, **kw):
    n = len(chunks)
    x = torch.randn(n, L, D, generator=g, dtype=torch.float64) * scale
    x[:, 1::7] = 0.0  # zero rows: the output is the bias
    x[:, 2::7] *= 1e-14  # below the 1e-12 clamp
    x = x.float().numpy()
    w = (torch.randn(2, D, generator=g, dtype=torch.float64) * 0.4).float().numpy()
    b = np.array([0.75, -1.5], np.float32)
    out_count = max(c[3] + c[2] + c[5] for c in chunks) + 3
    beat, down = R.head_np(x, w, b, chunks, L, sum_head, out_count, **kw)
    rb, rd, eb, ed = R.head_ref(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(),
                                sum_head)
    worst = 0.0
    for got, ref, bnd in ((beat, rb, eb), (down, rd, ed)):
        r, bd = (R.head_scatter(chunks, L, t, out_count)[0].numpy() for t in (ref, bnd))
        owned = R.head_scatter(chunks, L, ref, out_count)[1].numpy() > 0
        if np.isnan(got[owned]).any() or not np.isnan(got[~owned]).all():
            return math.inf
        worst = max(worst, float((np.abs(got[owned] - r[owned]) / np.maximum(bd[owned], 1e-300)).max()))
    return worst


def test_emulations_stay_inside_and_mistakes_leave_the_bounds(lib_built):
    g = torch.Generator().manual_seed(11)
    tables = _tables(lib_built)
    stem_families, worst = [], {}
    for name, chunks, L, frames in tables:
        spect = _spect(frames, chunks, g)
        for kind in ("random", "padding"):
            stem_families.append((f"{name} {kind}", spect, chunks, L, _stem_inputs(g, kind)))
    # GELU sweep: identity BN, one-hot weights: a = the input, over [-12, 12] with both zeros
    sweep = np.concatenate([np.linspace(-12, 12, 32 * 128 - 2), [0.0, -0.0]]).astype(np.float32).reshape(32, 128)
    one_hot = np.zeros((32, 12), np.float32)
    one_hot[:, 1] = 1.0  # df 0, dt 1: the frame itself
    ident = [np.ones(128, np.float32), np.zeros(128, np.float32), one_hot, np.zeros(32, np.float32)]
    stem_families.append(("gelu sweep", sweep, [(0, 32, 0, 0, 0, 32, 32)], 32, ident))
    _, _, packed = _packed("small0")
    prod = [packed[k].float().numpy() for k in ("stem.bn1_scale", "stem.bn1_shift", "stem.w", "stem.bias")]
    stem_families.append(("small0 weights", _spect(tables[1][3], tables[1][1], g), tables[1][1], tables[1][2], prod))

    for sign in (1.0, -1.0):
        for fam, spect, chunks, L, params in stem_families:
            ratio = _stem_ratio(spect, chunks, L, params, sign=sign)
            worst[f"stem {fam}"] = max(worst.get(f"stem {fam}", 0.0), ratio)
            assert ratio <= 1, (fam, sign, ratio)
    for mistake in R.STEM_MISTAKES:
        ratios = {fam: _stem_ratio(spect, chunks, L, params, mistake=mistake) for fam, spect, chunks, L, params in stem_families}
        print(f"stem mistake {mistake}: worst {max(ratios.values()):.3g} of the bound ({max(ratios, key=ratios.get)})")
        assert max(ratios.values()) > 1, (mistake, ratios)

    head_families = [(name, chunks, L, D, sh, scale) for name, chunks, L, _ in tables for D in (64, 128)
                     for sh in (False, True) for scale in (1.0, 1e3)]
    for name, chunks, L, D, sh, scale in head_families:
        ratio = _head_ratio(chunks, L, D, sh, torch.Generator().manual_seed(D), scale)
        worst[f"head {name}"] = max(worst.get(f"head {name}", 0.0), ratio)
        assert ratio <= 1, (name, D, sh, scale, ratio)
    for mistake in R.HEAD_MISTAKES:
        ratios = [_head_ratio(chunks, L, D, sh, torch.Generator().manual_seed(D), scale, mistake=mistake)
                  for _, chunks, L, D, sh, scale in head_families]
        print(f"head mistake {mistake}: worst {max(ratios):.3g} of the bound")
        assert max(ratios) > 1, mistake

    for name, chunks, L, _ in tables:
        for F, C in ((32, 32), (16, 64), (8, 128)):
            buf = np.random.default_rng(F).integers(1, 2**31, (len(chunks), F, L, C)).astype(np.int32)
            assert np.array_equal(R.zero_tail_np(buf, chunks, F, L), R.zero_tail_ref(torch.from_numpy(buf), chunks, F, L, C).numpy())
    for mistake in R.ZERO_TAIL_MISTAKES:
        caught = False
        for _, chunks, L, _ in tables:
            buf = np.ones((len(chunks), 8, L, 4), np.int32)
            ref = R.zero_tail_ref(torch.from_numpy(buf), chunks, 8, L, 4).numpy()
            caught = caught or not np.array_equal(R.zero_tail_np(buf, chunks, 8, L, mistake), ref)
        assert caught, mistake
    for k, v in worst.items():
        print(f"{k}: worst {v:.3f} of the bound")
