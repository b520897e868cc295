"""GPU parity tests (run on an H100: pytest -m gpu).  Every test calls the CUDA path
through the C ABI (ctypes) and compares with the CPU oracle (oracle/beat_this_oracle.py) or the
golden fixtures written from the reference's own outputs (tests/golden, oracle/make_golden.py).

Tolerances (stated):
  fp32 path  : frame logits within 1e-3 of the fp32 reference (measured ~1e-4).
  16-bit path: fp16 operands (the reference's float16=True autocast dtype), fp32 accumulate and residual stream:
               frame logits within H16_TOL = 0.05 absolute of the fp32 reference (logits have std ~2, range +-8);
               per-stage activations within H16_STAGE_TOL absolute.
"""
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from gemm_reference import GEMM_CASES, _check_gemm_case
from numerics import H16_TOL
from support import dev, small_h16  # noqa: F401  (fixtures)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

H16_STAGE_TOL = 0.03


def _engine(ckpt, half):
    from beat_this_b200.inference import load_model

    return load_model(ckpt, "cuda:0", float16=half)


@pytest.fixture(scope="module")
def small_f32(small0_ckpt, lib_built, dev):
    return _engine(small0_ckpt, False)


@pytest.fixture(scope="module")
def final_f32(final0_ckpt, lib_built, dev):
    return _engine(final0_ckpt, False)


@pytest.fixture(scope="module")
def final_h16(final0_ckpt, lib_built, dev):
    return _engine(final0_ckpt, True)


def _sd(path):
    from oracle import beat_this_oracle as O

    return O.strip_prefix(torch.load(path, weights_only=True)["state_dict"])


# ------------------------------------------------------------------------------ log-mel
def test_logmel_matches_reference_golden(lib_built, dev):
    from beat_this_b200 import synthetic
    from beat_this_b200.preprocessing import LogMelSpect

    g = np.load(os.path.join(GOLDEN, "logmel.npz"))
    mel = LogMelSpect(device=dev)
    for idx in (0, 1):
        x = synthetic.synth_clip(idx, float(g[f"clip{idx}_secs"]))
        out = mel(torch.tensor(x, dtype=torch.float32, device=dev)).cpu().numpy()
        ref = g[f"clip{idx}_mel"]
        assert out.shape == ref.shape
        err = np.abs(out - ref).max()
        print(f"logmel clip{idx}: max abs err vs reference {err:.3e}")
        assert err < 2e-3  # fp32 FFT round-off amplified by log1p(1000 x) near silence


def test_logmel_batch_and_edges(lib_built, dev):
    from beat_this_b200.engine import Engine
    from oracle import beat_this_oracle as O

    eng = Engine.mel_only(dev)
    rng = np.random.default_rng(0)
    lens = [513, 1024, 22050, 44100 + 17, 441 * 7]
    sigs = [rng.standard_normal(n).astype(np.float32) * 0.1 for n in lens]
    outs = eng.logmel(sigs)
    for s, o in zip(sigs, outs):
        ref = O.logmel(torch.tensor(s))
        assert o.shape == ref.shape == (1 + len(s) // 441, 128)
        assert (o.cpu() - ref).abs().max() < 2e-3
    with pytest.raises(Exception):
        eng.logmel([np.zeros(512, np.float32)])  # torch.stft reflect padding fails here too


# ------------------------------------------------------------------------------ peak picking
def test_peakpick_golden_bit_exact(lib_built, dev):
    from beat_this_b200.postprocessor import Postprocessor

    g = np.load(os.path.join(GOLDEN, "postp_minimal.npz"))
    post = Postprocessor("minimal", device=dev)
    n = int(g["n"])
    # one by one (unbatched API) ...
    for i in range(n):
        bt, dt = post(torch.tensor(g[f"beat_{i}"]), torch.tensor(g[f"down_{i}"]))
        assert bt.dtype == np.float64 and dt.dtype == np.float64
        assert np.array_equal(bt, g[f"beat_times_{i}"]), i
        assert np.array_equal(dt, g[f"down_times_{i}"]), i
    # ... and all clips in one launch
    fo = [0]
    for i in range(n):
        fo.append(fo[-1] + len(g[f"beat_{i}"]))
    b = torch.tensor(np.concatenate([g[f"beat_{i}"] for i in range(n)]), device=dev)
    d = torch.tensor(np.concatenate([g[f"down_{i}"] for i in range(n)]), device=dev)
    res = post.batch_cat(b, d, fo)
    for i in range(n):
        assert np.array_equal(res[i][0], g[f"beat_times_{i}"]), i
        assert np.array_equal(res[i][1], g[f"down_times_{i}"]), i


# ------------------------------------------------------------------------------ GEMM units
# (the attention kernels: tests/test_gpu_attention.py)
# plain D = A W^T through Engine.debug_gemm, no epilogue (M, N, K)
GEMM_SHAPES = [(300, 96, 32), (1500, 32, 128), (1000, 64, 64), (700, 192, 64), (1500, 1536, 512), (520, 512, 2048), (257, 128, 256)]


@pytest.mark.parametrize("half", [False, True])
def test_debug_gemm(small_f32, small_h16, half):
    """Every GEMM instantiation, tile policy, epilogue and slab shape against float64 (tests/gemm_reference.py).  Every
    case runs and prints its worst error; the failing ones are listed together at the end."""
    eng = (small_h16 if half else small_f32).engine
    g = torch.Generator(device="cpu").manual_seed(1)
    for M, N, K in GEMM_SHAPES:
        a = torch.randn(M, K, generator=g)
        w = torch.randn(N, K, generator=g) / math.sqrt(K)
        if half:  # the 16-bit path rounds its operands: compare on the rounded values (fp32 accumulation is what is tested)
            a, w = a.half().float(), w.half().float()
        ref = a.double() @ w.double().T
        d = eng.debug_gemm(a.cuda(), w.cuda()).cpu().double()
        err = (d - ref).abs().max().item()
        print(f"gemm half={half} {M}x{N}x{K}: max abs err {err:.3e}")
        assert err < 1e-4, (M, N, K)
    failures = []
    for case in GEMM_CASES:
        try:
            _check_gemm_case(eng, half, case)
        except AssertionError as e:
            failures.append(f"{case.id}: {str(e).splitlines()[0]}")
    assert not failures, f"{len(failures)} of {len(GEMM_CASES)} GEMM cases failed:\n" + "\n".join(failures)


@pytest.mark.parametrize("sr", [44100, 48000, 16000, 96000])
def test_resample_matches_direct_form(lib_built, dev, sr):
    """bt_resample (device polyphase FIR, stand-in for soxr.resample, inference.py:274-275) against the float64
    direct-form definition, ragged clips incl. one shorter than the filter."""
    from beat_this_b200.engine import Engine
    from oracle import beat_this_oracle as O

    eng = Engine(None, None, dev)  # no model parameters needed
    rng = np.random.default_rng(sr)
    clips = [rng.uniform(-1, 1, n) for n in (sr // 3 + 17, 50, 3 * sr // 4, 1)]
    so = [0]
    for c in clips:
        so.append(so[-1] + len(c))
    audio = torch.tensor(np.concatenate(clips), dtype=torch.float32, device=dev)
    out, oo = eng.resample_cat(audio, so, sr)
    worst = 0.0
    for i, c in enumerate(clips):
        ref = O.resample_direct(c.astype(np.float32).astype(np.float64), sr)
        got = out[oo[i] : oo[i + 1]].cpu().numpy()
        assert got.shape == ref.shape, (i, got.shape, ref.shape)
        if len(ref):
            worst = max(worst, float(np.abs(got - ref).max()))
    print(f"resample {sr} -> 22050: max abs err vs float64 direct form {worst:.3e}")
    assert worst < 2e-5


# ------------------------------------------------------------------------------ per-stage parity
TAPS = ["stem"] + [f"b{i}.{s}" for i in range(3) for s in ("attnF", "ffF", "attnT", "ffT", "conv")] + ["frontend"] + [
    f"l{l}.{s}" for l in range(6) for s in ("attn", "ff")
]


def _stage_errors(model, ckpt, T=138, nclips=2):
    from oracle import beat_this_oracle as O

    sd = _sd(ckpt)
    torch.manual_seed(3)
    spects = [torch.rand(T, 128) * 7 for _ in range(nclips)]
    chunks = torch.stack([O.split_piece(s)[0][0] for s in spects])  # [n, T+12, 128]
    taps = {}
    with torch.inference_mode():
        O.forward(sd, chunks, taps)
    fo = [i * T for i in range(nclips + 1)]
    cat = torch.cat(spects).cuda()
    rows = []
    for name in TAPS:
        ref = taps[name]
        got, _ = model.engine.tap(name, cat, fo, ref.numel())
        assert got.numel() == ref.numel(), name
        err = (got.cpu().view(ref.shape) - ref).abs().max().item()
        rows.append((name, err, ref.abs().max().item()))
    return rows


def test_stage_parity_fp32(small_f32, small0_ckpt):
    rows = _stage_errors(small_f32, small0_ckpt)
    for name, err, mag in rows:
        print(f"fp32 stage {name:10s} max abs err {err:.3e} (|ref| max {mag:.2f})")
    assert max(r[1] for r in rows) < 1e-3


def test_stage_parity_h16(small_h16, small0_ckpt):
    rows = _stage_errors(small_h16, small0_ckpt)
    for name, err, mag in rows:
        print(f"h16 stage {name:10s} max abs err {err:.3e} (|ref| max {mag:.2f})")
    assert max(r[1] for r in rows) < H16_STAGE_TOL


def _stage_errors_full_chunks(model, ckpt, nchunks=2, T=1500):
    """Per-stage taps on FULL 1500-frame chunks (the shape the bench runs: 256x64 GEMM tiles, 24 key tiles per
    attention row) through bt_forward_chunks, against the oracle forward of the same chunks."""
    from oracle import beat_this_oracle as O

    sd = _sd(ckpt)
    torch.manual_seed(4)
    chunks = torch.rand(nchunks, T, 128) * 7
    taps = {}
    with torch.inference_mode():
        rb, rd = O.forward(sd, chunks, taps)
    dev_chunks = chunks.cuda()
    rows = []
    for name in TAPS:
        ref = taps[name]
        got, _ = model.engine.tap_chunks(name, dev_chunks, ref.numel())
        assert got.numel() == ref.numel(), name
        rows.append((name, (got.cpu().view(ref.shape) - ref).abs().max().item(), ref.abs().max().item()))
    out = model(dev_chunks)
    rows.append(("logits", max((out["beat"].cpu() - rb).abs().max().item(), (out["downbeat"].cpu() - rd).abs().max().item()),
                 max(rb.abs().max().item(), rd.abs().max().item())))
    return rows


def test_stage_parity_final0_full_chunks_fp32(final_f32, final0_ckpt):
    rows = _stage_errors_full_chunks(final_f32, final0_ckpt)
    for name, err, mag in rows:
        print(f"final0 T=1500 fp32 stage {name:10s} max abs err {err:.3e} (|ref| max {mag:.2f})")
    assert max(r[1] for r in rows) < 1e-3


def test_stage_parity_final0_full_chunks_h16(final_h16, final0_ckpt):
    rows = _stage_errors_full_chunks(final_h16, final0_ckpt)
    for name, err, mag in rows:
        print(f"final0 T=1500 h16 stage {name:10s} max abs err {err:.3e} (|ref| max {mag:.2f})")
    assert max(r[1] for r in rows[:-1]) < H16_STAGE_TOL
    assert rows[-1][1] < H16_TOL


def test_postprocessor_batched_with_padding_mask(lib_built, dev):
    """Postprocessor API parity (reference postprocessor.py:39-83): batched [B,T] logits with a padding
    mask give, per piece, what the un-batched call gives on the un-padded logits."""
    from beat_this_b200.postprocessor import Postprocessor
    from oracle import beat_this_oracle as O

    rng = np.random.default_rng(11)
    T, lens = 400, [400, 250, 31]
    beat = torch.tensor(rng.standard_normal((3, T)).astype(np.float32) * 2)
    down = torch.tensor(rng.standard_normal((3, T)).astype(np.float32) * 2 - 1)
    mask = torch.zeros(3, T, dtype=torch.bool)
    for i, n in enumerate(lens):
        mask[i, :n] = True
    post = Postprocessor("minimal", device=dev)
    pb, pd = post(beat, down, mask)
    assert isinstance(pb, tuple) and len(pb) == 3
    for i, n in enumerate(lens):
        ob, od = O.postp_minimal(beat[i, :n], down[i, :n])
        assert np.array_equal(pb[i], ob) and np.array_equal(pd[i], od)
        ub, ud = post(beat[i, :n], down[i, :n])
        assert np.array_equal(ub, ob) and np.array_equal(ud, od)
    with pytest.raises(AssertionError):
        Postprocessor("viterbi")
