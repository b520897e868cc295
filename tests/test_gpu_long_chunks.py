"""GPU tests of chunks longer than 1500 frames, on models loaded with a larger max_chunk_size: the reference's own
logits (tests/golden/long_chunks.npz, oracle/make_golden_long_chunks.py), the batched path against the per-chunk route,
the default chunking unchanged on such a model, waves under the frame budget, the attention and RoPE GEMM kernels at
long L against their float64 references, and the refusals above a model's limit."""
import collections
import ctypes
import math
import os
import wave
import zlib

import numpy as np
import pytest
import torch

import attention_reference as R
from conftest import GOLDEN, ckpt_path
from gemm_reference import _kind1, _run_gemm, epilogue_ref, gemm_ref
from numerics import (EX2_APPROX_REL, EXPF_REL, F32_TOL, GEMM_ACC_TOL_F32, GEMM_ACC_TOL_H16, H16_TOL, LOG2E, QSCALE_H16,
                      S_F32, U, mma_error, rnd, ulp16)
from support import act_dtype, launch_twice

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

MODES = ("keep_first", "keep_last")
LONG = 8000  # max_chunk_size of the long-limit models
# (chunk_size, border_size, overlap_mode): the fixture's settings, and a chunk just past the default limit
SETTINGS = [(3000, 6, "keep_first"), (3000, 0, "keep_last"), (4500, 12, "keep_first"), (8000, 0, "keep_first"),
            (1501, 100, "keep_last")]


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "long_chunks.npz"))


def _s2f(name, float16, max_chunk_size=LONG):
    from beat_this_b200.inference import Spect2Frames

    return Spect2Frames(ckpt_path(name), "cuda:0", float16, max_chunk_size=max_chunk_size)


@pytest.mark.parametrize("float16", [False, True])
@pytest.mark.parametrize("model_name", ["small0", "final0"])
def test_reference_parity(gold, lib_built, model_name, float16):
    """split_predict_aggregate with chunks of 3000 to 8000 frames (whole pieces at 8000) and BeatThis.forward on a
    [2, 3000, 128] batch, against the reference on the CPU (our log-mel of the same samples in front)."""
    from beat_this_b200 import synthetic
    from beat_this_b200.inference import split_predict_aggregate
    from oracle import beat_this_oracle as O

    sd = O.strip_prefix(torch.load(ckpt_path(model_name), weights_only=True)["state_dict"])
    want_sum = float(gold[f"{model_name}_ckpt_sum"])
    assert abs(synthetic.tensor_checksum(sd) - want_sum) < 1e-6 * abs(want_sum)
    model = _s2f(model_name, float16).model
    assert model.max_chunk_size == LONG
    worst = 0.0

    def err(out, rb, rd):
        assert out["beat"].shape == rb.shape
        return max(np.abs(out["beat"].cpu().numpy() - rb).max(), np.abs(out["downbeat"].cpu().numpy() - rd).max())

    for j, (seed, secs) in enumerate(gold["clips"]):
        spect = model.engine.logmel([synthetic.synth_clip(int(seed), float(secs))])[0]
        assert spect.shape[0] == int(gold["clip_frames"][j])
        for i, (c, b, m) in enumerate(gold["settings"]):
            out = split_predict_aggregate(spect, int(c), int(b), MODES[int(m)], model)
            e = err(out, gold[f"{model_name}_beat_s{i}_c{j}"], gold[f"{model_name}_down_s{i}_c{j}"])
            print(f"{model_name} float16={float16} {spect.shape[0]} frames, chunking {c}/{b}/{MODES[int(m)]}: "
                  f"max abs logit err {e:.3e}")
            worst = max(worst, e)
    x = torch.rand(2, 3000, 128, generator=torch.Generator().manual_seed(int(gold["forward_seed"]))) * 7
    out = model(x.cuda())
    e = err({k: v.flatten() for k, v in out.items()}, gold[f"{model_name}_forward_beat"].flatten(),
            gold[f"{model_name}_forward_down"].flatten())
    print(f"{model_name} float16={float16} forward [2, 3000, 128]: max abs logit err {e:.3e}")
    worst = max(worst, e)
    print(f"{model_name} float16={float16}: worst max abs logit err {worst:.3e}")
    assert worst < (H16_TOL if float16 else F32_TOL)


@pytest.mark.parametrize("float16", [False, True])
@pytest.mark.parametrize("model_name", ["small0", "final0"])
def test_batched_equals_per_chunk_route_bitwise(lib_built, model_name, float16):
    """Every chunk of every piece in one call against one bt_forward_chunks call per chunk (BeatThisB200.__call__)
    stitched by aggregate_prediction: bit-identical."""
    from beat_this_b200.inference import split_predict_aggregate

    s2f = _s2f(model_name, float16)
    model = s2f.model
    per_chunk = lambda x: model(x)  # noqa: E731  (not a BeatThisB200: split_predict_aggregate walks the chunks)
    g = torch.Generator().manual_seed(7 + (model_name == "final0"))
    for c, b, mode in SETTINGS:
        lengths = sorted({1, c - 2 * b, c - 2 * b + 1, c, c + 1, 2 * c + 7, 7501})
        pieces = [torch.rand(T, 128, generator=g) * 7 for T in lengths]
        out = s2f.spects2frames([p.cuda() for p in pieces], c, b, mode)
        for p, (beat, down) in zip(pieces, out):
            ref = split_predict_aggregate(p.cuda(), c, b, mode, per_chunk)
            assert (ref["beat"] > -1000).all(), (c, b, mode, p.shape[0])
            assert torch.equal(beat, ref["beat"]) and torch.equal(down, ref["downbeat"]), (c, b, mode, p.shape[0])
        print(f"{model_name} float16={float16} chunking {c}/{b}/{mode}: {len(pieces)} pieces bitwise equal")


def _kernel_counts(eng, fn):
    """{launch class: launches} of fn() under the library's per-launch profiler (bt_profile_*), and fn's result."""
    eng.profile_reset()
    eng.profile_enable(True)
    try:
        res = fn()
        counts = {name: n for name, (_, n) in eng.profile_results().items() if n}
    finally:
        eng.profile_enable(False)
    return collections.Counter(counts), res


@pytest.mark.parametrize("float16", [False, True])
def test_default_chunking_is_unchanged_on_a_long_limit_model(small0_ckpt, lib_built, float16):
    """A model loaded with max_chunk_size=8000 and one loaded the default way, on a ragged batch of more than 128
    chunks: at 1500 / 6 / keep_first (and at 1000 / 0 / keep_first, the chunked entry point) the outputs are
    bitwise equal and the same kernels run the same number of times, so the waves are the same."""
    s2fs = [_s2f("small0", float16, 1500), _s2f("small0", float16, LONG)]
    assert [s.model.max_chunk_size for s in s2fs] == [1500, LONG]
    assert [s.model.engine.lib.bt_max_chunk(s.model.engine.ctx) for s in s2fs] == [1500, LONG]
    g = torch.Generator().manual_seed(3)
    pieces = [torch.rand(T, 128, generator=g).cuda() * 7 for T in [25, 250, 1485, 1501, 3051] + [30001] * 6 + [4750]]
    for chunking in ((1500, 6, "keep_first"), (1000, 0, "keep_first")):
        outs, counts, launches = [], [], []
        for s2f in s2fs:
            s2f.spects2frames(pieces, *chunking)  # workspace and plans in place
            n0 = s2f.model.engine.launches
            cnt, out = _kernel_counts(s2f.model.engine, lambda: s2f.spects2frames(pieces, *chunking))
            outs.append(out)
            counts.append(cnt)
            launches.append(s2f.model.engine.launches - n0)
        assert counts[0]["stem"] > 1  # more than one wave
        assert counts[0] == counts[1], (chunking, counts)
        assert launches[0] == launches[1], (chunking, launches)
        for (b0, d0), (b1, d1) in zip(*outs):
            assert torch.equal(b0, b1) and torch.equal(d0, d1), chunking
        print(f"float16={float16} chunking {chunking}: {launches[0]} launches, {counts[0]['stem']} waves, "
              f"{sum(counts[0].values())} profiled launches in {len(counts[0])} classes in both")


def _expected_waves(lengths, chunks, budget):
    """The waves run_chunks forms: longest first, closed before `chunks` chunks or `budget` padded frames."""
    order, waves, i = sorted(lengths, reverse=True), [], 0
    while i < len(order):
        j = i + 1
        while j < len(order) and j - i < chunks and (j - i + 1) * order[i] <= budget:
            j += 1
        waves.append((j - i, order[i]))
        i = j
    return waves


@pytest.mark.parametrize("float16", [False, True])
def test_wave_packing(small0_ckpt, lib_built, float16):
    """Whole pieces as single chunks of 1 to 8000 frames (chunking 8000 / 0): with 3, 5 and 128 chunks per wave the
    waves are those of the frame budget max(chunks x 1500, 8000), none holds more padded frames than the budget, and
    every piece's logits are bitwise those of the piece run alone."""
    s2f = _s2f("small0", float16)
    eng = s2f.model.engine
    lengths = [8000, 2500, 7999, 100, 4001, 3999, 1500, 1, 6000, 2000, 5000, 777, 3000, 1501]
    g = torch.Generator().manual_seed(11)
    pieces = [torch.rand(T, 128, generator=g).cuda() * 7 for T in lengths]
    alone = [s2f.spects2frames([p], LONG, 0, "keep_first")[0] for p in pieces]
    for chunks in (3, 5, 128):
        eng.set_wave_chunks(chunks)
        budget = max(chunks * 1500, LONG)
        waves = _expected_waves(lengths, chunks, budget)
        assert all(nb * L <= budget for nb, L in waves)
        s2f.spects2frames(pieces[:1], LONG, 0, "keep_first")  # workspace in place
        eng.profile_reset()
        eng.profile_enable(True)
        out = s2f.spects2frames(pieces, LONG, 0, "keep_first")
        prof = eng.profile_results()
        eng.profile_enable(False)
        assert prof["stem"][1] == len(waves), (chunks, prof["stem"], waves)
        for T, (b, d), (ab, ad) in zip(lengths, out, alone):
            assert torch.equal(b, ab) and torch.equal(d, ad), (chunks, T)
        print(f"float16={float16} {chunks} chunks per wave, budget {budget} frames: waves (chunks, padded length) {waves}")
    eng.set_wave_chunks(128)


# ---- kernel units at long L
# time cases past 1500 frames: (seqs, L, heads, key lens per chunk, sequences per chunk)
LONG_TIME_CASES = [R.TimeCase(2, 1501, 2), R.TimeCase(2, 1501, 2, (1501, 1000), 1),
                   R.TimeCase(2, 3000, 4), R.TimeCase(4, 3000, 2, (3000, 2999), 2),
                   R.TimeCase(1, 7501, 4), R.TimeCase(2, 7501, 1, (7501, 64), 1),
                   R.TimeCase(1, 24000, 1), R.TimeCase(2, 24000, 1, (24000, 17001), 1)]
ROWS = 2048  # query rows per slice of the float64 reference


def time_ref_rows(q, k, v, gates, lens, path, dt, r0, r1):
    """attention_reference.time_ref for the query rows [r0, r1) of every sequence only: the same operands, scores and
    softmax_ref arguments, on [r1 - r0, L] instead of [L, L] (an L x L float64 problem at L = 24000 does not fit in
    memory).  Returns (ref, bound, o, err), each [seqs, r1 - r0, C]."""
    seqs, L, C = q.shape
    H = C // 32
    hv = lambda t: t.reshape(seqs, L, H, 32).permute(0, 2, 1, 3).reshape(seqs * H, L, 32)  # noqa: E731
    if path == "tc":
        qh, kh, vh, sc = hv(rnd(R._f32mul(q, QSCALE_H16), dt)), hv(rnd(k, dt)), hv(rnd(v, dt)), 1.0
    else:
        qh, kh, vh, sc = hv(R._f32mul(q, S_F32)), hv(k), hv(v), LOG2E
    g = gates.reshape(seqs, L, H).permute(0, 2, 1).reshape(seqs * H, L)[:, r0:r1]
    qh = qh[:, r0:r1]
    lens_g = torch.as_tensor(lens, device=q.device).repeat_interleave(H)
    valid = torch.arange(L, device=q.device)[None, :] < lens_g[:, None]
    out = [torch.empty_like(qh) for _ in range(4)]
    for a in range(seqs * H):
        b = a + 1
        T2 = sc * (qh[a:b] @ kh[a:b].transpose(1, 2))
        vm = valid[a:b]
        S = qh[a:b].abs() @ kh[a:b].abs().transpose(1, 2)
        nkv = (vm.sum(-1) + R.AT_TILE - 1) // R.AT_TILE
        if path == "tc":
            pk = R.poly_keys(L, q.device)
            kw = dict(step=R.AT_TILE, alpha_rel=EX2_APPROX_REL + U, sub_ops=1, p_dt=dt, n_sum=16 * nkv + 2,
                      pv_error=lambda s, nnz: mma_error(nnz, s), out_dt=dt, n_pad=R.AT_TILE,
                      exp_rel=lambda x, e: torch.where(pk, R.EX2_POLY_REL, EX2_APPROX_REL).expand_as(x))
            E2 = mma_error(32, S)
        else:
            nk = R.SA_BLOCK * ((vm.sum(-1) + R.SA_BLOCK - 1) // R.SA_BLOCK)
            kw = dict(step=R.SA_BLOCK, alpha_rel=EXPF_REL + U, sub_ops=1, p_dt=None, n_sum=nk,
                      pv_error=lambda s, nnz: nk[:, None, None] * U * s, out_dt=None, n_pad=0,
                      exp_rel=lambda x, e: torch.full_like(x, EXPF_REL))
            E2 = 32 * U * S * LOG2E
        for o, r in zip(out, R.softmax_ref(T2, E2, vm, vh[a:b], g[a:b], **kw)):
            o[a:b] = r
    n = r1 - r0
    return tuple(t.view(seqs, H, n, 32).permute(0, 2, 1, 3).reshape(seqs, n, C) for t in out)


@pytest.fixture(scope="module")
def engines(lib_built):
    from beat_this_b200.engine import Engine

    return {half: Engine(None, None, "cuda:0", half=half) for half in (False, True)}


@pytest.mark.parametrize("half", [False, True])
def test_row_slices_are_the_reference(engines, half):
    """time_ref_rows over slices of rows equals attention_reference.time_ref on the whole problem, up to the last bits
    of float64 products that cuBLAS sums in another order for another row count (~1e-10 relative, 1e-16 absolute
    on an H100; the bounds are ~1e-4 relative)."""
    dev = torch.device("cuda:0")
    case = R.TimeCase(2, 1501, 2, (1501, 700), 1)
    g = torch.Generator(device=dev).manual_seed(5)
    q, k, v, gates = (t.double() for t in R.time_inputs(case, "random", g, dev))
    lens = torch.tensor(case.lens(), device=dev)
    path, dt = ("tc", act_dtype(engines[True])) if half else ("simt", None)
    full = R.time_ref(q, k, v, gates, lens, path, dt)
    for r0, r1 in ((0, 512), (512, 1024), (1024, 1501)):
        for f, s in zip(full, time_ref_rows(q, k, v, gates, lens, path, dt, r0, r1)):
            torch.testing.assert_close(s, f[:, r0:r1], rtol=1e-9, atol=1e-14)


@pytest.mark.parametrize("half", [False, True])
def test_attention_at_long_L(engines, half):
    """attn_time_kernel (16-bit) and attn_time_simt_kernel (fp32) at L = 1501, 3000, 7501 and 24000, with and without
    key lengths per chunk, on random inputs and on a late maximum (the online softmax rescales over every tile of the
    row): every element within the derived bound of attention_reference, finite, no store past M, repeatable."""
    eng = engines[half]
    dev = torch.device("cuda:0")
    path, dt = ("tc", act_dtype(eng)) if half else ("simt", None)
    failures, worst = [], {}
    for case in LONG_TIME_CASES:
        families = ["random", "late_max"] + (["masked_garbage"] if case.key_lens is not None else [])
        for family in families:
            g = torch.Generator(device=dev).manual_seed(zlib.crc32(f"{case.id} {family}".encode()))
            q, k, v, gates = R.time_inputs(case, family, g, dev)
            M, C = case.seqs * case.L, 32 * case.heads
            got = launch_twice(lambda out: eng.debug_attention(q, k, v, gates, case.key_lens, case.spc, out=out),
                                M, C, dev).view(case.seqs, case.L, C)
            lens = torch.tensor(case.lens(), device=dev)
            ratio = 0.0
            for r0 in range(0, case.L, ROWS):
                r1 = min(case.L, r0 + ROWS)
                ref, bound, _, _ = time_ref_rows(q.double(), k.double(), v.double(), gates.double(), lens, path, dt, r0, r1)
                part = got[:, r0:r1]
                if not torch.isfinite(part).all():
                    ratio = math.inf
                    break
                err = (part - ref).abs()
                ratio = max(ratio, torch.where(err == 0, 0.0, err / bound).max().item())
            print(f"{path} {case.id} {family}: worst error {ratio:.3f} of its bound")
            worst[family] = max(worst.get(family, 0.0), ratio)
            if not ratio <= 1:
                failures.append(f"{case.id} {family}: {ratio:.2f} x its bound")
    print(f"{path}: worst error per family {worst}")
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("half", [False, True])
def test_rope_gemm_past_1500(engines, half):
    """The RoPE epilogue (kind 1) of gemm_tc_kernel / gemm_simt_kernel at positions up to 8000 and 24000, with tables of
    that many rows, against gemm_reference (the GEMM tolerances of numerics.py)."""
    from beat_this_b200.weights import rope_tables

    eng = engines[half]
    dev = torch.device("cuda:0")
    freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
    for case, P in ((_kind1("qkv-time-C32-L8000", 2, 8000, 32), 8000), (_kind1("qkv-time-C64-L8000", 1, 8000, 64), 8000),
                    (_kind1("qkv-time-C512-L3000", 2, 3000, 512), 8000), (_kind1("qkv-time-C128-L24000", 1, 24000, 128), 24000)):
        sh, M, N = case.shape, case.M, case.shape["N"]
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(case.id.encode()))
        a = torch.randn(sh["planes_in"] * sh["L"], sh["lda"], generator=g, device=dev)
        w = torch.randn(N, sh["Kslab"], generator=g, device=dev) / math.sqrt(sh["Kslab"])
        rope = tuple(t.contiguous().to(dev) for t in rope_tables(freqs, P))
        _, _, oa = _run_gemm(eng, case, a, w, None, None, rope)
        assert torch.isnan(oa[M * N :]).all(), "activation store past the last row"
        adt = act_dtype(eng)
        dt = adt if half else None
        ref, _ = epilogue_ref(case, gemm_ref(sh, rnd(a.double(), dt), rnd(w.double(), dt)), None, None, half,
                              *(t.double() for t in rope))
        tol = (GEMM_ACC_TOL_H16 if half else GEMM_ACC_TOL_F32) * (1 + ref.abs())
        got = oa[: M * N].view(M, N).double()
        if half:
            ref = ref.to(adt).double()
            tol = ulp16(ref, adt) + tol
        err = (got - ref).abs().nan_to_num(float("inf"))
        ratio = (err / tol).max().item()
        print(f"gemm {'h16' if half else 'f32'} {case.id}, table of {P} rows: max abs err {err.max().item():.3e} = "
              f"{ratio:.2f} of its bound")
        assert ratio <= 1, case.id


# ---- refusals
def _write_wav(path, pcm):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(22050)
        w.writeframes(pcm.tobytes())


@pytest.mark.parametrize("limit", [1500, 3000])
def test_chunks_above_the_limit_are_refused_before_any_launch(small0_ckpt, lib_built, tmp_path, limit):
    """A chunk longer than the model's max_chunk_size raises ValueError (Python) or returns BT_ERR_ARG (C ABI) and
    launches nothing; a model loaded the default way still refuses 1501."""
    from beat_this_b200 import _lib, synthetic
    from beat_this_b200.inference import File2Beats, split_predict_aggregate

    f2b = File2Beats(small0_ckpt, "cuda:0", False, max_chunk_size=limit) if limit != 1500 else \
        File2Beats(small0_ckpt, "cuda:0", False)
    model, eng = f2b.model, f2b.model.engine
    assert model.max_chunk_size == limit == eng.lib.bt_max_chunk(eng.ctx)
    spect = torch.rand(7501, 128, device="cuda:0") * 7
    path = tmp_path / "clip.wav"
    pcm = np.round(synthetic.synth_clip(90, 5.0) * 32767).astype(np.int16)
    _write_wav(path, pcm)
    f2b.frames_batch([path], limit, 0, "keep_first")  # workspace and staging ring in place
    f2b.spects2frames([spect], limit, 6, "keep_first")
    model(spect[None, :limit].contiguous())
    torch.cuda.synchronize()
    n0 = eng.launches
    for c, b, mode in [(limit + 1, 0, "keep_first"), (limit + 1, 6, "keep_last"), (2 * limit, 0, "keep_first")]:
        for call in (lambda: split_predict_aggregate(spect, c, b, mode, model),
                     lambda: f2b.spects2frames([spect], c, b, mode),
                     lambda: f2b.frames_batch([path], c, b, mode),
                     lambda: eng.spect2frames_cat(spect, [0, 7501], (c, b, mode))):
            with pytest.raises(ValueError, match="max_chunk_size"):
                call()
    with pytest.raises(ValueError, match="max_chunk_size"):
        model(spect[None, : limit + 1].contiguous())
    out = torch.empty(2, 7501, device="cuda:0")
    audio = torch.from_numpy(pcm.astype(np.float32) / 32768).cuda()
    so, fo = [0, len(pcm)], eng.frame_offsets([0, len(pcm)])
    st = eng._stream()
    for c in (limit + 1, 30001):
        ck = _lib.bt_chunking(c, 0, 0)
        assert eng.lib.bt_spect2frames_chunked(eng.ctx, ctypes.c_void_p(spect.data_ptr()), _lib.i64_array([0, 7501]), 1,
                                               ctypes.c_void_p(out[0].data_ptr()), ctypes.c_void_p(out[1].data_ptr()),
                                               ctypes.byref(ck), st) == -1
        assert b"bt_max_chunk" in eng.lib.bt_last_error(eng.ctx)
        assert eng.lib.bt_audio2frames_chunked(eng.ctx, ctypes.c_void_p(audio.data_ptr()), _lib.i64_array(so), 1,
                                               ctypes.c_void_p(out[0].data_ptr()), ctypes.c_void_p(out[1].data_ptr()),
                                               _lib.i64_array(fo), ctypes.byref(ck), st) == -1
        assert eng.lib.bt_forward_chunks(eng.ctx, ctypes.c_void_p(spect.data_ptr()), 1, c,
                                         ctypes.c_void_p(out[0].data_ptr()), ctypes.c_void_p(out[1].data_ptr()), st) == -1
        assert b"bt_max_chunk" in eng.lib.bt_last_error(eng.ctx)
    assert eng.launches == n0
    assert f2b.pipeline.free and not f2b.pipeline.inflight


def test_finalize_checks_the_rope_tables(small0_ckpt, lib_built):
    """bt_finalize takes RoPE tables of P x 16 elements for 1500 <= P <= 384000 and sets bt_max_chunk to P; a shorter
    table, a partial row, a cos / sin mismatch or a longer one is BT_ERR_PARAM."""
    from beat_this_b200._lib import BTError
    from beat_this_b200.engine import Engine
    from beat_this_b200.weights import filter_hparams, pack_parameters

    ckpt = torch.load(small0_ckpt, weights_only=True)
    hp = filter_hparams(ckpt["hyper_parameters"])
    sd = {k.replace("model.", ""): v for k, v in ckpt["state_dict"].items()}
    assert Engine(pack_parameters(sd, hp, 1501), hp, "cuda:0").max_chunk == 1501
    packed = pack_parameters(sd, hp, 1500)
    long = pack_parameters(sd, hp, 384001)
    bad = [{"rope.cos": packed["rope.cos"][:-16], "rope.sin": packed["rope.sin"][:-16]},
           {"rope.cos": long["rope.cos"][: 1501 * 16 - 8], "rope.sin": long["rope.sin"][: 1501 * 16 - 8]},
           {"rope.cos": long["rope.cos"][: 1600 * 16], "rope.sin": long["rope.sin"][: 1601 * 16]},
           {"rope.cos": long["rope.cos"], "rope.sin": long["rope.sin"]}]
    for rope in bad:
        with pytest.raises(BTError, match="error -4"):
            Engine({**packed, **rope}, hp, "cuda:0")
