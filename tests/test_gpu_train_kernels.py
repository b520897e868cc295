"""Every training kernel (csrc/kernels_train.cu) alone through bt_debug_train_kernel against its float64 restatement
and elementwise bound (tests/train_kernels_reference.py).  Each case also runs twice for a bitwise repeat, starts its
outputs NaN-filled (an element never written stays NaN and fails), and pads every output with sentinels the kernel
must leave alone.  Refused geometries return BT_ERR_ARG without a launch.  The worst ratio to the bound per op is
printed (pytest -s) and kept in RATIOS."""
import math

import pytest
import torch

import train_kernels_reference as R
from beat_this_b200 import _lib
from beat_this_b200.engine import Engine
from numerics import REL_2ULP, worst
from support import rnd

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = "cuda:0"
PAD = 37           # sentinel elements after every output
SENTINEL = 1234.5
RATIOS = {}
COVERED = set()    # kernels the cases launch (tests/test_cpu_train_sass.py lists the library's)


@pytest.fixture(scope="module")
def eng(lib_built):
    return Engine(None, None, DEV)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def out(n):
    """An output of n elements, NaN-filled, followed by PAD sentinels: (device buffer, view of the n elements)."""
    b = torch.full((n + PAD,), math.nan, device=DEV)
    b[n:] = SENTINEL
    return b, b[:n]


def dev(t):
    return torch.as_tensor(t).float().contiguous().to(DEV)


def run(eng, op, arrays, **desc):
    """The op twice on fresh copies of the in/out arrays (in-place ops start from the given values): returns the
    arrays after the first run; asserts the second is bitwise the same and that every pad is untouched."""
    results = []
    for _ in range(2):
        bufs = []
        for a in arrays:
            if a is None:
                bufs.append(None)
            elif isinstance(a, tuple):  # (buffer with its pad, view): copy both
                bufs.append(a[0].clone())
            else:
                bufs.append(a.clone())
        views = [None if b is None else (b[: b.numel() - PAD] if isinstance(a, tuple) else b)
                 for a, b in zip(arrays, bufs)]
        eng.debug_train_kernel(op, views, **desc)
        torch.cuda.synchronize()
        results.append(bufs)
    for a, x, y in zip(arrays, *results):
        if x is None:
            continue
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f"{op}: not bitwise repeatable"
        if isinstance(a, tuple):
            assert (x[x.numel() - PAD:] == SENTINEL).all(), f"{op}: wrote past its output"
    COVERED.update(R.KERNELS[op])
    return [None if b is None else (b[: b.numel() - PAD] if isinstance(a, tuple) else b).cpu()
            for a, b in zip(arrays, results[0])]


def check(op, case, got, ref, bound):
    r = worst(got, ref, bound)
    RATIOS[op] = max(RATIOS.get(op, 0.0), r)
    assert r <= 1.0, f"{op} {case}: {r:.3g} x the bound"


def padded(t):
    """A device output initialised from t (in-place ops), followed by PAD sentinels."""
    b, v = out(t.numel())
    v.copy_(dev(t).reshape(-1))
    return b, v


# ------------------------------------------------------------------------------------ GEMM
def _gemm_case(eng, M, N, K, layout, splits, bias=False, resid=False, gelu=False, seed=0):
    g = _g(seed)
    A, B = rnd(M, K, g=g), rnd(N, K, g=g)
    # store A and B in the layout's memory order; A(m, k) at a_rs m + a_cs k
    if layout == "xw":      # X W^T: both row-major over K
        Am, a_rs, a_cs, Bm, b_rs, b_cs = A, K, 1, B, K, 1
    elif layout == "dyw":   # dY W: B stored [K, N] (W [N_out, K_in] read as B(n, k) = W[k, n])
        Am, a_rs, a_cs, Bm, b_rs, b_cs = A, K, 1, B.T.contiguous(), 1, N
    else:                   # dY^T X: A stored [K, M], B stored [K, N]
        Am, a_rs, a_cs, Bm, b_rs, b_cs = A.T.contiguous(), 1, M, B.T.contiguous(), 1, N
    bias_t = rnd(N, g=g) if bias else None
    resid_t = rnd(M, N, g=g) if resid else None
    eff = splits or _policy_splits(M, N, K)
    parts = -(-K // R.gemm_kc(K, eff))
    C = padded(resid_t) if resid else out(M * N)
    gel = out(M * N) if gelu else None
    part = out(parts * M * N) if parts > 1 else None
    arrays = [dev(Am).reshape(-1), dev(Bm).reshape(-1), C, None if bias_t is None else dev(bias_t),
              None, gel, part]
    if resid:  # resid aliases C, as grad_input runs it in place
        arrays[4] = "C"
    res = _run_alias(eng, arrays, M=M, N=N, K=K, a_rs=a_rs, a_cs=a_cs, b_rs=b_rs, b_cs=b_cs, ldc=N, ldr=N,
                     splits=splits, scale=1.0)
    ref, e, gref, ge = R.gemm_ref(A, B, bias_t, resid_t, splits=eff)
    case = f"M{M} N{N} K{K} {layout} splits {splits}->{eff}"
    check("gemm", case, res[2].reshape(M, N), ref, e)
    if gelu:
        check("gemm", case + " gelu", res[5].reshape(M, N), gref, ge)


def _run_alias(eng, arrays, **desc):
    """run() where slot 4 may be the string "C": resid is the C buffer itself."""
    if arrays[4] != "C":
        return run(eng, "gemm", arrays, **desc)
    results = []
    for _ in range(2):
        cb = arrays[2][0].clone()
        c = cb[: cb.numel() - PAD]
        bufs = [arrays[0], arrays[1], c, arrays[3], c,
                None if arrays[5] is None else arrays[5][0].clone(), None if arrays[6] is None else arrays[6][0].clone()]
        views = bufs[:5] + [None if b is None else b[: b.numel() - PAD] for b in bufs[5:]]
        eng.debug_train_kernel("gemm", views, **desc)
        torch.cuda.synchronize()
        assert (cb[cb.numel() - PAD:] == SENTINEL).all()
        results.append([cb[: cb.numel() - PAD].cpu()] + [None if b is None else b[: b.numel() - PAD].cpu()
                                                           for b in bufs[5:]])
    assert torch.equal(results[0][0], results[1][0])
    COVERED.update(R.KERNELS["gemm"])
    return [None, None, results[0][0], None, None, results[0][1], results[0][2]]


def _policy_splits(M, N, K):
    """tr_dw_splits of the GEMM's output (rows K of a weight gradient dW [M, N])."""
    tiles = -(-M // 64) * -(-N // 64)
    s = min(-(-264 // tiles), max(1, K // 256))
    return max(1, min(s, (8 << 20) // (M * N)))


GEMM_SHAPES = [(M, N, K) for M in (1, 63, 64, 65) for N in (1, 63, 65) for K in (1, 12, 15, 16, 17, 192)] + \
    [(130, 129, 4096)]


@pytest.mark.parametrize("layout", ["xw", "dyw", "dytx"])
def test_gemm_shapes(eng, layout):
    for i, (M, N, K) in enumerate(GEMM_SHAPES):
        _gemm_case(eng, M, N, K, layout, 1, seed=i)


def test_gemm_splits_and_epilogues(eng):
    for K in (17, 192, 4096, 4099):
        for splits in (1, 2, 0, 7):  # 7: a ragged last part
            _gemm_case(eng, 65, 63, K, "dytx", splits, seed=K + splits)
    _gemm_case(eng, 65, 130, 192, "xw", 1, bias=True, gelu=True)
    _gemm_case(eng, 65, 130, 192, "dyw", 1, resid=True)
    _gemm_case(eng, 64, 64, 16, "xw", 1, bias=True, resid=True, gelu=True)


@pytest.mark.parametrize("M,N,K", [(96, 32, 12000), (32, 512, 12000), (2048, 512, 12000), (512, 2048, 12000),
                                   (32, 12, 8 * 1500 * 32), (64, 192, 8 * 1500 * 4)])
def test_gemm_production_weight_gradients(eng, M, N, K):
    """dW = dY^T X at final0, B = 8, L = 1500 (12 000 rows), and frontend shapes over B L F rows, split as the
    training pass splits them."""
    _gemm_case(eng, M, N, K, "dytx", 0, seed=M + N)


# ------------------------------------------------------------------------------------ reductions
def test_colsum_and_reduce(eng):
    for N in (1, 2, 31, 32, 33, 1024, 4096):
        for M in (1, 7, 511, 512, 513, 1025, 3000):
            if M * N > 4 << 20:
                continue
            g = _g(M * 7 + N)
            A, B, rs = rnd(M, N, g=g), rnd(M, N, g=g), rnd(M, g=g)
            for splits, withB in ((0, False), (1, True), (3, True)):
                eff = splits or max(1, min(-(-M // 512), (8 << 20) // N))
                _, Z = R.colsum_parts(M, eff)
                res = run(eng, "colsum", [dev(A).reshape(-1), dev(B).reshape(-1) if withB else None,
                                          dev(rs) if withB else None, out(Z * N), out(N)], M=M, N=N, splits=splits,
                          scale=0.5)
                ref, e, parts, ep = R.colsum_ref(A, B if withB else None, rs if withB else None, eff, 0.5)
                check("colsum", f"M{M} N{N} s{splits}", res[4], ref, e)
                check("colsum", f"M{M} N{N} s{splits} parts", res[3].reshape(Z, N), parts, ep)
    for Z, n in ((1, 1), (2, 33), (7, 1000), (23, 4097)):
        part = rnd(Z, n, g=_g(Z))
        res = run(eng, "reduce", [dev(part).reshape(-1), out(n)], M=n, splits=Z, scale=0.25)
        ref, e = R.reduce_ref(part, 0.25)
        check("reduce", f"Z{Z} n{n}", res[1], ref, e)


# ------------------------------------------------------------------------------------ RMSNorm
@pytest.mark.parametrize("C", [32, 64, 128, 256, 512, 1024])
def test_rmsnorm(eng, C):
    g = _g(C)
    M = 37
    x = rnd(M, C, g=g)
    x[3] = 0
    for i, nrm in zip((4, 5, 6), (1e-13, 1e-12, 1e-11)):  # clamped, at the clamp and just above it
        x[i] = x[i] / x[i].norm() * nrm
    x[7] = rnd(C, g=g, scale=1e-20)
    gamma = rnd(C, g=g)
    res = run(eng, "rms_fwd", [dev(x).reshape(-1), dev(gamma), out(M * C), out(M)], M=M, C=C)
    xn, e, inv, ei = R.rms_fwd_ref(x, gamma)
    check("rms_fwd", f"C{C}", res[2].reshape(M, C), xn, e)
    check("rms_fwd", f"C{C} inv", res[3], inv, ei)
    dxn, dres0 = rnd(M, C, g=g), rnd(M, C, g=g)
    inv32 = res[3]
    for add in (0, 1):
        d = padded(dres0) if add else out(M * C)
        r2 = run(eng, "rms_bwd", [dev(dxn).reshape(-1), dev(x).reshape(-1), dev(inv32), dev(gamma), d], M=M, C=C,
                 flag=add)
        ref, eb = R.rms_bwd_ref(dxn, x, inv32, gamma, dres0 if add else None)
        check("rms_bwd", f"C{C} add{add}", r2[4].reshape(M, C), ref, eb)


# ------------------------------------------------------------------------------------ BatchNorm, GELU
def _bn(C, g):
    return (rnd(C, g=g), rnd(C, g=g), rnd(C, g=g), 0.5 + torch.rand(C, generator=g).float())


@pytest.mark.parametrize("C", [1, 32, 64, 128, 33])
def test_bn_gelu(eng, C):
    g = _g(C + 100)
    n = C * 301
    bn = _bn(C, g)
    z = rnd(n, g=g, scale=3.0)
    bnd = [dev(a) for a in bn]
    res = run(eng, "bn_gelu_fwd", [dev(z), *bnd, out(n)], M=n, C=C)
    ref, e = R.bn_gelu_fwd_ref(z, bn, C)
    check("bn_gelu_fwd", f"C{C}", res[5], ref, e)
    dy = rnd(n, g=g)
    res = run(eng, "bn_gelu_bwd", [dev(dy), dev(z), *bnd, out(n), out(n)], M=n, C=C)
    dbn, e1, dz, e2 = R.bn_gelu_bwd_ref(dy, z, bn, C)
    check("bn_gelu_bwd", f"C{C} dbn", res[6], dbn, e1)
    check("bn_gelu_bwd", f"C{C} dz", res[7], dz, e2)
    sgz, sg = rnd(C, g=g, scale=30.0), rnd(C, g=g, scale=30.0)
    res = run(eng, "bn_grads", [dev(sgz), dev(sg), *bnd, out(C), out(C)], C=C)
    dw, ew, db = R.bn_grads_ref(sgz, sg, bn)
    check("bn_grads", f"C{C}", res[6], dw, ew)
    assert torch.equal(res[7], sg)
    res = run(eng, "bn_scale", [dev(dy), *bnd, out(n)], M=n, C=C)
    ref, e = R.bn_scale_ref(dy, bn, C)
    check("bn_scale", f"C{C}", res[5], ref, e)


def test_gelu_bwd_sweep(eng):
    h = torch.linspace(-12, 12, 200001).float()
    h = torch.cat([h, torch.tensor([-0.7517916, -0.75179, -0.7518, 0.0, -0.0, 1e-30])])  # GELU' = 0 near -0.7518
    n = h.numel()
    da = rnd(n, g=_g(5))
    res = run(eng, "gelu_bwd", [dev(da), dev(h), out(n)], M=n)
    ref, e = R.gelu_bwd_ref(da, h)
    check("gelu_bwd", "sweep", res[2], ref, e)
    # in place: dh is da
    buf = dev(da)
    eng.debug_train_kernel("gelu_bwd", [buf, dev(h), buf], M=n)
    torch.cuda.synchronize()
    check("gelu_bwd", "in place", buf.cpu(), ref, e)


# ------------------------------------------------------------------------------------ convolution slabs, concat
def _img(kind, B, L):
    """(TrImg tuple, input elements) of the stem (S 4, C 1 over [B, L, 128]) or a conv block (S 2) of C, F."""
    if kind == "stem":
        Fo, S, C = 32, 4, 1
        return (B, Fo, S, L, C, L * 128, 1, 128, 0), B * L * 128
    C, Fi = {"conv0": (32, 32), "conv1": (64, 16), "conv2": (128, 8)}[kind]
    return (B, Fi // 2, 2, L, C, Fi * L * C, L * C, C, 1), B * Fi * L * C


@pytest.mark.parametrize("kind", ["stem", "conv0", "conv1", "conv2"])
@pytest.mark.parametrize("L", [1, 2, 17, 1500])
def test_im2col_col2im(eng, kind, L):
    B = 2 if L < 1500 else 1
    gm, n_in = _img(kind, B, L)
    Bq, Fo, S, Lq, C = gm[:5]
    K = C * S * 3
    rows = B * Fo * L
    g = _g(L)
    x = rnd(n_in, g=g)
    desc = dict(B=Bq, F=Fo, S=S, L=Lq, C=C, sb=gm[5], sf=gm[6], st=gm[7], sc=gm[8])
    res = run(eng, "im2col", [dev(x), out(rows * K)], **desc)
    ref, _ = R.im2col_ref(x, gm)
    assert torch.equal(res[1].double(), ref.reshape(-1)), "im2col without BatchNorm is a gather"
    COVERED.add("tr_im2col_kernel")
    if kind == "stem":
        bn = _bn(Fo * S, g)
        res = run(eng, "im2col", [dev(x), out(rows * K), *[dev(a) for a in bn]], flag=1, **desc)
        ref, e = R.im2col_ref(x, gm, bn)
        check("im2col", f"{kind} L{L} bn", res[1].reshape(rows, K), ref, e)
    dcol = rnd(rows * K, g=g)
    res = run(eng, "col2im", [dev(dcol), out(n_in)], **desc)
    ref, e = R.col2im_ref(dcol, gm, n_in)
    check("col2im", f"{kind} L{L}", res[1], ref, e)
    if L <= 17:  # the float64 adjoint: <im2col(x), y> = <x, col2im(y)>
        lhs = float((R.im2col_ref(x, gm)[0].reshape(-1) * dcol.double()).sum())
        rhs = float((x.double() * ref).sum())
        assert abs(lhs - rhs) <= 1e-9 * (1 + abs(lhs))


@pytest.mark.parametrize("B,F,L,C", [(1, 1, 1, 1), (2, 4, 17, 256), (3, 8, 5, 128)])
def test_concat_and_head(eng, B, F, L, C):
    n = B * F * L * C
    x = rnd(n, g=_g(n))
    for bw in (0, 1):
        res = run(eng, "concat", [dev(x), out(n)], B=B, F=F, L=L, C=C, flag=bw)
        assert torch.equal(res[1].double(), R.concat_ref(x, B, F, L, C, bw))
    RATIOS["concat"] = 0.0
    M = B * L
    o, db, dd = rnd(M, 2, g=_g(1)), rnd(M, g=_g(2)), rnd(M, g=_g(3))
    for sh in (0, 1):
        res = run(eng, "head_fwd", [dev(o).reshape(-1), out(M), out(M)], M=M, flag=sh)
        beat, down = R.head_fwd_ref(o, sh)
        assert torch.equal(res[1].double(), beat.float().double()) and torch.equal(res[2].double(), down)
        res = run(eng, "head_bwd", [dev(db), dev(dd), out(2 * M)], M=M, flag=sh)
        assert torch.equal(res[2].double(), R.head_bwd_ref(db, dd, sh).float().double())
    RATIOS["head_fwd"] = RATIOS["head_bwd"] = 0.0


# ------------------------------------------------------------------------------------ RoPE, gates
def _freqs():
    return (1.0 / 10000 ** (torch.arange(0, 32, 2).float() / 32)).float()


@pytest.mark.parametrize("posmode,F,L,M,C", [(0, 1, 1500, 3000, 512), (0, 1, 384000, 384000, 32),
                                             (1, 32, 17, 32 * 17 * 2, 32), (1, 16, 5, 16 * 5 * 3, 64),
                                             (1, 8, 3, 8 * 3 * 2, 128)])
def test_rope(eng, posmode, F, L, M, C):
    qkv = rnd(M, 3 * C, g=_g(M))
    fr = _freqs()
    for inv in (0, 1):
        res = run(eng, "rope", [padded(qkv), dev(fr)], M=M, C=C, L=L, F=F, posmode=posmode, flag=inv)
        ref, e = R.rope_ref(qkv, fr, L, F, posmode, inv)
        got = res[0].reshape(M, 3 * C)
        check("rope", f"pm{posmode} M{M} inv{inv}", got, ref, e)
        assert torch.equal(got[:, 2 * C:], qkv[:, 2 * C:]), "v columns changed"
    fwd = run(eng, "rope", [padded(qkv), dev(fr)], M=M, C=C, L=L, F=F, posmode=posmode, flag=0)[0]
    back = run(eng, "rope", [padded(fwd), dev(fr)], M=M, C=C, L=L, F=F, posmode=posmode, flag=1)[0]
    ident = (REL_2ULP + 3 * R.U) * 4 * (qkv.abs().reshape(M, 3 * C) + qkv.abs().reshape(M, 3 * C).roll(1, 1)
                                      + qkv.abs().reshape(M, 3 * C).roll(-1, 1)).double() + 1e-37
    check("rope", f"pm{posmode} identity", back.reshape(M, 3 * C), qkv.double(), ident)


@pytest.mark.parametrize("M,C", [(1, 32), (77, 64), (300, 512), (33, 1024)])
def test_gates(eng, M, C):
    g = _g(M + C)
    O, dG = rnd(M, C, g=g), rnd(M, C, g=g)
    gl = torch.linspace(-30, 30, M * (C // 32)).float()[torch.randperm(M * (C // 32), generator=g)]
    res = run(eng, "gate_fwd", [dev(O).reshape(-1), dev(gl), out(M * C)], M=M, C=C)
    G, e = R.gate_fwd_ref(O, gl.reshape(M, C // 32))
    check("gate_fwd", f"M{M} C{C}", res[2].reshape(M, C), G, e)
    H = C // 32
    res = run(eng, "gate_bwd", [padded(dG), dev(O).reshape(-1), dev(gl), out(M * H), out(M * H)], M=M, C=C)
    dO, e0, dg, e1, delta, e2 = R.gate_bwd_ref(dG, O, gl.reshape(M, H))
    check("gate_bwd", f"M{M} C{C} dO", res[0].reshape(M, C), dO, e0)
    check("gate_bwd", f"M{M} C{C} dg", res[3].reshape(M, H), dg, e1)
    check("gate_bwd", f"M{M} C{C} delta", res[4].reshape(M, H), delta, e2)


# ------------------------------------------------------------------------------------ attention
def _attn_inputs(tokens, H, family, g):
    C = 32 * H
    qkv = rnd(tokens, 3 * C, g=g)
    if family == "dominant":
        qkv[:, :C] *= 4.0
        qkv[:, C:2 * C] *= 4.0
    elif family == "flat":
        qkv[:, :C] *= 1e-3
    elif family == "large":  # |scores| near 80
        qkv[:, :C] = qkv[:, :C] / qkv[:, :C].norm(dim=1, keepdim=True) * 16.0
        qkv[:, C:2 * C] = qkv[:, C:2 * C] / qkv[:, C:2 * C].norm(dim=1, keepdim=True) * 28.0
    return qkv


def _seqs_desc(layout, n, H, nseq):
    if layout == "time":  # sequences (b, f) over t: TrSeqs {B F, L, heads, 1, L, 0, 1}
        return dict(seqs=nseq, n=n, heads=H, seq_in=1, s_out=n, s_in=0, s_pos=1), nseq * n
    B, L = nseq  # frequency: sequences (b, t) over f: {B L, F, heads, L, F L, 1, L}
    return dict(seqs=B * L, n=n, heads=H, seq_in=L, s_out=n * L, s_in=1, s_pos=L), B * n * L


ATTN_CASES = [("time", n, H, 2, fam) for n in (1, 31, 32, 33, 63, 64, 65) for H in (1, 2) for fam in ("random",)] + \
    [("time", 1500, 1, 1, fam) for fam in ("random", "dominant", "flat", "large")] + \
    [("time", 65, 16, 1, "random"), ("time", 33, 32, 1, "large")] + \
    [("freq", F, H, (2, L), fam) for F, H in ((32, 1), (16, 2), (8, 4)) for L in (1, 17)
     for fam in ("random", "dominant", "flat", "large")]


@pytest.mark.parametrize("layout,n,H,nseq,family", ATTN_CASES)
def test_attention(eng, layout, n, H, nseq, family):
    desc, tokens = _seqs_desc(layout, n, H, nseq)
    C = 32 * H
    g = _g(n * 131 + H)
    qkv = _attn_inputs(tokens, H, family, g)
    rows = R.seq_rows(desc["seqs"], n, desc["seq_in"], desc["s_out"], desc["s_in"], desc["s_pos"])
    res = run(eng, "attn_fwd", [dev(qkv).reshape(-1), out(tokens * C), out(tokens * H)], **desc)
    O, eO, lse, el = R.attn_fwd_ref(qkv, rows, H)
    got_O = R._heads(res[1].double().reshape(tokens, C), rows, H, 0, C)
    got_l = res[2].double().reshape(tokens, H)[rows.reshape(-1)].reshape(rows.shape[0], n, H).permute(0, 2, 1)
    check("attn_fwd", f"{layout} n{n} H{H} {family}", got_O, O, eO)
    check("attn_fwd", f"{layout} n{n} H{H} {family} lse", got_l.reshape(-1, n), lse, el)
    # the backward on float64 lse and delta (rounded to fp32) of a random dO
    dO = rnd(tokens, C, g=g)
    Ofull = R.heads_back(O, rows, H, tokens, 0, C)
    lse_t = torch.zeros(tokens, H, dtype=torch.float64)
    lse_t[rows.reshape(-1)] = lse.reshape(rows.shape[0], H, n).permute(0, 2, 1).reshape(-1, H)
    delta_t = (dO.double() * Ofull).reshape(tokens, H, 32).sum(-1)
    lse32, delta32 = lse_t.float(), delta_t.float()
    dq, edq, dk, edk, dv, edv = R.attn_bwd_ref(qkv, dO, lse32, delta32, rows, H)
    ins = [dev(qkv).reshape(-1), dev(dO).reshape(-1), dev(lse32).reshape(-1), dev(delta32).reshape(-1)]
    res = run(eng, "attn_dq", ins + [out(tokens * 3 * C)], **desc)
    got = res[4].double().reshape(tokens, 3 * C)
    check("attn_dq", f"{layout} n{n} H{H} {family}", R._heads(got, rows, H, 0, C), dq, edq)
    assert torch.isnan(got[:, C:]).all(), "dq wrote the k / v columns"
    res = run(eng, "attn_dkv", ins + [out(tokens * 3 * C)], **desc)
    got = res[4].double().reshape(tokens, 3 * C)
    check("attn_dkv", f"{layout} n{n} H{H} {family} dk", R._heads(got, rows, H, C, C), dk, edk)
    check("attn_dkv", f"{layout} n{n} H{H} {family} dv", R._heads(got, rows, H, 2 * C, C), dv, edv)
    assert torch.isnan(got[:, :C]).all(), "dkv wrote the q columns"


# ------------------------------------------------------------------------------------ refusals
def _refused(eng, op, arrays, **desc):
    before = eng.launches
    with pytest.raises(_lib.BTError, match="error -1"):
        eng.debug_train_kernel(op, arrays, **desc)
    assert eng.launches == before


def test_refused_geometries(eng):
    z = lambda n: torch.zeros(n, device=DEV)  # noqa: E731
    M, N, K = 8, 8, 8
    g = dict(M=M, N=N, K=K, a_rs=K, a_cs=1, b_rs=K, b_cs=1, ldc=N, ldr=N, splits=1, scale=1.0)
    _refused(eng, "gemm", [z(M * K - 1), z(N * K), z(M * N)], **g)                 # A too short
    _refused(eng, "gemm", [z(M * K), z(N * K), z(M * N - 1)], **g)                 # C too short
    _refused(eng, "gemm", [z(M * K), z(N * K), z(M * N)], **dict(g, a_rs=-1))     # negative stride
    _refused(eng, "gemm", [z(M * K), z(N * K), z(M * N)], **dict(g, ldc=N - 1))   # ldc < N
    _refused(eng, "gemm", [z(M * 64), z(N * 64), z(M * N), z(N), None, None, z(4 * M * N)],
             **dict(g, K=64, a_rs=64, b_rs=64, splits=2))                          # split with a bias
    _refused(eng, "gemm", [z(M * 64), z(N * 64), z(M * N), None, None, None, z(M * N)],
             **dict(g, K=64, a_rs=64, b_rs=64, splits=2))                          # part too short
    _refused(eng, "reduce", [z(15), z(8)], M=8, splits=2)
    _refused(eng, "colsum", [z(M * N), None, None, z(N - 1), z(N)], M=M, N=N, splits=1)
    _refused(eng, "rms_fwd", [z(M * 32), z(32), z(M * 32), z(M - 1)], M=M, C=32)
    _refused(eng, "bn_gelu_bwd", [z(64), z(64), z(32), z(32), z(32), z(31), z(64), z(64)], M=64, C=32)
    _refused(eng, "im2col", [z(3 * 128 - 1), z(32 * 3 * 12)], B=1, F=32, S=4, L=3, C=1, sb=3 * 128,
             sf=1, st=128, sc=0)
    _refused(eng, "im2col", [z(128 * 3), z(32 * 3 * 12), z(128), z(128), z(128)], B=1, F=32, S=4, L=3, C=1,
             sb=3 * 128, sf=1, st=128, sc=0, flag=1)                               # BatchNorm without rv
    _refused(eng, "rope", [z(10 * 96 - 1), z(16)], M=10, C=32, L=10, F=1, posmode=0)
    _refused(eng, "rope", [z(10 * 96), z(16)], M=10, C=48, L=10, F=1, posmode=0)
    _refused(eng, "gate_bwd", [z(64), z(64), z(2), z(2), z(1)], M=2, C=32)
    a = dict(seqs=2, n=5, heads=1, seq_in=1, s_out=5, s_in=0, s_pos=1)
    _refused(eng, "attn_fwd", [z(10 * 96 - 1), z(10 * 32), z(10)], **a)
    _refused(eng, "attn_fwd", [z(10 * 96 + 1)[1:], z(10 * 32), z(10)], **a)       # qkv not 16-byte aligned
    _refused(eng, "attn_dq", [z(10 * 96), z(10 * 32 + 1)[1:], z(10), z(10), z(10 * 96)], **a)
    _refused(eng, "attn_dkv", [z(10 * 96), z(10 * 32), z(10), z(9), z(10 * 96)], **a)
    _refused(eng, "attn_fwd", [z(14 * 96), z(14 * 32), z(14)], **dict(a, s_out=6, s_pos=2))  # row 14 past the arrays
    _refused(eng, "head_bwd", [z(8), z(8), z(15)], M=8)
    with pytest.raises(_lib.BTError):
        Engine(None, None, DEV, half=True).debug_train_kernel("head_fwd", [z(16), z(8), z(8)], M=8)


def test_zz_every_kernel_covered_and_report():
    """Runs last: every training kernel was launched by some case, and the worst ratios are printed."""
    want = {k for ks in R.KERNELS.values() for k in ks}
    assert want <= COVERED, f"not launched: {sorted(want - COVERED)}"
    for op in sorted(RATIOS):
        print(f"train kernel {op:12s} worst |err| / bound = {RATIOS[op]:.3g}")
