"""Paths of the C library that allocate or drop device resources outside the steady state: the bounded plan cache
evicting and rebuilding geometries, and a call rejected after it has allocated.  Both must leave the context giving
exactly the results of a fresh one."""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


def _h16_engine(ckpt):
    from beat_this_b200.inference import load_model

    return load_model(ckpt, "cuda:0", float16=True).engine


def _chunk(T, seed):
    return torch.randn(1, T, 128, generator=torch.Generator().manual_seed(seed)).cuda().contiguous()


def test_plan_cache_eviction_rebuilds_identical_plans(small0_ckpt, lib_built):
    """50 chunk lengths are 50 plan geometries; the cache keeps 48, so the first three lengths are evicted and rebuilt
    when they come round again."""
    eng = _h16_engine(small0_ckpt)
    lengths = list(range(100, 150))
    first = {T: eng.forward_chunks(_chunk(T, T)) for T in lengths}
    again = {T: eng.forward_chunks(_chunk(T, T)) for T in lengths[:3]}
    fresh = _h16_engine(small0_ckpt)
    for T, (beat, down) in again.items():
        fb, fd = fresh.forward_chunks(_chunk(T, T))
        assert torch.equal(beat, first[T][0]) and torch.equal(down, first[T][1]), T
        assert torch.equal(beat, fb) and torch.equal(down, fd), T


def test_rejection_after_allocation_leaves_context_usable(small0_ckpt, lib_built):
    """F = 8 with one head passes the argument check of bt_debug_attention_freq and allocates its buffers; only plan
    creation then rejects it."""
    from beat_this_b200._lib import BTError

    g = torch.Generator().manual_seed(0)

    def qkv_gates(B, F, L, heads):
        M, C = B * F * L, heads * 32
        return [torch.randn(M, C, generator=g).cuda() for _ in range(3)] + [torch.rand(M, heads, generator=g).cuda()]

    eng = _h16_engine(small0_ckpt)
    with pytest.raises(BTError, match="no tensor-core kernel"):
        eng.debug_attention_freq(*qkv_gates(1, 8, 5, 1), 1, 8)
    args = qkv_gates(2, 16, 7, 2)
    chunks = torch.randn(2, 300, 128, generator=g).cuda()
    fresh = _h16_engine(small0_ckpt)
    assert torch.equal(eng.debug_attention_freq(*args, 2, 16), fresh.debug_attention_freq(*args, 2, 16))
    for a, b in zip(eng.forward_chunks(chunks), fresh.forward_chunks(chunks)):
        assert torch.equal(a, b)
