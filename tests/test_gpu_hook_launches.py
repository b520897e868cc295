"""Launch accounting of the kernel test hooks (include/beatthis.h, "Kernel test hooks"): a call adds exactly the kernel
under test to bt_launch_count and to the profile, under its documented name, in every context the hook runs in; and
every hook also runs on a context created with BT_SYNC_DEBUG=1, where each launch is checked as it is made."""
import os

import numpy as np
import pytest
import torch

from support import dev  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

H16_ONLY = {"fused_qkv", "fused_ff"}


def _engines(dev):
    """Weight-less contexts: {False: fp32, True: 16-bit}."""
    from beat_this_b200.engine import Engine

    return {half: Engine(None, None, dev, half=half) for half in (False, True)}


@pytest.fixture(scope="module")
def engines(lib_built, dev):
    return _engines(dev)


@pytest.fixture(scope="module")
def sync_engines(lib_built, dev):
    """Contexts created under BT_SYNC_DEBUG=1 (bt_create reads it); the variable is restored afterwards."""
    old = os.environ.get("BT_SYNC_DEBUG")
    os.environ["BT_SYNC_DEBUG"] = "1"
    try:
        return _engines(dev)
    finally:
        if old is None:
            del os.environ["BT_SYNC_DEBUG"]
        else:
            os.environ["BT_SYNC_DEBUG"] = old


def _hooks(dev):
    """{hook: (call(engine), {profile name: launches})} on small valid inputs."""
    from beat_this_b200.dbn import _BarModel

    g = torch.Generator(device=dev).manual_seed(0)

    def r(*shape):
        return 0.1 * torch.randn(*shape, generator=g, device=dev)

    def z(*shape):
        return torch.zeros(*shape, device=dev)

    M, C, L, D = 13, 64, 16, 64
    q = [r(2, 70, 64) for _ in range(3)]  # 2 sequences of 70 tokens, 2 heads
    qf = [r(80, 64) for _ in range(3)] + [torch.rand(80, 2, generator=g, device=dev)]  # B 1, F 16, L 5, 2 heads
    rope = (r(1500, 16), r(1500, 16))
    ok = [(3, 10, -2, 3, 2, 12, 14)]  # bt_debug_chunk fields, as tests/test_gpu_chunk_kernels.py
    stem = [torch.ones(128, device=dev), z(128), z(32, 12), z(32)]
    m = _BarModel(3, 60.0 * 10 / 215.0, 60.0 * 10 / 55.0, None, 100, 16)
    dens = torch.from_numpy(m.log_densities(np.full((40, 2), 0.1))).to(dev)
    return {
        "gemm": (lambda e: e.debug_gemm(r(128, 64), r(64, 64)), {"debug_gemm": 1}),
        "attention": (lambda e: e.debug_attention(*q), {"debug_attention": 1}),
        "attention_freq": (lambda e: e.debug_attention_freq(*qf, 1, 16), {"debug_attention_freq": 1}),
        "norm": (lambda e: e.debug_norm(r(M, C), z(M, C), M, C), {"debug_norm": 1}),
        "fused_qkv": (lambda e: e.debug_fused_qkv(r(M, C), r(3 * C, C), r(2, C), r(2), *rope, z(M, 3 * C), z(M, 2), M, C,
                                                  13, 1, 0, 1.0), {"debug_fused_qkv": 1}),
        "fused_ff": (lambda e: e.debug_fused_ff(r(M, C), r(4 * C, C), r(4 * C), r(C, 4 * C), r(C), M, C),
                     {"debug_fused_ff": 1}),
        "stem": (lambda e: e.debug_stem(z(16, 128), ok, L, *stem, z(32 * L * 32)), {"stem": 1}),
        "zero_tail": (lambda e: e.debug_zero_tail(z(2 * 4 * L * 32), ok + ok, 4, L, 32), {"zero_tail": 1}),
        "head": (lambda e: e.debug_head(z(2 * L * D), D, z(2 * D), z(2), ok + [(3, 10, 0, 3, 0, 0, 1)], L, 1, z(16), z(16)),
                 {"head": 1}),
        "dbn_viterbi": (lambda e: e.debug_dbn_viterbi(dens, m.beats, m.intervals, m.log_tempo, m.pointers),
                        {"dbn_viterbi": 1, "dbn_backtrace": 1}),
    }


CASES = [(name, half) for name in ("gemm", "attention", "attention_freq", "norm", "fused_qkv", "fused_ff", "stem",
                                   "zero_tail", "head", "dbn_viterbi") for half in (False, True)
         if half or name not in H16_ONLY]


@pytest.mark.parametrize("name,half", CASES, ids=[f"{n}-{'16bit' if h else 'fp32'}" for n, h in CASES])
def test_hook_counts_and_profiles_only_the_kernel_under_test(engines, dev, name, half):
    eng = engines[half]
    call, names = _hooks(dev)[name]
    eng.profile_enable(True)
    try:
        eng.profile_reset()
        before = eng.launches
        call(eng)
        added = eng.launches - before
        prof = {k: n for k, (_, n) in eng.profile_results().items() if n}
    finally:
        eng.profile_enable(False)
    assert added == sum(names.values())
    assert prof == names


@pytest.mark.parametrize("half", [False, True])
def test_every_hook_runs_under_sync_debug(sync_engines, dev, half):
    eng = sync_engines[half]
    for name, (call, names) in _hooks(dev).items():
        if half or name not in H16_ONLY:
            before = eng.launches
            call(eng)
            assert eng.launches - before == sum(names.values()), name
