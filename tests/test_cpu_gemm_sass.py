"""CPU tests (no GPU) of the wgmma GEMM: its machine code in the built library and the coverage of its unit tests.

The GEMM kernels of epilogue kinds 0 and 1 (every linear layer and convolution of the 16-bit path) contain no function
call: a call anywhere in a kernel that issues wgmma makes ptxas serialise all of its wgmma instructions (warning
C7510), each MMA waiting for the previous one.  Every instantiation of the kernel in the library has a case in the GPU
unit tests (tests/gemm_reference.py), so a new tile or epilogue cannot ship untested."""
import re

import torch

from gemm_reference import GEMM_CASES, GEMM_TC_KERNEL as KERNEL, GEMM_TILES
from numerics import gelu_erf, gelu_tanh, rope_ref
from support import sass


def test_gemm_kernels_have_no_call(lib_built):
    calls, checked, fn = {}, set(), None
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            m = KERNEL.search(line)
            fn = m.group(0) if m and m.group(3) != "2" else None
            if fn:
                checked.add(fn)
        elif fn and re.search(r"\bCALL\b", line):
            calls[fn] = calls.get(fn, 0) + 1
    assert checked, "no gemm_tc_kernel instantiation found in the library"
    assert not calls, f"CALL instructions in wgmma GEMM kernels: {calls}"


def test_every_gemm_instantiation_has_a_unit_test(lib_built):
    """The (BN, BK, KIND) instantiations in the SASS are exactly GEMM_TILES, and the GPU cases reach each of them
    (the GPU test asserts that the plan of every case picks the tile expected_tile names)."""
    found = set()
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            m = KERNEL.search(line)
            if m:
                found.add((int(m.group(1)), int(m.group(2)), int(m.group(3) or 0)))
    assert found == set(GEMM_TILES), f"in the library only: {sorted(found - set(GEMM_TILES))}, " \
                                     f"listed only: {sorted(set(GEMM_TILES) - found)}"
    assert len(GEMM_TILES) == 18
    reached = {(*c.tile, c.kind) for c in GEMM_CASES}
    assert set(GEMM_TILES) <= reached, f"instantiations without a case: {sorted(set(GEMM_TILES) - reached)}"
    ids = [c.id for c in GEMM_CASES]
    assert len(ids) == len(set(ids))


def test_gelu_tanh_form_gap():
    """epilogue.cuh: the tanh-form GELU of the 16-bit path differs from the exact erf form by <= 5e-4 absolute."""
    x = torch.linspace(-12, 12, 2_400_001, dtype=torch.float64)
    gap = (gelu_erf(x) - gelu_tanh(x)).abs().max().item()
    print(f"max |gelu_erf - gelu_tanh| = {gap:.3e}")
    assert gap <= 5e-4


def test_rope_reference_is_oracle_rope():
    """The per-row rotation the GEMM tests apply with the fp32 tables equals oracle.rope (interleaved pairs)."""
    from beat_this_b200.weights import rope_tables
    from oracle import beat_this_oracle as O

    freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
    cos, sin = rope_tables(freqs)
    x = torch.randn(3, 1500, 64, generator=torch.Generator().manual_seed(0))
    ref = torch.stack([torch.cat([O.rope(x[s, :, 32 * h : 32 * h + 32], freqs) for h in range(2)], -1) for s in range(3)])
    got = rope_ref(x.double().reshape(-1, 64), cos.double().repeat(3, 1), sin.double().repeat(3, 1)).view(3, 1500, 64)
    assert (got - ref.double()).abs().max().item() < 1e-5  # oracle.rope rotates in fp32
