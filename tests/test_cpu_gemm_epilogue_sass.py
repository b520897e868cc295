"""CPU test (no GPU) of the staged epilogue of the wgmma GEMM in the built library's machine code.

Every gemm_tc_kernel of epilogue kind 0 or 1 writes its results through shared memory and TMA stores: it contains at
least one UTMASTG, no STG, and no global load but the read-only (.CONSTANT) loads of the bias and the RoPE tables.  The
residual arrives by TMA as well, so a residual read in registers (a load after the previous column's store, one HBM
round trip each) cannot come back unnoticed.  The gates GEMM (kind 2) keeps its register epilogue."""
import re

from gemm_reference import GEMM_TC_KERNEL as KERNEL
from support import sass


def _counts(listing):
    counts, fn = {}, None
    for line in listing.splitlines():
        if "Function :" in line:
            m = KERNEL.search(line)
            fn = (int(m.group(1)), int(m.group(2)), int(m.group(3) or 0)) if m else None
            if fn and fn[2] != 2:
                counts[fn] = {"UTMASTG": 0, "STG": 0, "LDG": 0}
            else:
                fn = None
        elif fn:
            c = counts[fn]
            c["UTMASTG"] += "UTMASTG" in line
            c["STG"] += bool(re.search(r"\bSTG\b", line))
            c["LDG"] += bool(re.search(r"\bLDG\b", line)) and ".CONSTANT" not in line
    return counts


def test_staged_gemm_epilogues_store_by_tma(lib_built):
    counts = _counts(sass(lib_built))
    assert len(counts) == 16, f"kind-0/1 instantiations found: {sorted(counts)}"
    bad = {k: c for k, c in counts.items() if c["UTMASTG"] == 0 or c["STG"] or c["LDG"]}
    for k in sorted(counts):
        print(f"gemm_tc_kernel<{k[0]}, {k[1]}, {k[2]}>: {counts[k]}")
    assert not bad, f"kernels with global stores, non-constant global loads or no TMA store: {bad}"
