"""CPU test (no GPU) of the time-direction attention's machine code in the built library: attn_time_kernel keeps its
whole key loop in registers.  A spill puts local-memory loads and stores into the loop that every key tile runs."""
import re

from support import sass

KERNEL = re.compile(r"_ZN2bt16attn_time_kernelE")


def test_attn_time_kernel_has_no_local_memory_access(lib_built):
    local, fn, found = [], False, False
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            fn = bool(KERNEL.search(line))
            found |= fn
        elif fn and re.search(r"\b(STL|LDL)\b", line):
            local.append(line.split(";")[0].strip())
    assert found, "attn_time_kernel not found in the library"
    assert not local, f"local-memory accesses (spills) in attn_time_kernel: {local}"
