"""CPU test (no GPU) of the training kernels' machine code in the built library: the set of tr_* kernels equals the
set tests/test_gpu_train_kernels.py launches (train_kernels_reference.KERNELS), so a new training kernel without a
unit test fails here; and no training kernel touches local memory except tr_rope_kernel, whose 32-byte stack frame
holds the slow path of cosf / sinf (the Payne-Hanek reduction of large angles)."""
import re

from support import sass
from train_kernels_reference import KERNELS

NAME = re.compile(r"Function : _ZN2bt(\d+)(tr_\w+?_kernel)")


def _kernels(listing):
    """{kernel name: [local-memory instructions]} of the tr_* kernels."""
    out, cur = {}, None
    for line in listing.splitlines():
        if "Function :" in line:
            m = NAME.search(line)
            cur = m.group(2) if m else None
            if cur:
                out[cur] = []
        elif cur and re.search(r"\b(STL|LDL)(\.\w+)*\b", line):
            out[cur].append(line.split(";")[0].strip())
    return out


def test_every_training_kernel_has_a_unit_test(lib_built):
    found = set(_kernels(sass(lib_built)))
    tested = {k for ks in KERNELS.values() for k in ks}
    assert found == tested, f"without a unit test: {sorted(found - tested)}; not in the library: {sorted(tested - found)}"


def test_no_training_kernel_spills(lib_built):
    local = {k: v for k, v in _kernels(sass(lib_built)).items() if v and k != "tr_rope_kernel"}
    assert not local, f"local-memory accesses: {local}"
