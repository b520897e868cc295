"""CPU test (no GPU) of the built library's machine code: the wgmma GEMM kernels of epilogue kinds 0 and 1 (every
linear layer and convolution of the 16-bit path) contain no function call.  A call anywhere in a kernel that issues
wgmma makes ptxas serialise all of its wgmma instructions (warning C7510), each MMA waiting for the previous one."""
import os
import re
import subprocess

from beat_this_b200 import _lib

# gemm_tc_kernel<BN, BK, KIND>; KIND 2 (the N = 32 attention gates) keeps the IEEE-division sigmoid
KERNEL = re.compile(r"_ZN2bt14gemm_tc_kernelILi(\d+)ELi(\d+)E(?:Li(\d+)E)?E")


def test_gemm_kernels_have_no_call(lib_built):
    cuobjdump = os.path.join(os.path.dirname(_lib._nvcc()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    calls, checked, fn = {}, set(), None
    for line in sass.splitlines():
        if "Function :" in line:
            m = KERNEL.search(line)
            fn = m.group(0) if m and m.group(3) != "2" else None
            if fn:
                checked.add(fn)
        elif fn and re.search(r"\bCALL\b", line):
            calls[fn] = calls.get(fn, 0) + 1
    assert checked, "no gemm_tc_kernel instantiation found in the library"
    assert not calls, f"CALL instructions in wgmma GEMM kernels: {calls}"
