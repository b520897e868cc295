"""Alternative kernel paths selected by environment switches (DESIGN.md "Environment switches").

The library reads the switches once per process, so every variant runs the kernel-level parity
tests (attention vs SDPA in float64, per-stage taps vs the oracle) in a fresh interpreter."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

VARIANTS = [
    {"BT_ATTN_VARIANT": "32"},                        # attention: every exponential on MUFU
    {"BT_ATTN_VARIANT": "40"},                        # ... 4 of every 8 score pairs on the packed FMA-pipe polynomial
    {"BT_ATTN_FREQ_SIMT": "1"},                       # CUDA-core frequency attention
    {"BT_FUSE_FF": "0"},                              # unfused frontend blocks (norm + GEMMs)
    {"BT_FUSE_OUTPROJ": "0"},                         # separate attention out-projection GEMM in front of the fused FFN
    {"BT_GATES_IN_NORM_MAX": "4"},                    # gates of the 4-head block inside the norm kernel
]


@pytest.mark.gpu
@pytest.mark.parametrize("env", VARIANTS, ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()))
def test_variant_kernel_parity(env, lib_built):
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run(
        [sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_kernels.py"), "-m", "gpu", "-q", "-x",
         "-p", "no:cacheprovider", "-k", "debug_attention or stage_parity_h16 or debug_gemm"],
        cwd=ROOT, env=e, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
