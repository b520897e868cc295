"""Plumbing more than one test file uses: the CUDA device and engine fixtures (import them by name), bit views,
repeat-launch checks, the built library's machine code, seeded inputs, and the training tests' model and bounds."""
import os
import subprocess

import pytest
import torch

NAN = float("nan")
DEV = "cuda:0"
GRAD_BOUND = 1e-4  # per tensor: ||g - g64|| / ||g64||
LOGIT_TOL = 1e-3   # the fp32 inference path's bound against the oracle (numerics.F32_TOL, smoke())


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device")
    return torch.device(DEV)


@pytest.fixture(scope="module")
def small_h16(small0_ckpt, lib_built, dev):
    from beat_this_b200.inference import load_model

    return load_model(small0_ckpt, DEV, float16=True)


def act_dtype(eng):
    """The torch type of an engine's 16-bit activations."""
    return torch.float16 if eng.act_dtype == "f16" else torch.bfloat16


def bits(t):
    """The bits of t as integers of its element size (4 or 2 bytes), for bitwise comparisons."""
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


def launch_twice(call, M, C, dev):
    """Two launches on fresh NaN buffers of M + 1 rows; returns the first after checking the sentinel row and bits."""
    outs = []
    for _ in range(2):
        out = torch.full(((M + 1) * C,), NAN, device=dev)
        call(out)
        outs.append(out)
    assert torch.equal(bits(outs[0]), bits(outs[1])), "a second launch gives other bits"
    assert torch.isnan(outs[0][M * C :]).all(), "store past the last row"
    return outs[0][: M * C].view(M, C).double()


def sass(lib):
    """The SASS of the built library (lib: the lib_built fixture, which builds it)."""
    from beat_this_b200 import _lib

    cuobjdump = os.path.join(os.path.dirname(_lib._nvcc()), "cuobjdump")
    return subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout


def rnd(*shape, g, scale=1.0):
    """fp32 N(0, scale^2) values of the given shape from generator g."""
    return (torch.randn(*shape, generator=g) * scale).float()


# ---- the training tests' model and inputs
def _module(family, seed=0, **overrides):
    """A module on a seeded synthetic checkpoint of `family`, with hyper-parameters overridden as given."""
    from beat_this_b200 import synthetic
    from beat_this_b200.train import BeatThisModule

    ckpt = synthetic.make_checkpoint(family, seed)
    if overrides:
        hp = dict(ckpt["hyper_parameters"], **overrides)
        ckpt = dict(ckpt, hyper_parameters=hp,
                    state_dict={"model." + k: v for k, v in synthetic.make_state_dict(hp, seed).items()})
    return BeatThisModule.from_checkpoint(ckpt, DEV), ckpt


def _spect(B, L, seed, lengths=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, L, 128, generator=g) * 4.0
    if lengths is not None:  # zero-padded as TrainingBatches yields a batch of shorter pieces
        for b, n in enumerate(lengths):
            x[b, n:] = 0
    return x


def _rel(g, ref):
    g = g.detach().double().cpu()
    return float((g - ref).norm() / ref.norm().clamp_min(1e-300))
