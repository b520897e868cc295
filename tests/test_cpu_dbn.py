"""CPU checks (no GPU) of the device DBN post-processor's host side: the command line option, the one place the tracker
parameters come from, and the machine code of the kernels in the built library."""
import os
import re
import subprocess

import pytest

from beat_this_b200 import _lib


def test_cli_dbn_impl_option():
    from beat_this_b200 import cli

    args = cli.build_parser().parse_args(["a.wav", "--dbn"])
    assert args.dbn and args.dbn_impl == "auto"
    for impl in ("auto", "madmom", "native", "device"):
        assert cli.build_parser().parse_args(["a.wav", "--dbn", "--dbn-impl", impl]).dbn_impl == impl
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["a.wav", "--dbn-impl", "gpu"])


def test_track_params_are_the_trackers():
    from beat_this_b200.dbn import DBNDownBeatTracker

    p = DBNDownBeatTracker().track_params
    assert p == dict(beats_per_bar=[3, 4], min_bpm=55.0, max_bpm=215.0, num_tempi=60, transition_lambda=100.0,
                     observation_lambda=16.0, threshold=0.05, correct=True, fps=50.0)
    p = DBNDownBeatTracker(num_tempi=None, correct=False, threshold=None).track_params
    assert p["num_tempi"] == 0 and p["correct"] is False and p["threshold"] == 0.0


def test_library_exports_the_device_dbn(lib_built):
    for name in ("bt_dbn_track_device", "bt_debug_dbn_viterbi"):
        assert hasattr(lib_built, name)


def _kernel_sass(name):
    cuobjdump = os.path.join(os.path.dirname(_lib._nvcc()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    body, inside = [], False
    for line in sass.splitlines():
        if "Function :" in line:
            inside = name in line
        elif inside:
            body.append(line)
    assert body, f"{name} not found in the library"
    return "\n".join(body)


def test_viterbi_kernel_adds_without_fma(lib_built):
    """The Viterbi recursion is adds and compares only: an FMA would round differently from the host decoder."""
    sass = _kernel_sass("dbn_viterbi_kernel")
    assert re.search(r"\bDADD\b", sass) and not re.search(r"\bDFMA\b", sass)
    assert not re.search(r"\b(STL|LDL)\b", sass), "local memory (spills) in dbn_viterbi_kernel"
