"""CPU test (no GPU) of the dropout-mask restatement the training-mode tests use (oracle/philox.py): Philox4x32-10's
known answers, the keep rule and its element numbering, and the site numbering include/beatthis.h states."""
import os

import numpy as np

import torch

import train_mode_reference as TM
from beat_this_b200 import synthetic
from oracle import philox

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hex(words):
    return " ".join(f"{int(w):08x}" for w in words)


def test_philox_known_answers():
    assert _hex(philox.philox4x32_10((0, 0, 0, 0), (0, 0))) == "6627e8d5 e169c58d bc57ac4c 9b00dbd8"
    assert _hex(philox.philox4x32_10((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2)) == "408f276d 41c83b0e a20bc7c6 6d5451fd"
    assert _hex(philox.philox4x32_10((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0))) == \
        "d16cfe09 94fdcceb 5001e420 24126ea1"


def test_element_numbering():
    seed, site = 0x0123456789ABCDEF, 5
    for e0 in (0, 3, 2 ** 32 - 2, 5 * 2 ** 32 + 1):
        w = philox.words(seed, site, e0, 11)
        for k in range(11):
            e = e0 + k
            c = (e // 4) & 0xFFFFFFFF, (e // 4) >> 32, site, 0
            ref = philox.philox4x32_10(c, (seed & 0xFFFFFFFF, seed >> 32))[e % 4]
            assert int(w[k]) == int(ref)
    # a window is the same elements as the whole
    assert np.array_equal(philox.words(seed, site, 0, 40)[7:29], philox.words(seed, site, 7, 22))


def test_keep_rule():
    assert philox.threshold(0.0) == 0 and philox.keep(1, 2, 0.0, 9).all()
    assert philox.threshold(0.5) == 2 ** 31
    assert philox.threshold(0.9) == int(np.float32(0.9) * np.float64(2 ** 32)) != int(0.9 * 2 ** 32)  # the float rate
    w = philox.words(9, 3, 100, 1000)
    assert np.array_equal(philox.keep(9, 3, 0.25, 1000, 100), w >= 2 ** 30)


def test_site_numbering_is_the_header_s():
    header = open(os.path.join(ROOT, "include", "beatthis.h")).read()
    assert "site: 2 s + k for step s" in header
    assert "((s heads + h) n + i) n + j" in header
    assert [TM.site(s, k) for s in range(3) for k in range(2)] == [0, 1, 2, 3, 4, 5]


def test_fp32_itself_misses_1e4_on_biases_upstream_of_batch_statistics():
    """The conditioning behind the GPU tests' bias bound: torch's fp32 autograd of the training-mode restatement, on
    the case where the library's worst bias error was measured (small0-nosum, (3, 17), rates 0.5 / 0.9), misses float64
    by more than 1e-4 on a bias gradient, while every non-bias gradient stays within 1e-4."""
    family, B, L, seed, rates = "small0-nosum", 3, 17, 1234567, (0.5, 0.9)
    sd0 = {k.replace("model.", ""): v for k, v in synthetic.make_checkpoint(family, 0)["state_dict"].items()}
    x = torch.rand(B, L, 128, generator=torch.Generator().manual_seed(1)) * 4.0  # tests/test_gpu_train.py's _spect
    g = torch.Generator().manual_seed(2)
    dbeat, ddown = torch.randn(B, L, generator=g), torch.randn(B, L, generator=g)
    grads = {}
    for dt in (torch.float64, torch.float32):
        sd = {k: v.to(dt).requires_grad_(v.is_floating_point() and "running" not in k and "freqs" not in k)
              if v.is_floating_point() else v for k, v in sd0.items()}
        b, d, _ = TM.forward_train(sd, x.to(dt), seed, *rates, sum_head=False)
        names = [k for k, v in sd.items() if v.is_floating_point() and v.requires_grad]
        grads[dt] = dict(zip(names, torch.autograd.grad((b, d), [sd[n] for n in names], (dbeat.to(dt), ddown.to(dt)))))
    err = {n: float((grads[torch.float32][n].double() - r).norm() / r.norm()) for n, r in grads[torch.float64].items()}
    assert max(e for n, e in err.items() if n.endswith(".bias")) > 1e-4
    assert max(e for n, e in err.items() if not n.endswith(".bias")) <= 1e-4
