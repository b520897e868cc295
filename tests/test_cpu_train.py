"""The training parameter table (bt_train_param_count / bt_train_param_info, pure host) against the reference's
BeatThis.state_dict() layout, for every model family."""
import ctypes
import os

import pytest

from beat_this_b200 import _lib, synthetic

FAMILIES = ["small0", "small0-nosum", "small0-nopartial", "final0", "64", "1024"]
NO_GRAD = (".running_mean", ".running_var", ".num_batches_tracked", ".rotary_embed.freqs")


@pytest.mark.parametrize("family", FAMILIES)
def test_table_is_the_state_dict(family):
    hp = synthetic.model_hparams(family)
    table = _lib.train_param_table(hp)
    sd = synthetic.make_state_dict(hp)  # key order and shapes of the reference module (oracle/make_golden.py pins it)
    assert [name for name, _, _ in table] == list(sd)
    for name, shape, trainable in table:
        assert shape == tuple(sd[name].shape), name
        assert trainable == (not name.endswith(NO_GRAD)), name


def test_table_follows_the_hyper_parameters():
    hp = synthetic.model_hparams("small0")
    base = len(_lib.train_param_table(hp))
    assert len(_lib.train_param_table(dict(hp, n_layers=7))) == base + 11  # one attention (6) and one FFN (5)
    ff = dict(_lib.train_param_table(dict(hp, ff_mult=2, transformer_dim=192))[i][:2] for i in range(base))
    assert ff["transformer_blocks.layers.0.1.net.1.weight"] == (384, 192)
    assert ff["frontend.linear.weight"] == (192, 1024)


def test_param_info_refuses_bad_arguments():
    lib = _lib.load()
    hp = _lib.hparams_struct(synthetic.model_hparams("small0"))
    n = lib.bt_train_param_count(ctypes.byref(hp))
    name, shape, ndim, trainable = ctypes.create_string_buffer(64), (ctypes.c_int64 * 4)(), ctypes.c_int32(), \
        ctypes.c_int32()
    args = (shape, ctypes.byref(ndim), ctypes.byref(trainable))
    assert lib.bt_train_param_info(ctypes.byref(hp), 0, name, 64, *args) == 0
    assert name.value == b"frontend.stem.bn1d.weight" and ndim.value == 1 and shape[0] == 128 and trainable.value == 1
    assert lib.bt_train_param_info(ctypes.byref(hp), n, name, 64, *args) == -1
    assert lib.bt_train_param_info(ctypes.byref(hp), -1, name, 64, *args) == -1
    assert lib.bt_train_param_info(ctypes.byref(hp), 0, name, 5, *args) == -1  # name longer than the buffer
    assert lib.bt_train_param_count(None) == -1


def _golden_cases():
    import numpy as np

    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "train_grads.npz"))
    k = 0
    while f"family{k}" in z:
        yield k, {name[: -len(str(k))]: z[name] for name in z.files if name.endswith(str(k)) and
                  name[: -len(str(k))] in GOLDEN_KEYS}
        k += 1


GOLDEN_KEYS = {"family", "seed", "spect", "beat", "downbeat", "dbeat", "ddown", "dspect", "names", "fp"}


def test_oracle_gradients_match_the_reference_fixture():
    """The float64 restatement's gradients against the unmodified reference's (oracle/make_golden_train_grads.py)."""
    import numpy as np
    import torch

    from oracle import beat_this_oracle as O
    from oracle.train_fingerprint import bounds, fingerprint

    n_cases = 0
    for _, c in _golden_cases():
        family = str(c["family"])
        hp = synthetic.model_hparams(family)
        sd0 = synthetic.make_state_dict(hp, int(c["seed"]))
        names = [str(n) for n in c["names"]]
        assert names == [n for n, _, trainable in _lib.train_param_table(hp) if trainable]
        sd = {n: v.double().requires_grad_(n in names) for n, v in sd0.items()}
        x = torch.tensor(c["spect"], dtype=torch.float64, requires_grad=True)
        beat, down = O.forward(sd, x, sum_head=hp["sum_head"])
        assert np.abs(beat.detach().numpy() - c["beat"]).max() < 1e-5
        assert np.abs(down.detach().numpy() - c["downbeat"]).max() < 1e-5
        grads = torch.autograd.grad((beat, down), [x] + [sd[n] for n in names],
                                    (torch.tensor(c["dbeat"]), torch.tensor(c["ddown"])))
        ref = torch.tensor(c["dspect"])
        assert float((grads[0] - ref).norm() / ref.norm()) < 1e-6
        index = {n: i for i, n in enumerate(sd0)}
        for n, g, fp in zip(names, grads[1:], c["fp"]):
            i = index[n]
            assert (np.abs(fingerprint(g.numpy(), i) - fp) <= bounds(fp, g.numel(), i, 1e-6)).all(), n
        n_cases += 1
    assert n_cases == 4
