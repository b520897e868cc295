"""GPU tests of bt_finalize's parameter checks: the stem's packed arrays have the lengths stem_kernel reads."""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


@pytest.mark.parametrize("name", ["stem.bn1_scale", "stem.bn1_shift", "stem.bias"])
def test_finalize_checks_the_stem_lengths(small0_ckpt, lib_built, name):
    """stem.bn1_scale and stem.bn1_shift need spect_dim elements and stem.bias stem_dim: one element short is
    BT_ERR_PARAM, naming the parameter, before stem_kernel could read past its end."""
    from beat_this_b200._lib import BTError
    from beat_this_b200.engine import Engine
    from beat_this_b200.weights import filter_hparams, pack_parameters

    ckpt = torch.load(small0_ckpt, weights_only=True)
    hp = filter_hparams(ckpt["hyper_parameters"])
    packed = pack_parameters({k.replace("model.", ""): v for k, v in ckpt["state_dict"].items()}, hp)
    assert packed[name].size == (hp["spect_dim"] if "bn1" in name else hp["stem_dim"])
    with pytest.raises(BTError, match=f"error -4: .*'{name}'"):
        Engine({**packed, name: packed[name][:-1]}, hp, "cuda:0")
