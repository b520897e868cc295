"""The launch schedule of the forward pass: which kernel classes one bt_spect2frames call launches, and how often.

One wave of three clips (two of 1500+ frames, one short), so the wave is varlen and every coupling between
neighbouring layers runs: fused out-projections, the 16-bit copy in front of each convolution, zero_tail, and the
last convolution writing frontend.linear's input.  The tables were recorded at the commit before the forward pass
was driven from one layer list; the classes are the names bench.py's kernel_time_shares reports."""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

FRAME_OFFSETS = [0, 1600, 3300, 3600]  # 2 + 2 chunks of 1500 frames and one of 312

SCHEDULES = {
    ("final0", True): ({
        "attn_freq": 3, "attn_time_tc": 9, "ff_fused_c32": 2, "ff_fused_c64": 2, "gemm_attn_out": 6,
        "gemm_attn_out_front": 2, "gemm_conv": 3, "gemm_ff1": 6, "gemm_ff1_front": 2, "gemm_ff2": 6,
        "gemm_ff2_front": 2, "gemm_frontend_linear": 1, "gemm_gates": 6, "gemm_gates_front": 2, "gemm_qkv": 6,
        "gemm_qkv_front": 2, "head": 1, "norm": 12, "norm_front": 4, "qkv_fused_c32": 2, "qkv_fused_c64": 2,
        "stem": 1, "zero_tail": 3,
    }, 85),
    ("final0", False): ({
        "attn_freq": 3, "attn_time_simt": 9, "gemm_attn_out": 6, "gemm_attn_out_front": 6, "gemm_conv": 3,
        "gemm_ff1": 6, "gemm_ff1_front": 6, "gemm_ff2": 6, "gemm_ff2_front": 6, "gemm_frontend_linear": 1,
        "gemm_gates": 6, "gemm_gates_front": 2, "gemm_qkv": 6, "gemm_qkv_front": 6, "head": 1, "norm": 12,
        "norm_front": 8, "norm_gates": 4, "stem": 1, "zero_tail": 3,
    }, 101),
    ("small0-nopartial", True): ({
        "attn_time_tc": 6, "f32_to_h16": 3, "gemm_attn_out": 6, "gemm_conv": 3, "gemm_ff1": 6, "gemm_ff2": 6,
        "gemm_frontend_linear": 1, "gemm_gates": 6, "gemm_qkv": 6, "head": 1, "norm": 12, "stem": 1, "zero_tail": 3,
    }, 60),
    ("small0-nosum", True): ({
        "attn_freq": 3, "attn_time_tc": 9, "ff_fused_c32": 2, "ff_fused_c64": 2, "gemm_attn_out": 6,
        "gemm_attn_out_front": 2, "gemm_conv": 3, "gemm_ff1": 6, "gemm_ff1_front": 2, "gemm_ff2": 6,
        "gemm_ff2_front": 2, "gemm_frontend_linear": 1, "gemm_gates": 6, "gemm_gates_front": 2, "gemm_qkv": 6,
        "gemm_qkv_front": 2, "head": 1, "norm": 12, "norm_front": 4, "qkv_fused_c32": 2, "qkv_fused_c64": 2,
        "stem": 1, "zero_tail": 3,
    }, 85),
}


def schedule(ckpt, half):
    """({kernel class: launches}, bt_launch_count) of one forward pass over FRAME_OFFSETS."""
    from beat_this_b200.inference import load_model

    eng = load_model(ckpt, "cuda:0", float16=half).engine
    spect = torch.rand(FRAME_OFFSETS[-1], 128, generator=torch.Generator().manual_seed(0)).cuda() * 7
    eng.profile_enable(True)
    eng.profile_reset()
    n0 = eng.launches
    eng.spect2frames_cat(spect, FRAME_OFFSETS)
    counts = {k: n for k, (_, n) in eng.profile_results().items() if n}
    return counts, eng.launches - n0


@pytest.mark.parametrize("name,half", list(SCHEDULES), ids=lambda v: v if isinstance(v, str) else ("h16" if v else "fp32"))
def test_launch_schedule(name, half, lib_built):
    from conftest import ckpt_path

    counts, launches = schedule(ckpt_path(name), half)
    want_counts, want_launches = SCHEDULES[(name, half)]
    assert counts == want_counts
    assert launches == want_launches
