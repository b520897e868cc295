"""ctypes binding of libbeatthis_sm90.so (C ABI in include/beatthis.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``beat_this_b200._lib.build()``
(nvcc, sm_90a).  There is no fallback: if the shared object is missing or no sm_90 GPU is
present, loading / ``bt_create`` fails loudly.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_void_p

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# BT_LIB_PATH: an instrumented build of the same sources (e.g. build(extra_flags=("-DBT_FF_PROF",), out_path=...))
LIB_PATH = os.environ.get("BT_LIB_PATH") or os.path.join(HERE, "libbeatthis_sm90.so")
SOURCES = ["bt_api.cu", "api_signal.cu", "api_post.cu", "api_data.cu", "api_train.cu", "api_debug.cu", "kernels_simt.cu", "kernels_misc.cu", "kernels_signal.cu", "kernels_gemm.cu", "kernels_attn.cu", "kernels_fused.cu", "kernels_dbn.cu", "kernels_eval.cu", "kernels_loss.cu", "kernels_data.cu", "kernels_train.cu", "kernels_optim.cu", "kernels_dp.cu", "kernels_flac.cu", "api_flac.cu", "kernels_mp3.cu", "api_mp3.cu", "kernels_vorbis.cu", "api_vorbis.cu", "dbn_host.cpp", "host_stage.cpp"]
HEADERS = ["common.cuh", "epilogue.cuh", "fft.cuh", "tc_common.cuh", "chunk_table.cuh", "flac.cuh", "mp3.cuh", "vorbis.cuh", "host_pool.h", "bt_kernels.h", "bt_train.h", "cuda_owned.h",
           "dbn_model.h",
           "api_internal.h", os.path.join("..", "..", "include", "beatthis.h")]

BT_DTYPE_F32 = 0
BT_DTYPE_H16 = 1


class bt_wav_info(ctypes.Structure):
    _fields_ = [
        ("sample_rate", c_int32),
        ("channels", c_int32),
        ("bytes_per_sample", c_int32),
        ("is_float", c_int32),
        ("frames", c_int64),
        ("data_offset", c_int64),
    ]


class bt_flac_info(ctypes.Structure):
    _fields_ = [
        ("sample_rate", c_int32),
        ("channels", c_int32),
        ("bits_per_sample", c_int32),
        ("min_block", c_int32),
        ("max_block", c_int32),
        ("reserved_", c_int32),
        ("total_samples", c_int64),
        ("frames_offset", c_int64),
        ("frames_bytes", c_int64),
        ("max_frames", c_int64),
        ("md5", ctypes.c_uint8 * 16),
    ]


class bt_flac_frame(ctypes.Structure):
    _fields_ = [
        ("offset", c_int64),
        ("first_sample", c_int64),
        ("bytes", c_int32),
        ("block_size", c_int32),
    ]


class bt_flac_stream(ctypes.Structure):
    _fields_ = [
        ("byte_offset", c_int64),
        ("byte_count", c_int64),
        ("frame_offset", c_int64),
        ("n_frames", c_int64),
        ("n_samples", c_int64),
        ("out_offset", c_int64),
        ("channels", c_int32),
        ("bits_per_sample", c_int32),
    ]


BT_FLAC_MONO_F32 = 0
BT_FLAC_CHANNELS_F64 = 1


class bt_mp3_info(ctypes.Structure):
    _fields_ = [
        ("sample_rate", c_int32),
        ("channels", c_int32),
        ("n_frames", c_int64),
        ("n_samples", c_int64),
        ("skip", c_int64),
        ("padding", c_int64),
        ("frames_offset", c_int64),
        ("frames_bytes", c_int64),
        ("max_frames", c_int64),
        ("main_bytes", c_int64),
        ("gapless", c_int32),
        ("reserved_", c_int32),
    ]


class bt_mp3_frame(ctypes.Structure):
    _fields_ = [
        ("main_start", c_int64),
        ("first_sample", c_int64),
        ("header", ctypes.c_uint32),
        ("main_bytes", c_int32),
        ("side_info", ctypes.c_uint8 * 32),
    ]


class bt_mp3_stream(ctypes.Structure):
    _fields_ = [
        ("byte_offset", c_int64),
        ("byte_count", c_int64),
        ("frame_offset", c_int64),
        ("n_frames", c_int64),
        ("skip", c_int64),
        ("n_samples", c_int64),
        ("out_offset", c_int64),
        ("channels", c_int32),
        ("sample_rate", c_int32),
    ]


# the MP3 output modes are FLAC's
BT_MP3_MONO_F32 = BT_FLAC_MONO_F32
BT_MP3_CHANNELS_F64 = BT_FLAC_CHANNELS_F64


class bt_vorbis_info(ctypes.Structure):
    _fields_ = [
        ("sample_rate", c_int32),
        ("channels", c_int32),
        ("blocksize0", c_int32),
        ("blocksize1", c_int32),
        ("n_packets", c_int64),
        ("packet_bytes", c_int64),
        ("table_bytes", c_int64),
        ("skip", c_int64),
        ("n_samples", c_int64),
    ]


class bt_vorbis_packet(ctypes.Structure):
    _fields_ = [
        ("byte_offset", c_int64),
        ("end_sample", c_int64),
        ("block_offset", c_int64),
        ("bytes", c_int32),
        ("mode", ctypes.c_uint8),
        ("blockflag", ctypes.c_uint8),
        ("prev_long", ctypes.c_uint8),
        ("next_long", ctypes.c_uint8),
    ]


class bt_vorbis_stream(ctypes.Structure):
    _fields_ = [
        ("byte_offset", c_int64),
        ("byte_count", c_int64),
        ("table_offset", c_int64),
        ("table_bytes", c_int64),
        ("packet_offset", c_int64),
        ("n_packets", c_int64),
        ("block_samples", c_int64),
        ("skip", c_int64),
        ("n_samples", c_int64),
        ("out_offset", c_int64),
        ("channels", c_int32),
        ("sample_rate", c_int32),
    ]


# the Vorbis output modes are FLAC's
BT_VORBIS_MONO_F32 = BT_FLAC_MONO_F32
BT_VORBIS_CHANNELS_F64 = BT_FLAC_CHANNELS_F64


class bt_hparams(ctypes.Structure):
    _fields_ = [
        ("spect_dim", c_int32),
        ("transformer_dim", c_int32),
        ("ff_mult", c_int32),
        ("n_layers", c_int32),
        ("head_dim", c_int32),
        ("stem_dim", c_int32),
        ("sum_head", c_int32),
        ("partial_transformers", c_int32),
    ]


class bt_debug_gemm_desc(ctypes.Structure):
    _fields_ = [
        ("planes_out", c_int32),
        ("planes_in", c_int32),
        ("L", c_int32),
        ("N", c_int32),
        ("Kslab", c_int32),
        ("nslab", c_int32),
        ("plane_mul", c_int32),
        ("lda", c_int32),
        ("plane_add", c_int32 * 6),
        ("t_shift", c_int32 * 6),
        ("resid_epilogue", c_int32),
        ("kind", c_int32),
        ("gelu", c_int32),
        ("C", c_int32),
        ("heads", c_int32),
        ("posmode", c_int32),
        ("F", c_int32),
        ("qscale", c_float),
    ]


class bt_debug_train_desc(ctypes.Structure):
    _fields_ = [
        ("op", c_int32),
        ("splits", c_int32),
        ("M", c_int64),
        ("N", c_int32),
        ("K", c_int32),
        ("C", c_int32),
        ("flag", c_int32),
        ("scale", c_float),
        ("a_rs", c_int64),
        ("a_cs", c_int64),
        ("b_rs", c_int64),
        ("b_cs", c_int64),
        ("ldc", c_int64),
        ("ldr", c_int64),
        ("B", c_int32),
        ("F", c_int32),
        ("L", c_int32),
        ("S", c_int32),
        ("posmode", c_int32),
        ("heads", c_int32),
        ("sb", c_int64),
        ("sf", c_int64),
        ("st", c_int64),
        ("sc", c_int64),
        ("seqs", c_int32),
        ("n", c_int32),
        ("seq_in", c_int32),
        ("pad_", c_int32),
        ("s_out", c_int64),
        ("s_in", c_int64),
        ("s_pos", c_int64),
        ("seed", ctypes.c_uint64),
        ("p", c_float),
        ("site", ctypes.c_uint32),
        ("e0", c_int64),
        ("beta", c_float),
        ("pad2_", c_int32),
        ("bn_n", c_int64),
    ]


class bt_train_mode(ctypes.Structure):
    _fields_ = [
        ("seed", ctypes.c_uint64),
        ("dropout_frontend", c_float),
        ("dropout_transformer", c_float),
    ]


class bt_adamw_entry(ctypes.Structure):
    _fields_ = [
        ("param", c_void_p),
        ("grad", c_void_p),
        ("exp_avg", c_void_p),
        ("exp_avg_sq", c_void_p),
        ("numel", c_int64),
        ("lr", c_double),
        ("beta1", c_double),
        ("beta2", c_double),
        ("eps", c_double),
        ("weight_decay", c_double),
        ("step", c_int64),
    ]


class bt_grad_entry(ctypes.Structure):
    _fields_ = [
        ("grad", c_void_p),
        ("numel", c_int64),
    ]


# bt_debug_train_kernel's ops (BT_TRAIN_*), in the order of include/beatthis.h
TRAIN_OPS = ("gemm", "reduce", "colsum", "rms_fwd", "rms_bwd", "bn_gelu_fwd", "bn_gelu_bwd", "bn_grads", "bn_scale",
             "gelu_bwd", "im2col", "col2im", "concat", "rope", "gate_fwd", "gate_bwd", "head_fwd", "head_bwd", "attn_fwd",
             "attn_dq", "attn_dkv")


class bt_beat_metric_params(ctypes.Structure):
    _fields_ = [
        ("min_beat_time", c_double),
        ("f_window", c_double),
        ("cemgil_sigma", c_double),
        ("phase_threshold", c_double),
        ("period_threshold", c_double),
    ]


BT_CHUNK = 1500
MAX_CHUNK_CAP = 256 * BT_CHUNK  # the longest maximum chunk bt_finalize accepts (RoPE tables of up to this many rows)
BT_KEEP_FIRST = 0
BT_KEEP_LAST = 1
OVERLAP_MODES = {"keep_first": BT_KEEP_FIRST, "keep_last": BT_KEEP_LAST}
DEFAULT_CHUNKING = (BT_CHUNK, 6, "keep_first")  # what Spect2Frames.spect2frames uses (reference inference.py:244-254)


class bt_chunking(ctypes.Structure):
    _fields_ = [
        ("chunk_size", c_int32),
        ("border", c_int32),
        ("overlap_mode", c_int32),
    ]


class bt_loss_params(ctypes.Structure):
    _fields_ = [
        ("kind", c_int32),
        ("tolerance", c_int32),
        ("pos_weight", c_float),
    ]


class bt_debug_chunk(ctypes.Structure):
    _fields_ = [
        ("frame_base", c_int64),
        ("T", c_int32),
        ("start", c_int32),
        ("out_base", c_int64),
        ("write_lo", c_int32),
        ("write_hi", c_int32),
        ("len", c_int32),
    ]


BT_MEL_NORM_NONE = 0
BT_MEL_NORM_FRAME_LENGTH = 1
BT_MEL_NORM_WINDOW = 2


class bt_mel_config(ctypes.Structure):
    _fields_ = [
        ("n_fft", c_int32),
        ("hop_length", c_int32),
        ("n_mels", c_int32),
        ("norm_mode", c_int32),
        ("power", c_float),
        ("log_multiplier", c_float),
    ]


class bt_stft_config(ctypes.Structure):
    _fields_ = [
        ("n_fft", c_int32),
        ("hop_length", c_int32),
    ]


VOCODER_RATE_RANGE = (0.25, 4.0)  # BT_VOCODER_MIN_RATE, BT_VOCODER_MAX_RATE


# every symbol include/beatthis.h declares: name -> (restype, argtypes)
PROTOTYPES = {
    "bt_version": (c_int, []),
    "bt_act_dtype": (c_char_p, []),
    "bt_create": (c_int, [POINTER(c_void_p), c_int, POINTER(bt_hparams), c_int]),
    "bt_set_param": (c_int, [c_void_p, c_char_p, POINTER(c_float), c_int64]),
    "bt_finalize": (c_int, [c_void_p]),
    "bt_destroy": (None, [c_void_p]),
    "bt_last_error": (c_char_p, [c_void_p]),
    "bt_num_frames": (c_int64, [c_int64]),
    "bt_plan_chunks": (c_int64, [c_int64, POINTER(c_int64), POINTER(c_int64), c_int64]),
    "bt_plan_chunking": (
        c_int64, [c_int64, POINTER(bt_chunking), POINTER(c_int64), POINTER(c_int64), POINTER(c_int64), POINTER(c_int64), c_int64],
    ),
    "bt_plan_chunking_max": (
        c_int64,
        [c_int64, POINTER(bt_chunking), c_int32, POINTER(c_int64), POINTER(c_int64), POINTER(c_int64), POINTER(c_int64),
         c_int64],
    ),
    "bt_max_chunk": (c_int32, [c_void_p]),
    "bt_logmel": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, POINTER(c_int64), c_void_p]),
    "bt_logmel_config": (
        c_int,
        [c_void_p, POINTER(bt_mel_config), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64),
         c_int32, c_void_p, POINTER(c_int64), c_void_p],
    ),
    "bt_stage_audio": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_int32]),
    "bt_wav_probe": (c_int, [c_char_p, POINTER(bt_wav_info)]),
    "bt_stage_wav_files": (c_int, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_void_p]),
    "bt_flac_probe": (c_int, [c_char_p, POINTER(bt_flac_info)]),
    "bt_stage_flac_files": (
        c_int, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p],
    ),
    "bt_flac_decode": (
        c_int, [c_void_p, c_void_p, c_void_p, POINTER(bt_flac_stream), c_int32, c_int32, c_void_p, c_void_p, c_void_p],
    ),
    "bt_debug_flac_decode_host": (
        c_int, [c_void_p, c_void_p, POINTER(bt_flac_stream), c_int32, c_int32, c_void_p, c_void_p],
    ),
    "bt_mp3_probe": (c_int, [c_char_p, POINTER(bt_mp3_info)]),
    "bt_stage_mp3_files": (
        c_int, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p],
    ),
    "bt_mp3_decode": (
        c_int, [c_void_p, c_void_p, c_void_p, POINTER(bt_mp3_stream), c_int32, c_int32, c_void_p, c_void_p, c_void_p],
    ),
    "bt_debug_mp3_decode_host": (
        c_int, [c_void_p, c_void_p, POINTER(bt_mp3_stream), c_int32, c_int32, c_void_p, c_void_p],
    ),
    "bt_vorbis_probe": (c_int, [c_char_p, POINTER(bt_vorbis_info)]),
    "bt_stage_vorbis_files": (
        c_int, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                c_int32, c_void_p],
    ),
    "bt_vorbis_decode": (
        c_int, [c_void_p, c_void_p, c_void_p, POINTER(bt_vorbis_stream), c_int32, c_int32, c_void_p, c_void_p, c_void_p],
    ),
    "bt_debug_vorbis_decode_host": (
        c_int, [c_void_p, c_void_p, POINTER(bt_vorbis_stream), c_int32, c_int32, c_void_p, c_void_p],
    ),
    "bt_resample": (
        c_int,
        [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_int32, c_int32, c_int32, c_void_p, POINTER(c_int64), c_void_p],
    ),
    "bt_dbn_track": (
        c_int,
        [c_void_p, c_void_p, c_int32, c_void_p, c_int32, ctypes.c_double, ctypes.c_double, c_int32, ctypes.c_double,
         ctypes.c_double, ctypes.c_double, c_int32, ctypes.c_double, c_int32, c_void_p, c_void_p, c_void_p],
    ),
    "bt_dbn_viterbi": (
        c_int,
        [c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "bt_dbn_track_device": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_int32, c_double, c_double, c_int32,
         c_double, c_double, c_double, c_int32, c_double, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "bt_debug_dbn_viterbi": (
        c_int,
        [c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "bt_beat_metrics": (
        c_int, [c_void_p, c_void_p, POINTER(c_int64), c_void_p, POINTER(c_int64), c_int32, POINTER(bt_beat_metric_params),
                c_void_p, c_void_p],
    ),
    "bt_beat_loss": (
        c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_int32, POINTER(bt_loss_params), c_void_p,
                c_void_p, c_void_p],
    ),
    "bt_beat_loss_backward": (
        c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_int32, POINTER(bt_loss_params), c_void_p,
                c_void_p, c_void_p],
    ),
    "bt_stft": (
        c_int,
        [c_void_p, POINTER(bt_stft_config), c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p,
         POINTER(c_int64), c_void_p],
    ),
    "bt_phase_vocoder": (
        c_int,
        [c_void_p, c_int32, c_void_p, POINTER(c_int64), c_int32, POINTER(c_int32), POINTER(c_double), c_int32, c_void_p,
         POINTER(c_int64), c_void_p],
    ),
    "bt_istft": (
        c_int,
        [c_void_p, POINTER(bt_stft_config), c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p,
         POINTER(c_int64), c_void_p],
    ),
    "bt_train_batch": (
        c_int,
        [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_int32, POINTER(c_int32), POINTER(c_int32), POINTER(c_int64),
         POINTER(c_int32), POINTER(c_int64), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "bt_train_param_count": (c_int32, [POINTER(bt_hparams)]),
    "bt_train_param_info": (
        c_int, [POINTER(bt_hparams), c_int32, c_char_p, c_int32, POINTER(c_int64), POINTER(c_int32), POINTER(c_int32)],
    ),
    "bt_train_activation_bytes": (c_int64, [c_void_p, c_int32, c_int32]),
    "bt_train_forward": (
        c_int, [c_void_p, POINTER(c_void_p), c_int32, c_void_p, c_int32, c_int32, c_void_p, c_int64, c_void_p, c_void_p,
                c_void_p],
    ),
    "bt_train_backward": (
        c_int, [c_void_p, POINTER(c_void_p), c_int32, c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p,
                POINTER(c_void_p), c_void_p, c_void_p],
    ),
    "bt_train_activation_bytes_ex": (c_int64, [c_void_p, c_int32, c_int32, POINTER(bt_train_mode)]),
    "bt_train_forward_ex": (
        c_int, [c_void_p, POINTER(c_void_p), c_int32, POINTER(c_void_p), c_void_p, c_int32, c_int32,
                POINTER(bt_train_mode), c_void_p, c_int64, c_void_p, c_void_p, c_void_p],
    ),
    "bt_train_backward_ex": (
        c_int, [c_void_p, POINTER(c_void_p), c_int32, c_void_p, c_int64, c_int32, c_int32, POINTER(bt_train_mode),
                c_void_p, c_void_p, POINTER(c_void_p), c_void_p, c_void_p],
    ),
    "bt_adamw_step": (c_int, [c_void_p, POINTER(bt_adamw_entry), c_int32, c_void_p]),
    "bt_grad_pack": (c_int, [c_void_p, POINTER(bt_grad_entry), c_int32, c_void_p, c_void_p]),
    "bt_grad_ordered_sum": (c_int, [c_void_p, POINTER(bt_grad_entry), c_int32, POINTER(c_void_p), c_int32, c_void_p]),
    "bt_train_running_replay": (
        c_int, [c_void_p, POINTER(c_void_p), c_int32, POINTER(c_void_p), c_int32, c_int32, c_int32, c_void_p],
    ),
    "bt_debug_attention_backward": (
        c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p,
                c_void_p],
    ),
    "bt_debug_train_kernel": (
        c_int, [c_void_p, POINTER(bt_debug_train_desc), POINTER(c_void_p), POINTER(c_int64), c_int32, c_void_p],
    ),
    "bt_spect2frames": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_void_p]),
    "bt_forward_chunks": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "bt_audio2frames": (
        c_int,
        [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, POINTER(c_int64), c_void_p],
    ),
    "bt_spect2frames_chunked": (
        c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, POINTER(bt_chunking), c_void_p],
    ),
    "bt_audio2frames_chunked": (
        c_int,
        [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, POINTER(c_int64), POINTER(bt_chunking), c_void_p],
    ),
    "bt_peakpick": (
        c_int,
        [c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p],
    ),
    "bt_peakpick_fps": (
        c_int,
        [c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_int32, c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_int32,
         c_void_p],
    ),
    "bt_set_wave_chunks": (c_int, [c_void_p, c_int32]),
    "bt_launch_count": (c_int64, [c_void_p]),
    "bt_profile_enable": (c_int, [c_void_p, c_int]),
    "bt_profile_collect": (c_int, [c_void_p]),
    "bt_profile_reset": (c_int, [c_void_p]),
    "bt_profile_count": (c_int, [c_void_p]),
    "bt_profile_get": (c_int, [c_void_p, c_int, c_char_p, c_int, POINTER(c_double), POINTER(c_int64)]),
    "bt_debug_request_tap": (c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    "bt_debug_tap_count": (c_int64, [c_void_p]),
    "bt_debug_gemm": (
        c_int,
        [c_void_p, POINTER(bt_debug_gemm_desc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
         c_void_p, c_void_p, POINTER(c_int32), c_void_p],
    ),
    "bt_debug_attention": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_int32, POINTER(c_int32),
         c_int32, c_void_p],
    ),
    "bt_debug_attention_freq": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_int32, c_int32, c_void_p],
    ),
    "bt_debug_norm": (
        c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_int32, c_void_p],
    ),
    "bt_debug_fused_qkv": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32,
         c_int32, c_int32, c_int32, c_float, c_void_p],
    ),
    "bt_debug_fused_ff": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32,
         c_void_p],
    ),
    "bt_debug_stem": (
        c_int,
        [c_void_p, c_void_p, c_int64, POINTER(bt_debug_chunk), c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
         c_void_p, c_int64, c_void_p],
    ),
    "bt_debug_zero_tail": (
        c_int, [c_void_p, c_void_p, c_int32, POINTER(bt_debug_chunk), c_int32, c_int32, c_int32, c_int32, c_int64, c_void_p],
    ),
    "bt_debug_head": (
        c_int,
        [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, POINTER(bt_debug_chunk), c_int32, c_int32, c_int32, c_void_p,
         c_void_p, c_int64, c_void_p],
    ),
}

_lib = None


OBJ_DIR = os.path.join(CSRC, "_obj")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def hparams_struct(hp: dict) -> bt_hparams:
    """The bt_hparams of a BeatThis hyper-parameter dict (the reference's defaults for missing entries)."""
    return bt_hparams(
        int(hp.get("spect_dim", 128)),
        int(hp.get("transformer_dim", 512)),
        int(hp.get("ff_mult", 4)),
        int(hp.get("n_layers", 6)),
        int(hp.get("head_dim", 32)),
        int(hp.get("stem_dim", 32)),
        int(bool(hp.get("sum_head", True))),
        int(bool(hp.get("partial_transformers", True))),
    )


def train_param_table(hp: dict) -> list[tuple[str, tuple, bool]]:
    """bt_train_param_info of every entry: (state_dict name, shape, takes a gradient), in the table's order."""
    lib = load()
    chp = hparams_struct(hp)
    n = lib.bt_train_param_count(ctypes.byref(chp))
    if n < 0:
        raise ValueError(f"bt_train_param_count refused {hp}")
    name, shape, ndim, trainable = ctypes.create_string_buffer(256), (c_int64 * 4)(), c_int32(), c_int32()
    table = []
    for i in range(n):
        code = lib.bt_train_param_info(ctypes.byref(chp), i, name, 256, shape, ctypes.byref(ndim), ctypes.byref(trainable))
        if code != 0:
            raise RuntimeError(f"bt_train_param_info({i}) returned {code}")
        table.append((name.value.decode(), tuple(shape[: ndim.value]), bool(trainable.value)))
    return table


def _nvcc() -> str:
    return os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def nvcc_command(out_path: str = LIB_PATH) -> list[str]:
    """The one-shot command line equivalent to what build() does (documentation / manual builds)."""
    return [_nvcc(), *NVCC_FLAGS, "-shared", *[os.path.join(CSRC, s) for s in SOURCES], "-o", out_path]


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, extra_flags: tuple = (), out_path: str = LIB_PATH) -> str:
    """Compile the CUDA library for sm_90a (cross-compiles without a GPU): one nvcc -c per source, in parallel,
    objects cached under csrc/_obj (keyed by flags), then one link step."""
    from concurrent.futures import ThreadPoolExecutor

    if not (force or out_path != LIB_PATH or needs_build()):
        return LIB_PATH
    tag = "".join(c if c.isalnum() else "_" for c in "".join(extra_flags)) or "default"
    odir = os.path.join(OBJ_DIR, tag)
    os.makedirs(odir, exist_ok=True)
    hdr_t = max(os.path.getmtime(os.path.join(CSRC, h)) for h in HEADERS)

    def compile_one(src):
        sp = os.path.join(CSRC, src)
        obj = os.path.join(odir, os.path.splitext(src)[0] + ".o")
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(sp), hdr_t):
            return obj, None
        cmd = [_nvcc(), *NVCC_FLAGS, *extra_flags, "-c", sp, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        res = subprocess.run(cmd, capture_output=True, text=True)
        return obj, (None if res.returncode == 0 else f"{src}:\n{res.stdout}\n{res.stderr}")

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 1)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    errors = [e for _, e in results if e]
    if errors:
        raise RuntimeError("nvcc failed:\n" + "\n".join(errors))
    tmp = out_path + f".tmp{os.getpid()}"
    cmd = [_nvcc(), "-shared", *ARCH, *[o for o, _ in results], "-o", tmp]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc link failed:\n{res.stdout}\n{res.stderr}")
    os.replace(tmp, out_path)
    return out_path


def load() -> ctypes.CDLL:
    """Load the shared library and declare all prototypes.  Fails loudly when absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: the sm_90a CUDA library has not been built. Run "
            "`python -c 'import __graft_entry__ as g; g.build()'` (or beat_this_b200._lib.build()). "
            "There is no CPU or PyTorch fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


class BTError(RuntimeError):
    pass


def check(lib, ctx, code: int):
    if code != 0:
        msg = lib.bt_last_error(ctx)
        raise BTError(f"libbeatthis error {code}: {msg.decode() if msg else ''}")


def i64_array(values):
    arr = (c_int64 * len(values))(*[int(v) for v in values])
    return arr


def i32_array(values):
    """An int32 host table as a C array argument: a pointer that keeps its contiguous copy alive.  It goes through
    numpy because such tables can be long (a training batch's row maps have B * L entries)."""
    return np.ascontiguousarray(values, dtype=np.int32).ctypes.data_as(POINTER(c_int32))


def offsets(lengths) -> list:
    """CSR offsets of consecutive lengths: [0, l0, l0 + l1, ...]."""
    out = [0]
    for n in lengths:
        out.append(out[-1] + int(n))
    return out


# ---- entry points without a context --------------------------------------------------------------------------------
SIG_F32, SIG_F64, SIG_I16 = 0, 1, 2
SIGNAL_DTYPES = {np.dtype(np.float32): SIG_F32, np.dtype(np.float64): SIG_F64, np.dtype(np.int16): SIG_I16}


def stage_audio(arrays, dst, threads: int) -> list:
    """bt_stage_audio: mono mix + fp32 cast of C-contiguous ndarrays of SIGNAL_DTYPES (pipeline.as_signal_array) into
    `dst` (host fp32 tensor) on `threads` host threads; returns the sample offsets."""
    n = len(arrays)
    so = offsets(a.shape[0] for a in arrays)
    ptrs = (c_void_p * n)(*[a.ctypes.data for a in arrays])
    dts = (c_int32 * n)(*[SIGNAL_DTYPES[a.dtype] for a in arrays])
    frames = (c_int64 * n)(*[a.shape[0] for a in arrays])
    chans = (c_int32 * n)(*[1 if a.ndim == 1 else a.shape[1] for a in arrays])
    code = load().bt_stage_audio(ptrs, dts, frames, chans, n, c_void_p(dst.data_ptr()), i64_array(so), threads)
    if code != 0:
        raise BTError(f"bt_stage_audio failed ({code}): bad signal array")
    return so


def wav_probe(paths):
    """bt_wav_probe on every path: (ctypes array of bt_wav_info, list of ok flags).  Files that are not plain WAV are
    left to load_audio's backend chain."""
    lib = load()
    infos = (bt_wav_info * len(paths))()
    ok = [lib.bt_wav_probe(str(p).encode(), ctypes.byref(infos[i])) == 0 and infos[i].frames > 0
          for i, p in enumerate(paths)]
    return infos, ok


def stage_wav_files(paths, infos, dst, sample_offsets, threads: int):
    """bt_stage_wav_files: file k (bt_wav_info infos[k] from wav_probe) read, mixed to mono and cast to fp32 into `dst`
    (host fp32 tensor) from sample_offsets[k] on, on `threads` host threads.  RuntimeError names the files that
    failed."""
    n = len(paths)
    cpaths = (c_char_p * n)(*[str(p).encode() for p in paths])
    status = (c_int32 * n)()
    code = load().bt_stage_wav_files(cpaths, (bt_wav_info * n)(*infos), n, c_void_p(dst.data_ptr()), i64_array(sample_offsets),
                                     threads, status)
    if code != 0:
        bad = [str(paths[i]) for i in range(n) if status[i] != 0]
        raise RuntimeError(f"Could not load audio from {bad}")


def probe_audio(paths):
    """The container of every path as the native readers see it: a list of ("wav", bt_wav_info) (bt_wav_probe, with
    samples), ("flac", bt_flac_info) (bt_flac_probe, with frame bytes), ("mp3", bt_mp3_info) (bt_mp3_probe, with
    output samples), ("vorbis", bt_vorbis_info) (bt_vorbis_probe, with output samples) or (None, None) for anything
    else, which load_audio's backend chain takes.  WAV is tried first, then FLAC, then MP3, then Ogg Vorbis."""
    lib = load()
    out = []
    for p in paths:
        w, f, m, v = bt_wav_info(), bt_flac_info(), bt_mp3_info(), bt_vorbis_info()
        if lib.bt_wav_probe(str(p).encode(), ctypes.byref(w)) == 0 and w.frames > 0:
            out.append(("wav", w))
        elif lib.bt_flac_probe(str(p).encode(), ctypes.byref(f)) == 0 and f.frames_bytes > 0:
            out.append(("flac", f))
        elif lib.bt_mp3_probe(str(p).encode(), ctypes.byref(m)) == 0 and m.n_samples > 0:
            out.append(("mp3", m))
        elif lib.bt_vorbis_probe(str(p).encode(), ctypes.byref(v)) == 0 and v.n_samples > 0:
            out.append(("vorbis", v))
        else:
            out.append((None, None))
    return out


FLAC_FRAME_BYTES = ctypes.sizeof(bt_flac_frame)


def _compressed_layout(entries, entry_bytes: int, byte_counts):
    """Frame tables first (entry k at byte entry_bytes * k; entries[i] per file), then one int32 status per file, then
    each file's bytes (byte_counts[i]): (frame-table entry offsets, status offset, byte offsets, total bytes)."""
    fo = offsets(entries)
    status_at = entry_bytes * fo[-1]
    bytes_at = status_at + 4 * (len(fo) - 1)
    bo = [bytes_at + v for v in offsets(byte_counts)]
    return fo, status_at, bo, bo[-1]


def flac_layout(infos):
    """Where bt_stage_flac_files puts the files `infos` in one byte buffer: (frame-table entry offsets, status offset,
    frame-byte offsets, total bytes).  The frame tables come first (entry k at byte FLAC_FRAME_BYTES * k), then one
    int32 status per file, then each file's frame bytes."""
    return _compressed_layout([info.max_frames for info in infos], FLAC_FRAME_BYTES,
                              [info.frames_bytes for info in infos])


def stage_flac_files(paths, infos, buf_ptr: int, threads: int):
    """bt_stage_flac_files into the byte buffer at host address buf_ptr, laid out as flac_layout(infos) says, with each
    file's status (BT_OK / BT_ERR_IO) stored at its slot of the buffer: (n_frames, n_samples, status) lists."""
    n = len(paths)
    fo, status_at, bo, _ = flac_layout(infos)
    cpaths = (c_char_p * n)(*[str(p).encode() for p in paths])
    nf, ns = (c_int64 * n)(), (c_int64 * n)()
    status = (c_int32 * n).from_address(buf_ptr + status_at)
    load().bt_stage_flac_files(cpaths, (bt_flac_info * n)(*infos), n, c_void_p(buf_ptr), i64_array(bo[:-1]),
                               c_void_p(buf_ptr), i64_array(fo[:-1]), nf, ns, threads, status)
    return list(nf), list(ns), list(status)


def flac_streams(infos, n_frames, n_samples, out_offsets):
    """The bt_flac_stream table of files staged by stage_flac_files (offsets relative to the same buffer), file i's
    output from out_offsets[i] on."""
    fo, _, bo, _ = flac_layout(infos)
    n = len(infos)
    return (bt_flac_stream * n)(*[
        bt_flac_stream(bo[i], infos[i].frames_bytes, fo[i], n_frames[i], n_samples[i], out_offsets[i],
                       infos[i].channels, infos[i].bits_per_sample) for i in range(n)])


MP3_FRAME_BYTES = ctypes.sizeof(bt_mp3_frame)


def mp3_layout(infos):
    """Where bt_stage_mp3_files puts the files `infos` in one byte buffer, as flac_layout does: frame tables
    (MP3_FRAME_BYTES per entry), one int32 status per file, then each file's compacted main data."""
    return _compressed_layout([info.max_frames for info in infos], MP3_FRAME_BYTES, [info.main_bytes for info in infos])


def stage_mp3_files(paths, infos, buf_ptr: int, threads: int):
    """bt_stage_mp3_files into the byte buffer at host address buf_ptr, laid out as mp3_layout(infos) says, each file's
    status stored at its slot of the buffer: (n_frames, main_bytes, status) lists."""
    n = len(paths)
    fo, status_at, bo, _ = mp3_layout(infos)
    cpaths = (c_char_p * n)(*[str(p).encode() for p in paths])
    nf, mb = (c_int64 * n)(), (c_int64 * n)()
    status = (c_int32 * n).from_address(buf_ptr + status_at)
    load().bt_stage_mp3_files(cpaths, (bt_mp3_info * n)(*infos), n, c_void_p(buf_ptr), i64_array(bo[:-1]),
                              c_void_p(buf_ptr), i64_array(fo[:-1]), mb, nf, threads, status)
    return list(nf), list(mb), list(status)


def mp3_streams(infos, n_frames, main_bytes, out_offsets):
    """The bt_mp3_stream table of files staged by stage_mp3_files (offsets relative to the same buffer), file i's
    output (infos[i].n_samples samples per channel) from out_offsets[i] on."""
    fo, _, bo, _ = mp3_layout(infos)
    n = len(infos)
    return (bt_mp3_stream * n)(*[
        bt_mp3_stream(bo[i], main_bytes[i], fo[i], n_frames[i], infos[i].skip, infos[i].n_samples, out_offsets[i],
                      infos[i].channels, infos[i].sample_rate) for i in range(n)])


VORBIS_PACKET_BYTES = ctypes.sizeof(bt_vorbis_packet)


def _vorbis_tables_at(info) -> int:
    """Where a staged Vorbis file's decode tables start after its packet bytes."""
    return (int(info.packet_bytes) + 3) // 4 * 4


def vorbis_layout(infos):
    """Where bt_stage_vorbis_files puts the files `infos` in one byte buffer, as flac_layout does: packet tables
    (VORBIS_PACKET_BYTES per entry), one int32 status per file, then each file's packet bytes followed by its decode
    tables."""
    return _compressed_layout([info.n_packets for info in infos], VORBIS_PACKET_BYTES,
                              [_vorbis_tables_at(info) + info.table_bytes for info in infos])


def stage_vorbis_files(paths, infos, buf_ptr: int, threads: int):
    """bt_stage_vorbis_files into the byte buffer at host address buf_ptr, laid out as vorbis_layout(infos) says, each
    file's status stored at its slot of the buffer: (n_packets, packet_bytes, block_samples, status) lists."""
    n = len(paths)
    fo, status_at, bo, _ = vorbis_layout(infos)
    cpaths = (c_char_p * n)(*[str(p).encode() for p in paths])
    npk, pb, bs = (c_int64 * n)(), (c_int64 * n)(), (c_int64 * n)()
    status = (c_int32 * n).from_address(buf_ptr + status_at)
    load().bt_stage_vorbis_files(cpaths, (bt_vorbis_info * n)(*infos), n, c_void_p(buf_ptr), i64_array(bo[:-1]),
                                 c_void_p(buf_ptr), i64_array(fo[:-1]), pb, npk, bs, threads, status)
    return list(npk), list(pb), list(bs), list(status)


def vorbis_streams(infos, n_packets, packet_bytes, block_samples, out_offsets):
    """The bt_vorbis_stream table of files staged by stage_vorbis_files (offsets relative to the same buffer), file i's
    output (infos[i].n_samples samples per channel) from out_offsets[i] on."""
    fo, _, bo, _ = vorbis_layout(infos)
    n = len(infos)
    return (bt_vorbis_stream * n)(*[
        bt_vorbis_stream(bo[i], packet_bytes[i], bo[i] + _vorbis_tables_at(infos[i]), infos[i].table_bytes, fo[i],
                         n_packets[i], block_samples[i], infos[i].skip, infos[i].n_samples, out_offsets[i],
                         infos[i].channels, infos[i].sample_rate) for i in range(n)])


def dbn_viterbi(log_densities, beats: int, intervals, log_tempo, pointers):
    """bt_dbn_viterbi (host C++) of one bar model on float64 log densities [T, 3]: (state path, log-probability)."""
    dens = np.ascontiguousarray(log_densities, dtype=np.float64)
    T = len(dens)
    path = np.empty(T, dtype=np.int64)
    logp = c_double()
    iv = np.ascontiguousarray(intervals, dtype=np.int32)
    lt = np.ascontiguousarray(log_tempo, dtype=np.float64)
    pt = np.ascontiguousarray(pointers, dtype=np.int32)
    code = load().bt_dbn_viterbi(dens.ctypes.data, T, int(beats), len(iv), iv.ctypes.data, lt.ctypes.data, pt.ctypes.data,
                                 path.ctypes.data, ctypes.byref(logp))
    if code != 0:
        raise RuntimeError(f"bt_dbn_viterbi failed ({code})")
    return path, float(logp.value)


def dbn_track(activations, frame_offsets, params: dict, n_threads: int = 0):
    """bt_dbn_track (host C++, one thread per piece) on [total_frames, 2] float64 activations for the tracker
    parameters `params` (dbn.DBNDownBeatTracker.track_params): (times, beat numbers, counts); piece i has counts[i]
    pairs from frame_offsets[i] on."""
    fo = np.ascontiguousarray(frame_offsets, dtype=np.int64)
    n = len(fo) - 1
    cat = np.ascontiguousarray(activations, dtype=np.float64).reshape(-1, 2)
    total = max(int(fo[-1]), 1)
    times = np.empty(total, dtype=np.float64)
    numbers = np.empty(total, dtype=np.int32)
    counts = np.zeros(max(n, 1), dtype=np.int64)
    bpb = np.asarray(params["beats_per_bar"], dtype=np.int32)
    p = params
    code = load().bt_dbn_track(cat.ctypes.data, fo.ctypes.data, n, bpb.ctypes.data, len(bpb), p["min_bpm"], p["max_bpm"],
                               p["num_tempi"], p["transition_lambda"], p["observation_lambda"], p["threshold"],
                               int(p["correct"]), p["fps"], int(n_threads), times.ctypes.data, numbers.ctypes.data,
                               counts.ctypes.data)
    if code != 0:
        raise RuntimeError(f"bt_dbn_track failed ({code})")
    return times, numbers, counts
