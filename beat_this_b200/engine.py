"""Thin Python owner of one ``bt_ctx`` (one per GPU / model).  PyTorch is used only for
device memory, streams and pinned host buffers; every FLOP runs in libbeatthis_sm100.so."""
from __future__ import annotations

import ctypes
import math
from ctypes import c_void_p

import numpy as np
import torch

from . import _lib
from ._lib import BT_DTYPE_H16, BT_DTYPE_F32, DEFAULT_CHUNKING, i32_array, i64_array

_SHARED = {}  # device -> the weight-less Engine of Engine.shared


def _cuda_device(device) -> torch.device:
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(
            f"beat_this_b200 runs on an sm_90a (H100) CUDA device only (got device={device!r}); "
            "there is no CPU fallback"
        )
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def chunking_struct(chunk_size: int, border_size: int, overlap_mode: str, max_chunk_size: int = _lib.BT_CHUNK
                    ) -> _lib.bt_chunking:
    """split_predict_aggregate's (chunk_size, border_size, overlap_mode) as the C library takes it
    (bt_plan_chunking_max, include/beatthis.h).  ``ValueError`` for what the library refuses: chunk_size outside
    [1, max_chunk_size] (the model's maximum chunk length: the rows of its RoPE tables, 1500 unless it was loaded with
    a larger max_chunk_size), a negative border, 2 * border_size >= chunk_size or an overlap_mode other than
    "keep_first" / "keep_last"."""
    if overlap_mode not in _lib.OVERLAP_MODES:
        raise ValueError("overlap_mode must be 'keep_first' or 'keep_last'")
    chunk_size, border_size = int(chunk_size), int(border_size)
    if not 1 <= chunk_size <= max_chunk_size:
        raise ValueError(f"chunk_size must be in [1, {max_chunk_size}] (the model's max_chunk_size), got {chunk_size}")
    if border_size < 0 or 2 * border_size >= chunk_size:
        raise ValueError(f"border_size must satisfy 0 <= 2 * border_size < chunk_size, got {border_size} for {chunk_size}")
    return _lib.bt_chunking(chunk_size, border_size, _lib.OVERLAP_MODES[overlap_mode])


class _PeakHandle:
    def __init__(self, slot, n):
        self.slot, self.n = slot, n

    def result(self):
        self.slot["event"].synchronize()
        cnt = self.slot["cnt_h"].numpy()
        times = self.slot["times_h"].numpy()
        out = [(times[0, i, : cnt[0, i]].copy(), times[1, i, : cnt[1, i]].copy()) for i in range(self.n)]
        self.slot["keep"] = None
        return out

    @property
    def d2h_bytes(self):
        return self.slot["times_h"].numel() * 8 + self.slot["cnt_h"].numel() * 4


class _DbnHandle:
    def __init__(self, slot, frame_offsets):
        self.slot, self.fo = slot, frame_offsets

    def result(self):
        self.slot["event"].synchronize()
        n = len(self.fo) - 1
        cnt = self.slot["counts_h"].numpy()
        times = self.slot["times_h"].numpy()
        numbers = self.slot["numbers_h"].numpy()
        out = []
        for i in range(n):  # as Postprocessor.batch_host splits the tracker's [n, 2] result
            a, k = self.fo[i], int(cnt[i])
            t = times[a : a + k].copy()
            out.append((t, t[numbers[a : a + k] == 1]))
        self.slot["keep"] = None
        return out

    @property
    def d2h_bytes(self):
        return (len(self.fo) - 1) * 8 + (self.fo[-1] if self.fo else 0) * 12


class Engine:
    def __init__(self, packed: dict | None, hparams: dict | None, device="cuda", half: bool = False, wave_chunks: int | None = None):
        self.lib = _lib.load()
        self.device = _cuda_device(device)
        self.half = bool(half)  # 16-bit tensor-core path (fp16 operands; see bt_act_dtype) instead of fp32 CUDA cores
        self.act_dtype = self.lib.bt_act_dtype().decode() if half else "f32"
        hp = hparams or {}
        self.hparams = dict(hp)
        chp = _lib.hparams_struct(hp)
        ctx = c_void_p()
        code = self.lib.bt_create(ctypes.byref(ctx), self.device.index, ctypes.byref(chp), BT_DTYPE_H16 if half else BT_DTYPE_F32)
        _lib.check(self.lib, None, code)
        self.ctx = ctx
        self._model_ready = False
        self._resample_banks = {}  # (sr_in, sr_out) -> (coef device tensor, L, M, K)
        if packed is not None:
            self.set_params(packed)
        if wave_chunks:
            self.set_wave_chunks(wave_chunks)

    # ---- construction -----------------------------------------------------------------------
    @classmethod
    def mel_only(cls, device="cuda"):
        from .preprocessing import mel_constants

        eng = cls(None, None, device, False)
        for k, v in mel_constants().items():
            eng._set_param(k, v)
        return eng

    @classmethod
    def shared(cls, device="cuda"):
        """The weight-less engine of `device` that the beat metrics, the losses and the training batches share."""
        dev = _cuda_device(device)
        if dev not in _SHARED:
            _SHARED[dev] = cls.mel_only(dev)
        return _SHARED[dev]

    def _set_param(self, name: str, arr: np.ndarray):
        arr = np.ascontiguousarray(arr, dtype=np.float32).reshape(-1)
        self._call("bt_set_param", name.encode(), arr.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), arr.size, stream=False)

    def set_params(self, packed: dict):
        for k, v in packed.items():
            self._set_param(k, v)
        self._call("bt_finalize", stream=False)
        self._model_ready = True

    @property
    def max_chunk(self) -> int:
        """The longest chunk this context runs (bt_max_chunk: the rows of its RoPE tables)."""
        return int(self.lib.bt_max_chunk(self.ctx))

    def set_wave_chunks(self, n: int):
        self._call("bt_set_wave_chunks", int(n), stream=False)

    def close(self):
        if getattr(self, "ctx", None) is not None and self.ctx.value:
            self.lib.bt_destroy(self.ctx)
            self.ctx = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self) -> int:
        return int(self.lib.bt_launch_count(self.ctx))

    def _stream(self):
        return c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _call(self, name: str, *args, stream: bool = True):
        """The context entry point `name` on (ctx, *args), followed by the current stream of this device for the entry
        points that enqueue work; a non-zero code raises BTError."""
        _lib.check(self.lib, self.ctx, getattr(self.lib, name)(self.ctx, *args, *((self._stream(),) if stream else ())))

    # The C library cannot see buffer sizes or types, so each tensor is checked here to be a contiguous device tensor
    # of the dtype the entry point reads (one of them, for a tuple) holding at least the n elements it touches.
    @staticmethod
    def _dev_ptr(t, n: int = 0, dtype=torch.float32):
        if t is None:
            return None
        assert t.is_cuda and t.is_contiguous() and t.dtype in (dtype if isinstance(dtype, tuple) else (dtype,)), \
            f"expected a contiguous CUDA tensor of {dtype}, got {t.dtype} on {t.device}"
        assert t.numel() >= n, f"tensor of {t.numel()} elements, the hook reads or writes {n}"
        return c_void_p(t.data_ptr())

    # ---- hot path ---------------------------------------------------------------------------
    @staticmethod
    def frame_offsets(sample_offsets, hop: int = 441):
        return _lib.offsets(1 + (int(b) - int(a)) // hop for a, b in zip(sample_offsets[:-1], sample_offsets[1:]))

    def resample_cat(self, audio: torch.Tensor, sample_offsets, sr: int, sr_out: int = 22050):
        """Concatenated fp32 device audio at `sr` Hz -> (audio at `sr_out` Hz, new sample offsets): the device
        stand-in for soxr.resample (reference inference.py:274-275), see preprocessing.resample_filter_bank."""
        from . import preprocessing as P

        key = (int(sr), int(sr_out))
        if key not in self._resample_banks:
            coef, L, M, K = P.resample_filter_bank(*key)
            self._resample_banks[key] = (torch.from_numpy(coef).to(self.device).contiguous(), L, M, K)
        coef, L, M, K = self._resample_banks[key]
        so = [int(v) for v in sample_offsets]
        oo = _lib.offsets(P.resampled_length(so[i + 1] - so[i], L, M) for i in range(len(so) - 1))
        out = torch.empty(max(oo[-1], 1), dtype=torch.float32, device=self.device)[: oo[-1]]
        p = self._dev_ptr
        self._call("bt_resample", p(audio), i64_array(so), len(so) - 1, p(coef), L, M, K, p(out), i64_array(oo))
        return out, oo

    def flac_decode(self, buf: torch.Tensor, streams, mode: int, out: torch.Tensor, status_at: int):
        """bt_flac_decode of the FLAC files staged in the uint8 device tensor `buf` as _lib.flac_layout lays them out
        (streams: _lib.flac_streams); their statuses, read and written, sit at byte status_at of buf.  out: fp32
        (BT_FLAC_MONO_F32) or float64 (BT_FLAC_CHANNELS_F64) device tensor."""
        dtype = torch.float32 if mode == _lib.BT_FLAC_MONO_F32 else torch.float64
        base = self._dev_ptr(buf, dtype=torch.uint8)
        need = max((s.out_offset + s.n_samples * (1 if mode == _lib.BT_FLAC_MONO_F32 else s.channels) for s in streams),
                   default=0)
        self._call("bt_flac_decode", base, base, streams, len(streams), int(mode), self._dev_ptr(out, need, dtype),
                   c_void_p(buf.data_ptr() + int(status_at)))

    def mp3_decode(self, buf: torch.Tensor, streams, mode: int, out: torch.Tensor, status_at: int):
        """bt_mp3_decode of the MP3 files staged in the uint8 device tensor `buf` as _lib.mp3_layout lays them out
        (streams: _lib.mp3_streams); their statuses, read and written, sit at byte status_at of buf.  out: fp32
        (BT_MP3_MONO_F32) or float64 (BT_MP3_CHANNELS_F64) device tensor."""
        dtype = torch.float32 if mode == _lib.BT_MP3_MONO_F32 else torch.float64
        base = self._dev_ptr(buf, dtype=torch.uint8)
        need = max((s.out_offset + s.n_samples * (1 if mode == _lib.BT_MP3_MONO_F32 else s.channels) for s in streams),
                   default=0)
        self._call("bt_mp3_decode", base, base, streams, len(streams), int(mode), self._dev_ptr(out, need, dtype),
                   c_void_p(buf.data_ptr() + int(status_at)))

    def vorbis_decode(self, buf: torch.Tensor, streams, mode: int, out: torch.Tensor, status_at: int):
        """bt_vorbis_decode of the Ogg Vorbis files staged in the uint8 device tensor `buf` as _lib.vorbis_layout lays
        them out (streams: _lib.vorbis_streams); their statuses, read and written, sit at byte status_at of buf.  out:
        fp32 (BT_VORBIS_MONO_F32) or float64 (BT_VORBIS_CHANNELS_F64) device tensor."""
        dtype = torch.float32 if mode == _lib.BT_VORBIS_MONO_F32 else torch.float64
        base = self._dev_ptr(buf, dtype=torch.uint8)
        need = max((s.out_offset + s.n_samples * (1 if mode == _lib.BT_VORBIS_MONO_F32 else s.channels)
                    for s in streams), default=0)
        self._call("bt_vorbis_decode", base, base, streams, len(streams), int(mode), self._dev_ptr(out, need, dtype),
                   c_void_p(buf.data_ptr() + int(status_at)))

    def logmel_cat(self, audio: torch.Tensor, sample_offsets):
        """audio: flat fp32 device tensor; returns (spect [total_frames,128], frame_offsets)."""
        fo = self.frame_offsets(sample_offsets)
        spect = torch.empty((fo[-1], 128), dtype=torch.float32, device=self.device)
        self._call("bt_logmel", self._dev_ptr(audio), i64_array(sample_offsets), len(sample_offsets) - 1,
                   self._dev_ptr(spect), i64_array(fo))
        return spect, fo

    def _per_clip(self, signals, cat):
        """cat(flat fp32 device audio, sample offsets) -> (spect, frame offsets) for the clips `signals`: per clip spect."""
        sigs = [torch.as_tensor(s, dtype=torch.float32, device=self.device).contiguous() for s in signals]
        spect, fo = cat(torch.cat(sigs) if len(sigs) > 1 else sigs[0], _lib.offsets(s.numel() for s in sigs))
        return [spect[fo[i] : fo[i + 1]] for i in range(len(sigs))]

    def logmel(self, signals):
        return self._per_clip(signals, self.logmel_cat)

    def logmel_config_cat(self, audio: torch.Tensor, sample_offsets, tables, device_tables: dict):
        """bt_logmel_config on flat fp32 device audio for the analysis of ``tables`` (preprocessing.MelTables, whose
        ``to(device)`` gave ``device_tables``): (spect [total_frames, n_mels], frame_offsets)."""
        fo = self.frame_offsets(sample_offsets, tables.hop_length)
        spect = torch.empty((fo[-1], tables.n_mels), dtype=torch.float32, device=self.device)
        t, p = device_tables, self._dev_ptr
        self._call("bt_logmel_config", ctypes.byref(tables.config), p(t["window"]), p(t["twiddle"]),
                   p(t["fb_start"], dtype=torch.int32), p(t["fb_ptr"], dtype=torch.int32), p(t["fb_w"]), p(audio),
                   i64_array(sample_offsets), len(sample_offsets) - 1, p(spect), i64_array(fo))
        return spect, fo

    def logmel_config(self, signals, tables, device_tables: dict):
        return self._per_clip(signals, lambda audio, so: self.logmel_config_cat(audio, so, tables, device_tables))

    # ---- tempo / pitch augmentation (augment.py; contracts in include/beatthis.h) -------------
    def stft_cat(self, audio: torch.Tensor, sample_offsets, tables):
        """bt_stft on flat fp32 device audio for the analysis of ``tables`` (augment.StftTables on this device):
        (complex64 spectrogram [total_frames, n_fft / 2 + 1], frame_offsets)."""
        fo = self.frame_offsets(sample_offsets, tables.hop_length)
        spec = torch.empty((fo[-1], tables.bins), dtype=torch.complex64, device=self.device)
        p = self._dev_ptr
        self._call("bt_stft", ctypes.byref(tables.config), p(tables.window), p(tables.twiddle), p(audio),
                   i64_array(sample_offsets), len(sample_offsets) - 1, p(spec, dtype=torch.complex64), i64_array(fo))
        return spec, fo

    def phase_vocoder_cat(self, spec: torch.Tensor, frame_offsets, variant_clip, variant_rate):
        """bt_phase_vocoder: variant v is clip variant_clip[v] of ``spec`` (complex64 [total_frames, bins]) at rate
        variant_rate[v].  Returns (complex64 [total_out_frames, bins], out_frame_offsets)."""
        assert spec.ndim == 2
        n_clips, nv = len(frame_offsets) - 1, len(variant_clip)

        def frames(clip, rate):
            T = int(frame_offsets[clip + 1]) - int(frame_offsets[clip]) if 0 <= clip < n_clips else 0
            return math.ceil(T / rate) if rate > 0 and math.isfinite(rate) else 0

        oo = _lib.offsets(frames(clip, rate) for clip, rate in zip(variant_clip, variant_rate))
        out = torch.empty((oo[-1], spec.shape[1]), dtype=torch.complex64, device=self.device)
        p = self._dev_ptr
        self._call("bt_phase_vocoder", 2 * (spec.shape[1] - 1), p(spec, dtype=torch.complex64), i64_array(frame_offsets),
                   n_clips, (ctypes.c_int32 * max(nv, 1))(*[int(v) for v in variant_clip]),
                   (ctypes.c_double * max(nv, 1))(*[float(r) for r in variant_rate]), nv, p(out, dtype=torch.complex64),
                   i64_array(oo))
        return out, oo

    def istft_cat(self, spec: torch.Tensor, frame_offsets, lengths, tables):
        """bt_istft: sequence s (frames frame_offsets[s]..) -> lengths[s] samples.  Returns (flat fp32 audio, sample
        offsets)."""
        so = _lib.offsets(lengths)
        out = torch.empty(max(so[-1], 1), dtype=torch.float32, device=self.device)[: so[-1]]
        p = self._dev_ptr
        self._call("bt_istft", ctypes.byref(tables.config), p(tables.window), p(tables.twiddle),
                   p(spec, dtype=torch.complex64), i64_array(frame_offsets), len(frame_offsets) - 1, p(out), i64_array(so))
        return out, so

    def spect2frames_cat(self, spect: torch.Tensor, frame_offsets, chunking: tuple | None = DEFAULT_CHUNKING):
        """Concatenated [total, 128] spectrograms -> (beat, downbeat) logits.  chunking: (chunk_size, border_size,
        overlap_mode) of split_predict_aggregate, checked by chunking_struct against max_chunk; None, which earlier
        versions took for the default, is DEFAULT_CHUNKING."""
        assert self._model_ready, "model parameters not loaded"
        ck = chunking_struct(*(chunking or DEFAULT_CHUNKING), self.max_chunk)
        total = int(frame_offsets[-1])
        beat = torch.empty(total, dtype=torch.float32, device=self.device)
        down = torch.empty(total, dtype=torch.float32, device=self.device)
        p = self._dev_ptr
        self._call("bt_spect2frames_chunked", p(spect), i64_array(frame_offsets), len(frame_offsets) - 1, p(beat), p(down),
                   ctypes.byref(ck))
        return beat, down

    def forward_chunks(self, chunks: torch.Tensor):
        """BeatThis.forward on [B, T<=max_chunk, 128] chunks (no chunk planning, no borders cut): flat (beat, downbeat)."""
        assert self._model_ready, "model parameters not loaded"
        assert chunks.ndim == 3
        B, T, _ = chunks.shape
        beat = torch.empty(B * T, dtype=torch.float32, device=self.device)
        down = torch.empty(B * T, dtype=torch.float32, device=self.device)
        self._call("bt_forward_chunks", self._dev_ptr(chunks), B, T, self._dev_ptr(beat), self._dev_ptr(down))
        return beat, down

    def audio2frames_cat(self, audio: torch.Tensor, sample_offsets, chunking: tuple | None = DEFAULT_CHUNKING):
        """Concatenated mono 22.05 kHz audio -> (beat, downbeat, frame offsets); chunking as in spect2frames_cat."""
        assert self._model_ready, "model parameters not loaded"
        ck = chunking_struct(*(chunking or DEFAULT_CHUNKING), self.max_chunk)
        fo = self.frame_offsets(sample_offsets)
        beat = torch.empty(fo[-1], dtype=torch.float32, device=self.device)
        down = torch.empty(fo[-1], dtype=torch.float32, device=self.device)
        p = self._dev_ptr
        self._call("bt_audio2frames_chunked", p(audio), i64_array(sample_offsets), len(sample_offsets) - 1, p(beat),
                   p(down), i64_array(fo), ctypes.byref(ck))
        return beat, down, fo

    def peakpick_cat(self, beat: torch.Tensor, down: torch.Tensor, frame_offsets, fps: float = 50):
        """Minimal postprocessor on device for logits at `fps` frames per second (bt_peakpick_fps); returns a list of
        (beat_times, downbeat_times) float64 numpy arrays, one pair per clip."""
        n = len(frame_offsets) - 1
        if n == 0:
            return []
        max_peaks = max(1, max(int(frame_offsets[i + 1]) - int(frame_offsets[i]) for i in range(n)))
        bt_t = torch.empty((n, max_peaks), dtype=torch.float64, device=self.device)
        dn_t = torch.empty((n, max_peaks), dtype=torch.float64, device=self.device)
        cnt = torch.zeros((2, n), dtype=torch.int32, device=self.device)
        self._peakpick(beat, down, frame_offsets, fps, bt_t, cnt[0], dn_t, cnt[1], max_peaks)
        cnt_h = cnt.cpu().numpy()
        width = int(cnt_h.max()) if cnt_h.size else 0
        if width > max_peaks:
            raise _lib.BTError("peak buffer overflow (internal error)")
        bt_h = bt_t[:, :width].cpu().numpy()
        dn_h = dn_t[:, :width].cpu().numpy()
        return [(bt_h[i, : cnt_h[0, i]].copy(), dn_h[i, : cnt_h[1, i]].copy()) for i in range(n)]

    def peakpick_async(self, beat: torch.Tensor, down: torch.Tensor, frame_offsets, slot: dict | None = None,
                       fps: float = 50):
        """Like peakpick_cat but without a host synchronisation: the timestamp arrays are copied to
        pinned host memory asynchronously on the current stream; call ``.result()`` on the returned
        handle (it waits on a CUDA event) to get the per-clip numpy arrays."""
        n = len(frame_offsets) - 1
        max_peaks = max(1, max(int(frame_offsets[i + 1]) - int(frame_offsets[i]) for i in range(n)))
        slot = slot if slot is not None else {}
        key = (n, max_peaks)
        if slot.get("key") != key:
            slot["key"] = key
            slot["times"] = torch.empty((2, n, max_peaks), dtype=torch.float64, device=self.device)
            slot["cnt"] = torch.zeros((2, n), dtype=torch.int32, device=self.device)
            slot["times_h"] = torch.empty((2, n, max_peaks), dtype=torch.float64).pin_memory()
            slot["cnt_h"] = torch.empty((2, n), dtype=torch.int32).pin_memory()
            slot["event"] = torch.cuda.Event()
        t, cnt = slot["times"], slot["cnt"]
        self._peakpick(beat, down, frame_offsets, fps, t[0], cnt[0], t[1], cnt[1], max_peaks)
        slot["times_h"].copy_(t, non_blocking=True)
        slot["cnt_h"].copy_(cnt, non_blocking=True)
        slot["event"].record(torch.cuda.current_stream(self.device))
        slot["keep"] = (beat, down)  # keep the logits alive until the kernels have run
        return _PeakHandle(slot, n)

    def _peakpick(self, beat, down, frame_offsets, fps, beat_times, beat_counts, down_times, down_counts, max_peaks):
        p = self._dev_ptr
        self._call("bt_peakpick_fps", p(beat), p(down), i64_array(frame_offsets), len(frame_offsets) - 1, float(fps),
                   p(beat_times, dtype=torch.float64), p(beat_counts, dtype=torch.int32), p(down_times, dtype=torch.float64),
                   p(down_counts, dtype=torch.int32), max_peaks)

    def _dbn_enqueue(self, beat, down, act, frame_offsets, params: dict, times, numbers, counts):
        bpb = np.ascontiguousarray(params["beats_per_bar"], dtype=np.int32)
        p = self._dev_ptr
        self._call("bt_dbn_track_device", p(beat), p(down), p(act, dtype=torch.float64), i64_array(frame_offsets),
                   len(frame_offsets) - 1, i32_array(bpb), len(bpb), float(params["min_bpm"]), float(params["max_bpm"]),
                   int(params["num_tempi"]), float(params["transition_lambda"]), float(params["observation_lambda"]),
                   float(params["threshold"]), int(bool(params["correct"])), float(params["fps"]),
                   p(times, dtype=torch.float64), p(numbers, dtype=torch.int32), p(counts, dtype=torch.int64))

    def dbn_async(self, beat: torch.Tensor | None, down: torch.Tensor | None, frame_offsets, slot: dict | None = None,
                  params: dict | None = None, activations: torch.Tensor | None = None):
        """Postprocessor("dbn") on the device (bt_dbn_track_device) for concatenated fp32 logits -- or, with
        `activations`, a [total, 2] float64 device tensor of (beat-but-not-downbeat, downbeat) probabilities -- without
        a host synchronisation: (time, beat number) pairs and counts are copied to pinned host memory on the current
        stream.  params: the tracker parameters (dbn.DBNDownBeatTracker.track_params).  ``.result()`` on the handle
        gives a list of (beat_times, downbeat_times)."""
        n = len(frame_offsets) - 1
        total = int(frame_offsets[-1]) if n > 0 else 0
        slot = slot if slot is not None else {}
        cap = max(total, 1)
        if slot.get("cap", -1) < cap or slot.get("n", -1) < n:
            cap = max(cap, slot.get("cap", 0))
            nn = max(n, slot.get("n", 0), 1)
            slot["cap"], slot["n"] = cap, nn
            slot["times"] = torch.empty(cap, dtype=torch.float64, device=self.device)
            slot["numbers"] = torch.empty(cap, dtype=torch.int32, device=self.device)
            slot["counts"] = torch.zeros(nn, dtype=torch.int64, device=self.device)
            slot["times_h"] = torch.empty(cap, dtype=torch.float64).pin_memory()
            slot["numbers_h"] = torch.empty(cap, dtype=torch.int32).pin_memory()
            slot["counts_h"] = torch.empty(nn, dtype=torch.int64).pin_memory()
            slot["event"] = torch.cuda.Event()
        if activations is None:
            assert beat is not None and down is not None, "logits or activations"
        self._dbn_enqueue(beat, down, activations, frame_offsets, params, slot["times"], slot["numbers"], slot["counts"])
        if n > 0:
            slot["times_h"][:total].copy_(slot["times"][:total], non_blocking=True)
            slot["numbers_h"][:total].copy_(slot["numbers"][:total], non_blocking=True)
            slot["counts_h"][:n].copy_(slot["counts"][:n], non_blocking=True)
        slot["event"].record(torch.cuda.current_stream(self.device))
        slot["keep"] = (beat, down, activations)  # keep the inputs alive until the kernels have run
        return _DbnHandle(slot, [int(v) for v in frame_offsets])

    def dbn_cat(self, beat, down, frame_offsets, params: dict, activations=None):
        """Synchronous dbn_async: list of (beat_times, downbeat_times) float64 numpy arrays, one pair per clip."""
        return self.dbn_async(beat, down, frame_offsets, None, params, activations).result()

    def debug_dbn_viterbi(self, log_dens: torch.Tensor, beats: int, intervals, log_tempo, pointers):
        """bt_debug_dbn_viterbi: the device Viterbi of one bar model on float64 log densities [T, 3] (device tensor);
        model tables as bt_dbn_viterbi takes them (host arrays).  Returns (path int64 numpy array, logp float)."""
        T = log_dens.shape[0]
        lt = np.ascontiguousarray(log_tempo, dtype=np.float64)
        path = torch.empty(max(T, 1), dtype=torch.int64, device=self.device)
        logp = torch.empty(1, dtype=torch.float64, device=self.device)
        p = self._dev_ptr
        self._call("bt_debug_dbn_viterbi", p(log_dens, dtype=torch.float64), T, int(beats), len(intervals),
                   i32_array(intervals), c_void_p(lt.ctypes.data), i32_array(pointers), p(path, dtype=torch.int64),
                   p(logp, dtype=torch.float64))
        return path[:T].cpu().numpy(), float(logp.item())

    # ---- scoring and training (evaluate.py, loss.py, dataset.py; contracts in include/beatthis.h) ----------------
    def beat_metrics(self, times: torch.Tensor, offsets, params, out: torch.Tensor):
        """bt_beat_metrics of n = out.shape[0] sets on one float64 device buffer of times: set i's estimates are
        times[offsets[i]:offsets[i + 1]], its references times[offsets[n + i]:offsets[n + i + 1]]; out [n, 12] float64."""
        n = out.shape[0]
        base = self._dev_ptr(times, dtype=torch.float64)  # both offset arrays index the one buffer
        self._call("bt_beat_metrics", base, i64_array(offsets[: n + 1]), base, i64_array(offsets[n:]), n,
                   ctypes.byref(params), self._dev_ptr(out, dtype=torch.float64))

    def beat_loss(self, preds, targets, mask, offsets, params, row_loss, mean):
        """bt_beat_loss of the rows [offsets[i], offsets[i + 1]) of fp32 preds, targets and mask (None: no mask):
        float64 row_loss per row and the fp32 mean over all rows."""
        p = self._dev_ptr
        self._call("bt_beat_loss", p(preds), p(targets), p(mask), i64_array(offsets), len(offsets) - 1,
                   ctypes.byref(params), p(row_loss, dtype=torch.float64), p(mean))

    def beat_loss_backward(self, preds, targets, mask, offsets, params, grad_mean, grad):
        """bt_beat_loss_backward: grad (fp32, like preds) of the mean of beat_loss scaled by the fp32 grad_mean."""
        p = self._dev_ptr
        self._call("bt_beat_loss_backward", p(preds), p(targets), p(mask), i64_array(offsets), len(offsets) - 1,
                   ctypes.byref(params), p(grad_mean), p(grad))

    def train_batch(self, rows, row_offsets, length, row_map, beat_frames, beat_offsets, downbeat_frames,
                    downbeat_offsets, spect, truth_beat, truth_downbeat, padding_mask):
        """One ``bt_train_batch`` launch on the current stream: rows, spect and the three [B, L] outputs are device
        tensors (rows and spect of 16-bit elements, the others of bytes); the tables are host arrays, row_map None for
        identity maps."""
        p, h16, byte = self._dev_ptr, (torch.int16, torch.float16), (torch.bool, torch.uint8)
        self._call("bt_train_batch", p(rows, dtype=h16), i64_array(row_offsets), len(row_offsets) - 1, int(length),
                   None if row_map is None else i32_array(row_map), i32_array(beat_frames), i64_array(beat_offsets),
                   i32_array(downbeat_frames), i64_array(downbeat_offsets), p(spect, dtype=h16),
                   p(truth_beat, dtype=byte), p(truth_downbeat, dtype=byte), p(padding_mask, dtype=byte))

    # ---- model gradients (bt_train_*) ----------------------------------------------------------------
    @staticmethod
    def _train_mode(mode):
        """mode: None (eval mode) or (seed, dropout_frontend, dropout_transformer) -> a bt_train_mode or None."""
        if mode is None:
            return None
        seed, p_front, p_trans = mode
        return _lib.bt_train_mode(int(seed) & (2 ** 64 - 1), float(p_front), float(p_trans))

    def train_activation_bytes(self, B: int, L: int, mode=None) -> int:
        """Bytes of the activation store: mode None (eval mode) or (seed, dropout_frontend, dropout_transformer)."""
        n = int(self.lib.bt_train_activation_bytes_ex(self.ctx, int(B), int(L), self._train_mode(mode)))
        if n < 0:
            raise ValueError(f"bt_train_activation_bytes_ex refused B={B}, L={L}")
        return n

    def _table_ptrs(self, tensors, what: str):
        """Host array of device pointers (None: NULL) for a parameter or gradient table in bt_train_param_info order.
        Every entry the kernels touch must be a contiguous fp32 tensor of its table shape on this engine's device: the
        library sees only addresses, so a host, double or strided tensor would be read as other bytes."""
        if getattr(self, "_param_table", None) is None:
            self._param_table = _lib.train_param_table(self.hparams)
        if len(tensors) != len(self._param_table):
            raise ValueError(f"{what}: {len(tensors)} entries, the model has {len(self._param_table)}")
        for t, (name, shape, _) in zip(tensors, self._param_table):
            if t is None or not shape:  # ndim-0 entries (num_batches_tracked) are never read
                continue
            if t.device != self.device or t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != shape:
                raise RuntimeError(f"{what} {name}: need a contiguous float32 tensor of shape {shape} on {self.device}, "
                                   f"got {t.dtype} {tuple(t.shape)} on {t.device}; there is no CPU fallback")
        return (c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])

    def train_forward(self, params, spect, act, beat, down, mode=None, running=None):
        """bt_train_forward_ex: params in bt_train_param_info order (device tensors), spect [B, L, 128] fp32, act a byte
        tensor of train_activation_bytes(B, L, mode), beat / down [B, L] fp32 outputs.  mode None: eval mode; else
        (seed, dropout_frontend, dropout_transformer), and running (parallel to params; None: params itself) holds the
        running statistics the pass updates in place."""
        B, L, _ = spect.shape
        p = self._dev_ptr
        run = None
        if mode is not None:
            run = self._table_ptrs(params if running is None else running, "running statistic")
        self._call("bt_train_forward_ex", self._table_ptrs(params, "parameter"), len(params), run, p(spect, B * L * 128),
                   B, L, self._train_mode(mode), p(act, dtype=torch.uint8), act.numel(), p(beat, B * L), p(down, B * L))

    def train_backward(self, params, act, B: int, L: int, dbeat, ddown, grads, dspect=None, mode=None):
        """bt_train_backward_ex after train_forward with the same params, act and mode: grads (None: not wanted)
        parallel to params; dspect [B, L, 128] or None."""
        p = self._dev_ptr
        self._call("bt_train_backward_ex", self._table_ptrs(params, "parameter"), len(params), p(act, dtype=torch.uint8),
                   act.numel(), int(B), int(L), self._train_mode(mode), p(dbeat, B * L), p(ddown, B * L),
                   self._table_ptrs(grads, "gradient"), p(dspect, B * L * 128))

    def adamw_step(self, entries):
        """One ``bt_adamw_step`` call on the current stream: entries is a sequence of _lib.bt_adamw_entry whose device
        pointers the caller has checked and keeps alive until the update has run."""
        n = len(entries)
        self._call("bt_adamw_step", (_lib.bt_adamw_entry * max(n, 1))(*entries), n)

    # ---- data-parallel training (bt_grad_pack, bt_grad_ordered_sum, bt_train_running_replay) -------------------------
    def _grad_table(self, grads, rows):
        """The bt_grad_entry table of `grads` (contiguous fp32 tensors on this device), after checking that every packed
        row (fp32 device tensors) holds their total numel."""
        total = 0
        for g in grads:
            if g.device != self.device or g.dtype != torch.float32 or not g.is_contiguous():
                raise RuntimeError(f"gradient: need a contiguous float32 tensor on {self.device}, got {g.dtype} "
                                   f"{tuple(g.shape)} on {g.device}; there is no CPU fallback")
            total += g.numel()
        for r in rows:
            if r.device != self.device or r.dtype != torch.float32 or not r.is_contiguous() or r.numel() < total:
                raise RuntimeError(f"packed row: need a contiguous float32 tensor of at least {total} elements on "
                                   f"{self.device}, got {r.dtype} {tuple(r.shape)} on {r.device}")
        return (_lib.bt_grad_entry * max(len(grads), 1))(*[_lib.bt_grad_entry(g.data_ptr(), g.numel()) for g in grads])

    def grad_pack(self, grads, row):
        """One ``bt_grad_pack`` launch on the current stream: the tensors of `grads` copied into `row`, densely in
        order."""
        self._call("bt_grad_pack", self._grad_table(grads, [row]), len(grads), row.data_ptr())

    def grad_ordered_sum(self, grads, rows):
        """One ``bt_grad_ordered_sum`` launch on the current stream: each tensor of `grads` becomes the sum, in the order
        of `rows`, of its elements in the packed rows (((r0 + r1) + r2) + ..., one fp32 add at a time)."""
        ptrs = (c_void_p * max(len(rows), 1))(*[r.data_ptr() for r in rows])
        self._call("bt_grad_ordered_sum", self._grad_table(grads, rows), len(grads), ptrs, len(rows))

    def train_batch_stat_floats(self, B: int, L: int) -> int:
        """Floats of the batch statistics a training-mode activation store keeps after the eval-mode layout."""
        return (self.train_activation_bytes(B, L, (0, 0.0, 0.0)) - self.train_activation_bytes(B, L)) // 4

    def train_running_replay(self, running, stats, B: int, L: int):
        """``bt_train_running_replay`` on the current stream: the batch statistics of the micro-batches in `stats` (fp32
        device tensors of train_batch_stat_floats(B, L) elements each, in micro-batch order) applied to the running
        statistics of `running` (a table parallel to the parameters, as train_forward takes it)."""
        need = self.train_batch_stat_floats(B, L)
        for s in stats:
            if s.device != self.device or s.dtype != torch.float32 or not s.is_contiguous() or s.numel() < need:
                raise RuntimeError(f"batch statistics: need a contiguous float32 tensor of at least {need} elements on "
                                   f"{self.device}, got {s.dtype} {tuple(s.shape)} on {s.device}")
        ptrs = (c_void_p * max(len(stats), 1))(*[s.data_ptr() for s in stats])
        self._call("bt_train_running_replay", self._table_ptrs(running, "running statistic"), len(running), ptrs,
                   len(stats), int(B), int(L))

    # ---- per-kernel-class timing (bench.py roofline) -------------------------------------------
    def profile_enable(self, on: bool = True):
        self._call("bt_profile_enable", int(on), stream=False)

    def profile_reset(self):
        self._call("bt_profile_reset", stream=False)

    def profile_results(self) -> dict:
        """{kernel class: (total device ms, launches)} accumulated since the last reset."""
        self._call("bt_profile_collect", stream=False)
        out = {}
        for i in range(int(self.lib.bt_profile_count(self.ctx))):
            name = ctypes.create_string_buffer(64)
            ms, n = ctypes.c_double(), ctypes.c_int64()
            self.lib.bt_profile_get(self.ctx, i, name, 64, ctypes.byref(ms), ctypes.byref(n))
            out[name.value.decode()] = (ms.value, n.value)
        return out

    # ---- test hooks --------------------------------------------------------------------------
    def tap(self, name: str, spect: torch.Tensor, frame_offsets, capacity: int):
        """Test hook: activation `name` of a spect2frames_cat call."""
        return self._tap(name, capacity, lambda: self.spect2frames_cat(spect, frame_offsets))

    def tap_chunks(self, name: str, chunks: torch.Tensor, capacity: int):
        """Test hook: activation `name` of a forward_chunks call (single wave)."""
        return self._tap(name, capacity, lambda: self.forward_chunks(chunks))

    def _tap(self, name: str, capacity: int, forward):
        buf = torch.zeros(capacity, dtype=torch.float32, device=self.device)
        self._call("bt_debug_request_tap", name.encode(), self._dev_ptr(buf), capacity, stream=False)
        try:
            out = forward()
            torch.cuda.synchronize(self.device)
            n = int(self.lib.bt_debug_tap_count(self.ctx))
        finally:
            self.lib.bt_debug_request_tap(self.ctx, b"", None, 0)
        return buf[:n], out

    def debug_gemm(self, a: torch.Tensor, w: torch.Tensor):
        """D[M, N] = A[M, K] W[N, K]^T (fp32 device tensors) through the ctx's GEMM, no epilogue."""
        M, K = a.shape
        N = w.shape[0]
        d = torch.empty((M, N), dtype=torch.float32, device=self.device)
        shape = dict(planes_out=1, planes_in=1, L=M, N=N, Kslab=K, nslab=1, plane_mul=1, lda=K, plane_add=[0], t_shift=[0])
        self.debug_gemm_full(shape, a.contiguous(), w.contiguous(), out_f32=d)
        return d

    def debug_gemm_full(self, shape: dict, a, w, bias=None, resid=None, out_f32=None, out_act=None, rope_cos=None,
                        rope_sin=None, resid_epilogue=False, kind=0, gelu=False, C=0, heads=0, posmode=0, F=1, qscale=1.0):
        """One GEMM through bt_debug_gemm.  shape: the GemmShape fields (planes_out, planes_in, L, N, Kslab, nslab,
        plane_mul, lda, plane_add, t_shift); tensors are fp32 on this device and are passed through as they are (the
        outputs are written in place, resid may be out_f32).  Returns the (BN, BK) tile of the 16-bit plan."""
        ptr = self._dev_ptr
        d = _lib.bt_debug_gemm_desc()
        for f in ("planes_out", "planes_in", "L", "N", "Kslab", "nslab", "plane_mul", "lda"):
            setattr(d, f, int(shape[f]))
        for s in range(6):
            d.plane_add[s] = int(shape["plane_add"][s]) if s < len(shape["plane_add"]) else 0
            d.t_shift[s] = int(shape["t_shift"][s]) if s < len(shape["t_shift"]) else 0
        d.resid_epilogue, d.kind, d.gelu, d.C, d.heads, d.posmode, d.F = int(resid_epilogue), kind, int(gelu), C, heads, posmode, F
        d.qscale = float(qscale)
        tile = (ctypes.c_int32 * 2)()
        self._call("bt_debug_gemm", ctypes.byref(d), ptr(a), ptr(w), ptr(bias), ptr(resid), ptr(out_f32), ptr(out_act),
                   out_act.numel() if out_act is not None else 0, ptr(rope_cos), ptr(rope_sin), tile)
        return int(tile[0]), int(tile[1])

    def debug_attention(self, q, k, v, gates=None, key_lens=None, seqs_per_chunk=1, out=None):
        """gates * SDPA through the time-direction attention kernel; q/k/v [seqs, L, heads*32], gates [seqs*L, heads]
        (None: ones); key_lens: keys per chunk of seqs_per_chunk sequences (None: all L).  out: an fp32 device tensor
        of at least seqs*L*heads*32 elements (None: a new one shaped like q), written in place: the first
        seqs*L*heads*32 elements are the output, the rest keep their values.  Returns out."""
        seqs, L, C = q.shape
        if gates is None:
            gates = torch.ones(seqs * L, C // 32, dtype=torch.float32, device=self.device)
        o = torch.empty_like(q) if out is None else out
        p = self._dev_ptr
        lens = i32_array(key_lens) if key_lens is not None else None
        self._call("bt_debug_attention", p(q, q.numel()), p(k, q.numel()), p(v, q.numel()), p(gates, seqs * L * (C // 32)),
                   p(o, q.numel()), o.numel(), seqs, L, C // 32, lens, seqs_per_chunk)
        return o

    def debug_attention_backward(self, qkv, gates, freqs, dy):
        """bt_debug_attention_backward on qkv [seqs, n, 3 * heads * 32] (pre-RoPE), gates [seqs, n, heads] (logits),
        freqs [16] and dy [seqs, n, heads * 32] -> (y, dqkv, dgates) shaped like dy, qkv and gates."""
        seqs, n, C3 = qkv.shape
        heads = C3 // 96
        y, dqkv, dgates = torch.empty_like(dy), torch.empty_like(qkv), torch.empty_like(gates)
        p = self._dev_ptr
        self._call("bt_debug_attention_backward", p(qkv, qkv.numel()), p(gates, seqs * n * heads), p(freqs, 16),
                   p(dy, seqs * n * heads * 32), seqs, n, heads, p(y, dy.numel()), p(dqkv, qkv.numel()),
                   p(dgates, gates.numel()))
        return y, dqkv, dgates

    def debug_train_kernel(self, op: str, arrays, **desc):
        """bt_debug_train_kernel: the training kernel(s) of `op` (one of _lib.TRAIN_OPS) on `arrays`, the op's slots in
        the order include/beatthis.h lists them (None: absent), each a contiguous fp32 device tensor whose whole length
        is its element count; outputs are written in place.  desc: the bt_debug_train_desc fields the op reads."""
        d = _lib.bt_debug_train_desc()
        d.op = _lib.TRAIN_OPS.index(op)
        for k, v in desc.items():
            if not hasattr(d, k):
                raise TypeError(f"bt_debug_train_desc has no field {k}")
            setattr(d, k, v)
        n = len(arrays)
        ptrs = (c_void_p * max(n, 1))(*[self._dev_ptr(a) for a in arrays])
        counts = (ctypes.c_int64 * max(n, 1))(*[0 if a is None else a.numel() for a in arrays])
        self._call("bt_debug_train_kernel", ctypes.byref(d), ptrs, counts, n)

    def debug_attention_freq(self, q, k, v, gates, B, F, out=None):
        """gates * softmax over the F planes of each (chunk, frame, head); q/k/v [B*F*L, heads*32], gates [B*F*L, heads].
        out as for debug_attention (None: a new tensor shaped like q).  Returns out."""
        M, C = q.shape
        o = torch.empty_like(q) if out is None else out
        p = self._dev_ptr
        self._call("bt_debug_attention_freq", p(q, M * C), p(k, M * C), p(v, M * C), p(gates, M * (C // 32)), p(o, M * C),
                   o.numel(), B, F, M // (B * F), C // 32)
        return o

    # The row-kernel hooks take fp32 device tensors and write their outputs in place, so a caller can surround the
    # M rows with sentinel values.  x and every output may have more than M rows; only the first M are the problem.

    def debug_norm(self, x, xn_out, M: int, C: int, wg=None, bg=None, gates_out=None, heads: int = 0):
        """bt_debug_norm: xn_out[:M] = rmsnorm(x[:M]) through norm_kernel (+ gates_out[:M] with heads > 0)."""
        p, n = self._dev_ptr, max(M, 0)
        self._call("bt_debug_norm", p(x, n * C), p(xn_out, n * C), M, C, p(wg, heads * C), p(bg, heads),
                   p(gates_out, n * heads), heads)

    def debug_fused_qkv(self, x, wqkv, wg, bg, rope_cos, rope_sin, qkv_out, gates_out, M: int, C: int, L: int, F: int,
                        posmode: int, qscale: float):
        """bt_debug_fused_qkv: qkv_out[:M] (3C columns) and gates_out[:M] from x[:M] through fused_qkv_kernel<C>."""
        p, n, heads, rows = self._dev_ptr, max(M, 0), C // 32, 1500  # RoPE tables: [BT_CHUNK, 16]
        self._call("bt_debug_fused_qkv", p(x, n * C), p(wqkv, 3 * C * C), p(wg, heads * C), p(bg, heads),
                   p(rope_cos, rows * 16), p(rope_sin, rows * 16), p(qkv_out, n * 3 * C), p(gates_out, n * heads), M, C, L,
                   F, posmode, float(qscale))

    def debug_fused_ff(self, x, w1, b1, w2, b2, M: int, C: int, o=None, wout=None, xb_out=None):
        """bt_debug_fused_ff: x[:M] updated in place through fused_ff_kernel<C, o is not None> (+ xb_out[:M])."""
        p, n = self._dev_ptr, max(M, 0)
        self._call("bt_debug_fused_ff", p(x, n * C), p(w1, 4 * C * C), p(b1, 4 * C), p(w2, 4 * C * C), p(b2, C),
                   p(o, n * C), p(wout, C * C), p(xb_out, n * C), M, C)

    # The chunk-table hooks take the table as a sequence of (frame_base, T, start, out_base, write_lo, write_hi, len)
    # tuples (bt_debug_chunk); the library checks the table against the buffer lengths it is given.
    @staticmethod
    def _chunk_table(chunks):
        return (_lib.bt_debug_chunk * max(len(chunks), 1))(*[_lib.bt_debug_chunk(*map(int, c)) for c in chunks])

    def debug_stem(self, spect, chunks, L: int, bn1_scale, bn1_shift, w, bias, out):
        """bt_debug_stem: out [len(chunks), 32, L, 32] (fp32, in place) from spect [frames, 128] through stem_kernel."""
        p = self._dev_ptr
        self._call("bt_debug_stem", p(spect), spect.numel() // 128, self._chunk_table(chunks), len(chunks), L,
                   p(bn1_scale, 128), p(bn1_shift, 128), p(w, 32 * 12), p(bias, 32), p(out), out.numel())

    def debug_zero_tail(self, buf, chunks, F: int, L: int, C: int):
        """bt_debug_zero_tail: rows [len, L) of every plane of buf [len(chunks), F, L, C] (fp32 or 16-bit, in place)
        cleared through zero_tail_kernel."""
        assert buf.element_size() in (2, 4)
        self._call("bt_debug_zero_tail", self._dev_ptr(buf, dtype=buf.dtype), buf.element_size(), self._chunk_table(chunks),
                   len(chunks), F, L, C, buf.numel() * buf.element_size())

    def debug_head(self, x, D: int, w, b, chunks, L: int, sum_head: bool, beat, down):
        """bt_debug_head: the owned frames of beat / down (fp32, in place) from x [len(chunks), L, D] through head_kernel."""
        p = self._dev_ptr
        assert beat.numel() == down.numel()
        self._call("bt_debug_head", p(x, len(chunks) * L * D), D, p(w, 2 * D), p(b, 2), self._chunk_table(chunks),
                   len(chunks), L, int(bool(sum_head)), p(beat), p(down), beat.numel())
