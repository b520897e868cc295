"""Host <-> device pipeline behind ``Audio2Frames.batch`` / ``Audio2Beats.batch`` / ``File2Beats.batch``.

The reference handles one clip at a time on one stream (reference beat_this/inference.py:215,269-281: numpy mono mix,
``torch.tensor(signal, device=...)``, model, ``.cpu()``).  Here a call is cut into *groups* of clips (one group =
one pass of every kernel); for every group

  host threads   mono mix + fp32 cast of all clips straight into a pinned ring slot (``bt_stage_audio`` /
                 ``bt_stage_wav_files``: C++, GIL released); for FLAC and MP3 files, their frame bytes and frame
                 tables (``bt_stage_flac_files``, ``bt_stage_mp3_files``)
  copy stream    one H2D copy of the slot
  compute stream [FLAC / MP3: decode and mono mix (``bt_flac_decode``, ``bt_mp3_decode``)] -> log-mel -> BeatThis forward -> (peak picking
                 | device DBN -> D2H of the timestamps | D2H of the logits for the host DBN)

and group g+1 is staged and copied while the kernels of group g run; results are collected in order.  Nothing in the
enqueue path waits for the GPU (the C library keeps its small tables in a ring of pinned slots), so the device queue
stays one group ahead of the host.
"""
from __future__ import annotations

import time
from collections import deque

import numpy as np
import torch

from . import _lib
from ._lib import DEFAULT_CHUNKING


def as_signal_array(signal) -> np.ndarray:
    """What Audio2Frames.signal2spect accepts (reference inference.py:269-273): 1-D or 2-D (time, channels) array-like.
    Returns a C-contiguous float32 / float64 / int16 ndarray without copying when the input already is one."""
    if isinstance(signal, torch.Tensor):
        signal = signal.detach().cpu().numpy()
    a = np.asarray(signal)
    if a.ndim not in (1, 2):
        raise ValueError(f"Expected 1D or 2D signal, got shape {a.shape}")
    if a.dtype not in _lib.SIGNAL_DTYPES:
        a = a.astype(np.float64)  # ints other than int16, float16, ...: the reference's mean(1) works in float64 too
    return np.ascontiguousarray(a)


def plan_groups(costs, max_cost: int, max_clips: int):
    """Consecutive clips -> groups of at most `max_clips` clips / `max_cost` total cost (a clip above the limit is a
    group of its own).  Returns a list of (first, last+1) index pairs."""
    groups, lo, acc = [], 0, 0
    for i, n in enumerate(costs):
        if i > lo and (acc + n > max_cost or i - lo >= max_clips):
            groups.append((lo, i))
            lo, acc = i, 0
        acc += int(n)
    if lo < len(costs):
        groups.append((lo, len(costs)))
    return groups


def padded_frames(n_samples: int, sr: int, chunk_size: int, border_size: int) -> int:
    """Frames a clip of n_samples at `sr` Hz occupies in the waves of the C library under a chunking: its chunks
    (split_piece, inference.py:119-125) times chunk_size, the most a chunk is padded to."""
    frames = 1 + (int(n_samples) * 22050 // max(1, int(sr))) // 441
    return max(1, -(-frames // (int(chunk_size) - 2 * int(border_size)))) * int(chunk_size)


def _check_frames_route(want: str, chunking) -> None:
    """Only framewise logits take another chunking than 1500 / 6 / keep_first: the beat routes keep the reference's
    Audio2Beats, which always cuts that way (inference.py:244-254)."""
    if chunking != DEFAULT_CHUNKING and want != "frames":
        raise ValueError(f'a chunking applies to want="frames" only, not want="{want}"')


class _Slot:
    def __init__(self):
        self.host = None      # pinned fp32 staging buffer
        self.dev = None       # device copy
        self.copied = None
        self.peak = {}        # reusable buffers of Engine.peakpick_async
        self.dbn = {}         # reusable buffers of Engine.dbn_async
        self.logits_h = None  # pinned logits (DBN path)
        self.done = None
        self.t0 = None        # events around the group's kernels (stats: GPU busy time)
        self.t1 = None
        self.flac_host = None  # pinned bytes of a FLAC or MP3 group (_lib.flac_layout, _lib.mp3_layout), its device
        self.flac_dev = None   # copy and the D2H copy of its files' statuses
        self.flac_status = None
        self.flac_files = 0    # FLAC or MP3 files of the group in flight (0: not a compressed group)


class BeatPipeline:
    """Ring of `depth` slots; `submit_*` enqueues one group, `collect` returns the oldest group's result."""

    # staging slots are sized once for a full group (128 chunks = 128 * 1488 frames of 441 samples, 336 MB of fp32):
    # page-locking hundreds of MB takes ~0.1 s, which must not recur while batches stream through
    SLOT_SAMPLES = 128 * 1488 * 441 + 6 * 441

    def __init__(self, engine, depth: int = 3, host_threads: int | None = None):
        self.engine = engine
        self.device = engine.device
        self.copy_stream = torch.cuda.Stream(self.device)
        self.compute_stream = torch.cuda.Stream(self.device)
        self.slots = [_Slot() for _ in range(depth)]
        self.free = deque(range(depth))
        self.inflight = deque()
        if host_threads is None:
            import os

            try:
                n = len(os.sched_getaffinity(0))
            except AttributeError:
                n = os.cpu_count() or 1
            host_threads = max(1, min(32, n))
        self.host_threads = int(host_threads)
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        self.dbn_params = None  # tracker parameters of want="dbn_device" (Postprocessor.dbn_params)
        self.last_status = None  # per-file statuses of the last collected FLAC or MP3 group (collect)
        # host seconds spent staging (mono mix / decode into pinned memory), enqueueing and waiting for results
        self.stats = {"stage_s": 0.0, "enqueue_s": 0.0, "collect_wait_s": 0.0, "gpu_busy_s": 0.0, "groups": 0}

    # ---- staging --------------------------------------------------------------------------------
    def _slot(self, n_samples: int):
        if not self.free:
            raise RuntimeError("pipeline full: collect() a result first")
        idx = self.free.popleft()
        s = self.slots[idx]
        if s.host is None or s.host.numel() < n_samples:
            cap = max(int(n_samples), self.SLOT_SAMPLES)
            s.host = torch.empty(cap, dtype=torch.float32, pin_memory=True)
            s.dev = torch.empty(cap, dtype=torch.float32, device=self.device)
            s.copied = torch.cuda.Event()
        return idx, s

    def stage_signals(self, arrays, dst: torch.Tensor):
        """Mono mix + fp32 cast of C-contiguous ndarrays (see as_signal_array) into `dst` (host fp32 tensor);
        returns the sample offsets."""
        return _lib.stage_audio(arrays, dst, self.host_threads)

    def _enqueue(self, idx, s, so, sr, want, chunking=DEFAULT_CHUNKING, flac=None):
        """flac: (decode, streams, status offset, bytes) of a compressed (FLAC or MP3) group staged in s.flac_host,
        decoded into s.dev on the compute stream by decode(buf, streams, mode, out, status offset) (an Engine
        method); otherwise s.host holds the group's mono fp32 samples."""
        n = so[-1]
        with torch.cuda.stream(self.copy_stream):
            if flac is None:
                s.dev[:n].copy_(s.host[:n], non_blocking=True)
            else:
                s.flac_dev[: flac[3]].copy_(s.flac_host[: flac[3]], non_blocking=True)
            s.copied.record(self.copy_stream)
        self.h2d_bytes += n * 4 if flac is None else flac[3]
        eng = self.engine
        if s.t0 is None:
            s.t0, s.t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(self.compute_stream):
            self.compute_stream.wait_event(s.copied)
            s.t0.record(self.compute_stream)
            s.flac_files = 0
            if flac is not None:
                decode, streams, status_at, _ = flac
                decode(s.flac_dev, streams, _lib.BT_FLAC_MONO_F32, s.dev, status_at)
                s.flac_files = len(streams)
                s.flac_status[: len(streams)].copy_(s.flac_dev[status_at : status_at + 4 * len(streams)].view(torch.int32),
                                                    non_blocking=True)
            audio, offs = s.dev[:n], so
            if sr != 22050:
                audio, offs = eng.resample_cat(audio, so, sr)
            beat, down, fo = eng.audio2frames_cat(audio, offs, chunking)
            if want == "beats":
                handle = eng.peakpick_async(beat, down, fo, s.peak)
                self.d2h_bytes += handle.d2h_bytes
                payload = ("beats", handle)
            elif want == "dbn_device":  # the DBN on the compute stream: no logits leave the device, no host thread
                if self.dbn_params is None:
                    raise RuntimeError('want="dbn_device" needs BeatPipeline.dbn_params')
                handle = eng.dbn_async(beat, down, fo, s.dbn, self.dbn_params)
                self.d2h_bytes += handle.d2h_bytes
                payload = ("beats", handle)
            elif want == "logits_host":
                total = fo[-1]
                if s.logits_h is None or s.logits_h.shape[1] < total:
                    s.logits_h = torch.empty((2, max(int(total * 1.25), 1024)), dtype=torch.float32, pin_memory=True)
                s.logits_h[0, :total].copy_(beat, non_blocking=True)
                s.logits_h[1, :total].copy_(down, non_blocking=True)
                s.done = torch.cuda.Event()
                s.done.record(self.compute_stream)
                self.d2h_bytes += total * 8
                payload = ("logits_host", (s, fo, (beat, down)))
            else:  # device logits
                s.done = torch.cuda.Event()
                s.done.record(self.compute_stream)
                payload = ("frames", (s, beat, down, fo))
            s.t1.record(self.compute_stream)
        self.inflight.append((idx, payload))

    def submit_signals(self, arrays, sr: int = 22050, want: str = "beats", chunking: tuple = DEFAULT_CHUNKING):
        """chunking (want="frames" only): (chunk_size, border_size, overlap_mode), see Engine.spect2frames_cat."""
        _check_frames_route(want, chunking)
        idx, s = self._slot(sum(a.shape[0] for a in arrays))
        try:
            t0 = time.perf_counter()
            so = self.stage_signals(arrays, s.host)
            t1 = time.perf_counter()
            self._enqueue(idx, s, so, int(sr), want, chunking)
            self.stats["stage_s"] += t1 - t0
            self.stats["enqueue_s"] += time.perf_counter() - t1
            self.stats["groups"] += 1
        except Exception:
            self.free.append(idx)
            raise

    def submit_wavs(self, paths, infos, sr: int, want: str = "beats", chunking: tuple = DEFAULT_CHUNKING):
        """paths: list of str; infos: list of bt_wav_info (all `sr` Hz) from _lib.wav_probe; chunking as in
        submit_signals."""
        _check_frames_route(want, chunking)
        so = _lib.offsets(info.frames for info in infos)
        idx, s = self._slot(so[-1])
        try:
            t0 = time.perf_counter()
            _lib.stage_wav_files(paths, infos, s.host, so, self.host_threads)
            t1 = time.perf_counter()
            self._enqueue(idx, s, so, int(sr), want, chunking)
            self.stats["stage_s"] += t1 - t0
            self.stats["enqueue_s"] += time.perf_counter() - t1
            self.stats["groups"] += 1
        except Exception:
            self.free.append(idx)
            raise

    def submit_flacs(self, paths, infos, sr: int, want: str = "beats", chunking: tuple = DEFAULT_CHUNKING):
        """paths: list of str; infos: list of bt_flac_info (all `sr` Hz, total_samples known) from _lib.probe_audio;
        chunking as in submit_signals.  Host threads stage the frame bytes and tables, the device decodes them and mixes
        to mono (bt_flac_decode), and the group runs on as submit_wavs's.  A file that fails to stage or decode runs as
        zeros of its STREAMINFO length; `last_status` gives every file's status when the group is collected."""

        def stage(buf_ptr):
            nf, ns, status = _lib.stage_flac_files(paths, infos, buf_ptr, self.host_threads)
            # staging checks the block sizes against STREAMINFO's total, so a staged file has its so length; one that
            # failed is not decoded and runs as zeros of that length
            return _lib.flac_streams(infos, nf, [info.total_samples for info in infos], so[:-1]), status

        so = _lib.offsets(info.total_samples for info in infos)
        self._submit_compressed(so, _lib.flac_layout(infos), stage, self.engine.flac_decode, len(paths), sr, want,
                                chunking)

    def submit_mp3s(self, paths, infos, sr: int, want: str = "beats", chunking: tuple = DEFAULT_CHUNKING):
        """paths: list of str; infos: list of bt_mp3_info (all `sr` Hz) from _lib.probe_audio; chunking as in
        submit_signals.  Host threads stage the main data and frame tables, the device decodes them and mixes to mono
        (bt_mp3_decode), and the group runs on as submit_wavs's.  A file that fails to stage or decode runs as zeros of
        its probed length; `last_status` gives every file's status when the group is collected."""

        def stage(buf_ptr):
            nf, mb, status = _lib.stage_mp3_files(paths, infos, buf_ptr, self.host_threads)
            return _lib.mp3_streams(infos, nf, mb, so[:-1]), status

        so = _lib.offsets(info.n_samples for info in infos)
        self._submit_compressed(so, _lib.mp3_layout(infos), stage, self.engine.mp3_decode, len(paths), sr, want,
                                chunking)

    def submit_vorbis(self, paths, infos, sr: int, want: str = "beats", chunking: tuple = DEFAULT_CHUNKING):
        """paths: list of str; infos: list of bt_vorbis_info (all `sr` Hz) from _lib.probe_audio; chunking as in
        submit_signals.  Host threads stage the audio packets, packet tables and decode tables, the device decodes them
        and mixes to mono (bt_vorbis_decode), and the group runs on as submit_wavs's.  A file that fails to stage or
        decode runs as zeros of its probed length; `last_status` gives every file's status when the group is
        collected."""

        def stage(buf_ptr):
            npk, pb, bs, status = _lib.stage_vorbis_files(paths, infos, buf_ptr, self.host_threads)
            return _lib.vorbis_streams(infos, npk, pb, bs, so[:-1]), status

        so = _lib.offsets(info.n_samples for info in infos)
        self._submit_compressed(so, _lib.vorbis_layout(infos), stage, self.engine.vorbis_decode, len(paths), sr, want,
                                chunking)

    def _submit_compressed(self, so, layout, stage, decode, n_files, sr, want, chunking):
        """One group of compressed files: so, their sample offsets; layout, where the staged frame tables, statuses and
        frame data sit (_lib.flac_layout, _lib.mp3_layout); stage(host address) fills a pinned buffer and returns (streams,
        statuses); decode is the Engine method that decodes the streams on the compute stream.  A file whose staging
        failed is not decoded (no frames) and runs as zeros."""
        _check_frames_route(want, chunking)
        _, status_at, _, total = layout
        idx, s = self._slot(so[-1])
        try:
            t0 = time.perf_counter()
            if s.flac_host is None or s.flac_host.numel() < total:
                cap = max(int(total * 1.25), 1 << 20)
                s.flac_host = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
                s.flac_dev = torch.empty(cap, dtype=torch.uint8, device=self.device)
            if s.flac_status is None or s.flac_status.numel() < n_files:
                s.flac_status = torch.empty(max(n_files, 64), dtype=torch.int32, pin_memory=True)
            streams, status = stage(s.flac_host.data_ptr())
            for i, st in enumerate(status):
                if st != 0:
                    if hasattr(streams[i], "n_packets"):
                        streams[i].n_packets = 0
                    else:
                        streams[i].n_frames = 0
            t1 = time.perf_counter()
            self._enqueue(idx, s, so, int(sr), want, chunking, (decode, streams, status_at, total))
            self.stats["stage_s"] += t1 - t0
            self.stats["enqueue_s"] += time.perf_counter() - t1
            self.stats["groups"] += 1
        except Exception:
            self.free.append(idx)
            raise

    def submit_pinned(self, audio_host: torch.Tensor, sample_offsets, sr: int = 22050, want: str = "beats"):
        """Mono fp32 audio already in one pinned host tensor (clips back to back)."""
        so = [int(v) for v in sample_offsets]
        idx, s = self._slot(so[-1])
        s.host[: so[-1]].copy_(audio_host[: so[-1]])
        self._enqueue(idx, s, so, int(sr), want)

    # ---- results ----------------------------------------------------------------------------------
    def collect(self):
        """Oldest group: list of (beat_times, downbeat_times) ["beats", "dbn_device"], (beat, down, fo) host arrays
        ["logits_host"] or device tensors ["frames"].  After it, last_status lists the status (BT_OK or BT_ERR_IO) of
        every file of a FLAC or MP3 group, and is None for other groups."""
        idx, (kind, p) = self.inflight.popleft()
        t0 = time.perf_counter()
        self.last_status = None
        try:
            if kind == "beats":
                out = p.result()
            elif kind == "logits_host":
                s, fo, _keep = p
                s.done.synchronize()
                total = fo[-1]
                out = s.logits_h[0, :total].numpy().copy(), s.logits_h[1, :total].numpy().copy(), fo
            else:
                s, beat, down, fo = p
                s.done.synchronize()
                out = beat, down, fo
            s = self.slots[idx]
            if s.flac_files:  # the status copy precedes the group's last event on the compute stream
                self.last_status = s.flac_status[: s.flac_files].tolist()
            return out
        finally:
            self.stats["collect_wait_s"] += time.perf_counter() - t0
            try:
                self.slots[idx].t1.synchronize()
                self.stats["gpu_busy_s"] += self.slots[idx].t0.elapsed_time(self.slots[idx].t1) / 1000.0
            except Exception:
                pass
            self.free.append(idx)

    def run(self, n_groups: int, submit):
        """Call submit(g) for g in range(n_groups), keeping the ring full; yields the results in order."""
        for g in range(n_groups):
            if not self.free:
                yield self.collect()
            submit(g)
        while self.inflight:
            yield self.collect()

    def drain(self):
        while self.inflight:
            try:
                self.collect()
            except Exception:
                pass
