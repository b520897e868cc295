"""Postprocessor mirror (reference beat_this/model/postprocessor.py:9-197).

``type="minimal"``: peak picking (max-pool 7 equality and logit > 0), adjacent-peak merging,
downbeat snapping and ``np.unique`` all run in one device kernel (``bt_peakpick_fps``); only the
final timestamp arrays come back to the host.  ``type="dbn"``: the DBN stays on the host as in the
reference (postprocessor.py:138-173): madmom's ``DBNDownBeatTrackingProcessor`` when madmom is
installed (exactly the reference's object), otherwise the restatement of its published algorithm in
``beat_this_b200/dbn.py`` (parity with madmom unpinned); ``dbn_impl`` forces one of the two ("madmom", "native").
``dbn_impl="device"`` decodes on the GPU instead (``bt_dbn_track_device``: sigmoid, clamps, Viterbi and beat
correction in three kernels, pinned to the host C++ tracker); only the beat times come back to the host.

``fps`` is the frame rate of the predictions, as in the reference: any finite rate > 0, an integer or not (a model
trained on another hop, madmom-style 100 fps activations).  The peak picker divides peak frames by it
(``bt_peakpick_fps``) and every DBN is built at it.
"""
from __future__ import annotations

import math
import numbers
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib


def check_fps(fps) -> None:
    """ValueError unless `fps` is a finite real number > 0 (bools are not frame rates)."""
    if isinstance(fps, bool) or not isinstance(fps, numbers.Real) or not math.isfinite(fps) or not fps > 0:
        raise ValueError(f"fps must be a finite number > 0, got {fps!r}")


class Postprocessor:
    def __init__(self, type: str = "minimal", fps: float = 50, engine=None, device="cuda", dbn_impl: str = "auto"):
        assert type in ["minimal", "dbn"]
        assert dbn_impl in ["auto", "madmom", "native", "device"]
        check_fps(fps)
        self.type = type
        self.dbn_impl = dbn_impl
        self.fps = fps
        if type == "dbn":
            kw = dict(beats_per_bar=[3, 4], min_bpm=55.0, max_bpm=215.0, fps=self.fps, transition_lambda=100)
            self.dbn = None
            if dbn_impl in ("auto", "madmom"):
                try:
                    from madmom.features.downbeats import DBNDownBeatTrackingProcessor

                    self.dbn = DBNDownBeatTrackingProcessor(**kw)
                except ImportError:
                    if dbn_impl == "madmom":
                        raise
            if self.dbn is None:
                from .dbn import DBNDownBeatTracker

                self.dbn = DBNDownBeatTracker(**kw)
        if engine is None:
            from .engine import Engine

            engine = Engine.mel_only(device)  # a weight-less context is enough for bt_peakpick
        self.engine = engine

    def __call__(self, beat: torch.Tensor, downbeat: torch.Tensor, padding_mask: torch.Tensor | None = None):
        """Works with batched ([B,T]) and unbatched ([T]) logits like the reference; returns
        (beat_times, downbeat_times) or tuples of them for batched input."""
        batched = beat.ndim != 1
        if not batched:
            beat, downbeat = beat.unsqueeze(0), downbeat.unsqueeze(0)
            if padding_mask is not None:
                padding_mask = padding_mask.unsqueeze(0)
        dev = self.engine.device
        beat = torch.as_tensor(beat, device=dev).float()
        downbeat = torch.as_tensor(downbeat, device=dev).float()
        if padding_mask is None:
            lengths = [beat.shape[1]] * beat.shape[0]
        else:
            # the reference truncates each piece to its un-padded frames (postprocessor.py:116-117);
            # padding is trailing by construction
            lengths = [int(m.sum()) for m in padding_mask.to(torch.bool).cpu()]
        fo = _lib.offsets(lengths)
        bcat = torch.cat([beat[i, :n] for i, n in enumerate(lengths)]).contiguous()
        dcat = torch.cat([downbeat[i, :n] for i, n in enumerate(lengths)]).contiguous()
        res = self.batch_cat(bcat, dcat, fo)
        if not batched:
            return res[0]
        return tuple(r[0] for r in res), tuple(r[1] for r in res)

    def batch_cat(self, beat: torch.Tensor, downbeat: torch.Tensor, frame_offsets):
        """Concatenated logits of many clips -> list of (beat_times, downbeat_times)."""
        if self.type == "minimal":
            return self.engine.peakpick_cat(beat, downbeat, frame_offsets, self.fps)
        return self._postp_dbn(beat, downbeat, frame_offsets)

    @property
    def on_device(self) -> bool:
        """True when the DBN runs on the GPU (dbn_impl="device")."""
        return self.type == "dbn" and self.dbn_impl == "device"

    @property
    def dbn_params(self) -> dict:
        """Tracker parameters of the device DBN (dbn.DBNDownBeatTracker.track_params)."""
        return self.dbn.track_params

    def _postp_dbn(self, beat, downbeat, frame_offsets):
        if self.on_device:
            beat = beat.to(self.engine.device, torch.float32).contiguous()
            downbeat = downbeat.to(self.engine.device, torch.float32).contiguous()
            return self.engine.dbn_cat(beat, downbeat, frame_offsets, self.dbn_params)
        return self.batch_host(beat.float().cpu().numpy(), downbeat.float().cpu().numpy(), frame_offsets)

    def batch_host(self, beat_logits: np.ndarray, downbeat_logits: np.ndarray, frame_offsets):
        """DBN post-processing of concatenated host logits (reference postprocessor.py:138-173, float64 on the host):
        list of (beat_times, downbeat_times)."""
        assert self.type == "dbn"
        if self.on_device:  # fp32 logits, as the model produces them
            dev = self.engine.device
            beat = torch.as_tensor(np.ascontiguousarray(beat_logits), dtype=torch.float32).to(dev)
            down = torch.as_tensor(np.ascontiguousarray(downbeat_logits), dtype=torch.float32).to(dev)
            return self.engine.dbn_cat(beat, down, frame_offsets, self.dbn_params)
        eps = 1e-5
        # beat.double().sigmoid() with the reference's own torch op (postprocessor.py:139-140) -- on ONE thread: a
        # 100 k element op gains nothing from torch's intra-op pool, and waking a 128-thread pool costs tens of ms
        nthr = torch.get_num_threads()
        torch.set_num_threads(1)
        try:
            bp = torch.from_numpy(np.ascontiguousarray(beat_logits)).double().sigmoid().numpy()
            dp = torch.from_numpy(np.ascontiguousarray(downbeat_logits)).double().sigmoid().numpy()
        finally:
            torch.set_num_threads(nthr)
        bp = bp * (1 - eps) + eps / 2
        dp = dp * (1 - eps) + eps / 2

        # the artificial multiclass prediction of postprocessor.py:159-167, for all pieces at once: [total, 2]
        act = np.stack((np.maximum(bp - dp, eps / 2), dp), axis=1)

        def split(out):
            return out[:, 0], out[out[:, 1] == 1][:, 0]

        n = len(frame_offsets) - 1
        if hasattr(self.dbn, "batch_cat"):  # native tracker: all pieces in one multi-threaded C++ call
            return [split(o) for o in self.dbn.batch_cat(act, frame_offsets)]
        with ThreadPoolExecutor() as ex:  # madmom: one piece per thread, as in the reference
            return list(ex.map(lambda i: split(self.dbn(act[frame_offsets[i] : frame_offsets[i + 1]])), range(n)))
