"""Drop-in mirror of the reference ``beat_this.inference`` API (reference beat_this/inference.py:16-315): same
function and class names, constructor and call signatures, return types and exceptions -- with everything between
"audio samples" and "beat timestamps" executed by the sm_90a CUDA library.

Differences a user can observe:
* ``device`` must be a CUDA device (default ``"cuda"``); ``device="cpu"`` raises.
* ``float16=False`` -> fp32 CUDA-core kernels (reference-exact numerics, <=1e-3 on logits);
  ``float16=True`` -> fp16-operand tensor-core kernels with fp32 accumulation and an fp32 residual stream
  (the reference autocasts to fp16 here as well, inference.py:245-246).
* every class has a ``batch(...)`` method that processes many clips per call through the host/device pipeline of
  ``beat_this_b200.pipeline`` (the reference is strictly one clip, one chunk at a time: inference.py:215).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib
from ._lib import BT_CHUNK, DEFAULT_CHUNKING, MAX_CHUNK_CAP
from .engine import Engine, chunking_struct
from .pipeline import BeatPipeline, as_signal_array, padded_frames, plan_groups
from .postprocessor import Postprocessor
from .preprocessing import LogMelSpect, load_audio
from .utils import replace_state_dict_key, save_beat_tsv
from .weights import filter_hparams, pack_parameters

CHECKPOINT_URL = "https://cloud.cp.jku.at/public.php/dav/files/7ik4RrBKTS273gp"

# one group = one pass of every kernel over up to GROUP_CHUNKS model passes (chunks of 1500 frames): 64 clips of 30 s
# (two chunks each, inference.py:119-125), one full wave of the C library
GROUP_CHUNKS = 128
GROUP_CLIPS = 256


def _checkpoint_source(name) -> tuple[str, str | None]:
    """(url, cache file name) for a checkpoint that is not a local file: a full URL is taken as is, anything else is
    a short name (``final0``, ``small1`` ...) below CHECKPOINT_URL (reference inference.py:34-45)."""
    name = str(name)
    if name.startswith(("https://", "http://")):
        return name, None
    return f"{CHECKPOINT_URL}/{name}.ckpt", f"beat_this-{name}.ckpt"


def load_checkpoint(checkpoint_path: str, device: str | torch.device = "cpu") -> dict:
    """Checkpoint dictionary from a local file, a short name or a URL (reference inference.py:16-53; names and URLs
    go through the torch.hub cache and need network).  ``ValueError`` when nothing can be loaded."""
    try:
        return torch.load(checkpoint_path, map_location=device, weights_only=True)
    except FileNotFoundError:
        pass
    url, file_name = _checkpoint_source(checkpoint_path)
    try:
        return torch.hub.load_state_dict_from_url(url, file_name=file_name, map_location=device)
    except Exception:
        raise ValueError("Could not load the checkpoint given the provided name", checkpoint_path)


class BeatThisB200:
    """What ``load_model`` returns in place of the reference ``BeatThis`` nn.Module: the packed
    weights living on one GPU inside a ``bt_ctx``."""

    def __init__(self, hparams: dict, packed: dict, device, float16: bool = False, wave_chunks: int | None = None):
        self.checkpoint_hparams = dict(hparams)  # all of them, the training ones (loss_type, pos_weights ...) included
        self.hparams = filter_hparams(hparams)
        self.engine = Engine(packed, self.hparams, device, half=float16, wave_chunks=wave_chunks)
        self.device = self.engine.device
        self.float16 = float16
        # the longest chunk the model runs: the rows of the packed RoPE tables (load_model's max_chunk_size)
        self.max_chunk_size = self.engine.max_chunk

    def eval(self):
        return self

    def to(self, device):
        if torch.device(device).type != "cuda":
            raise RuntimeError("beat_this_b200 models live on a CUDA device; there is no CPU fallback")
        return self

    def __call__(self, spect: torch.Tensor) -> dict:
        """BeatThis.forward (reference beat_tracker.py:188-192) for a batch of equal-length spectrogram chunks
        [B, T<=max_chunk_size, 128]: every chunk runs as its own piece without borders being cut."""
        if spect.ndim != 3 or spect.shape[2] != 128 or spect.shape[1] > self.max_chunk_size:
            raise ValueError(f"Expected [B, T<={self.max_chunk_size}, 128] chunks (T up to the model's max_chunk_size), "
                             f"got {tuple(spect.shape)}")
        B, T, _ = spect.shape
        beat, down = self.engine.forward_chunks(spect.to(self.device, torch.float32).contiguous())
        return {"beat": beat.view(B, T), "downbeat": down.view(B, T)}


def check_max_chunk_size(max_chunk_size) -> int:
    """The max_chunk_size keyword of load_model and the inference classes: an integer in [1500, 384000].  1500 is the
    reference's inference chunk; a model trained on longer sequences (train.py --train-length) may run longer ones."""
    if not isinstance(max_chunk_size, (int, np.integer)) or isinstance(max_chunk_size, bool) or \
            not BT_CHUNK <= max_chunk_size <= MAX_CHUNK_CAP:
        raise ValueError(f"max_chunk_size must be an integer in [{BT_CHUNK}, {MAX_CHUNK_CAP}], got {max_chunk_size!r}")
    return int(max_chunk_size)


def load_model(checkpoint_path: str | dict | None = "final0", device: str | torch.device = "cuda", float16: bool = False,
               wave_chunks: int | None = None, max_chunk_size: int = BT_CHUNK) -> BeatThisB200:
    """Load a BeatThis model from a checkpoint (reference inference.py:56-87).  Accepts the
    reference ``.ckpt`` layout unchanged (``hyper_parameters`` + ``state_dict`` with the
    ``model.`` prefix).  ``checkpoint_path`` may also be an already loaded checkpoint dict.
    max_chunk_size: the longest chunk the model will run (its RoPE tables' length), 1500 by default; chunk sizes up
    to it are accepted by split_predict_aggregate, spects2frames, frames_batch and the model call.  It is not read
    from the checkpoint."""
    from .engine import _cuda_device

    _cuda_device(device)  # fail before touching the checkpoint: there is no CPU path
    max_chunk_size = check_max_chunk_size(max_chunk_size)
    if checkpoint_path is None:
        raise ValueError("beat_this_b200 needs a checkpoint (the reference's random-init BeatThis() has no use here)")
    checkpoint = checkpoint_path if isinstance(checkpoint_path, dict) else load_checkpoint(checkpoint_path, "cpu")
    hparams = checkpoint["hyper_parameters"]
    state_dict = replace_state_dict_key(dict(checkpoint["state_dict"]), "model.", "")
    packed = pack_parameters(state_dict, filter_hparams(hparams), rope_positions=max_chunk_size)
    return BeatThisB200(hparams, packed, device, float16, wave_chunks)


# ------------------------------------------------------------------------------------------------------------
# Chunking helpers of the reference API (inference.py:90-230).  The CUDA path never calls them -- bt_plan_chunking
# plans natively and the stem / head kernels gather and scatter in place -- they serve users of the reference's
# function-level API and are pinned to the reference by tests/golden/chunking.npz and chunking_modes.npz.
# ------------------------------------------------------------------------------------------------------------
def chunk_starts(n_frames: int, chunk_size: int, border_size: int = 6, avoid_short_end: bool = True) -> np.ndarray:
    """First frame of every chunk: windows advance by chunk_size - 2*border_size from -border_size; with
    `avoid_short_end` the last window is pulled back so that it ends border_size frames past the piece
    (same plan as bt_plan_chunks for 1500 / 6)."""
    step = chunk_size - 2 * border_size
    if step <= 0:
        raise ValueError("chunk_size must exceed twice the border")
    count = max(0, math.ceil(n_frames / step))
    starts = step * np.arange(count, dtype=np.int64) - border_size
    if avoid_short_end and count and n_frames > step:
        starts[-1] = n_frames + border_size - chunk_size
    return starts


def zeropad(spect: torch.Tensor, left: int = 0, right: int = 0) -> torch.Tensor:
    """`left` / `right` zero frames around a [T, F] spectrogram (reference inference.py:90-97)."""
    if left <= 0 and right <= 0:
        return spect
    T = spect.shape[0]
    out = spect.new_zeros((left + T + right,) + tuple(spect.shape[1:]))
    out[left : left + T] = spect
    return out


def split_piece(spect: torch.Tensor, chunk_size: int, border_size: int = 6, avoid_short_end: bool = True):
    """Chunks (zero padded by up to border_size frames at the piece boundaries) and their start frames, as reference
    inference.py:100-135 returns them; all chunks are views of ONE padded copy of the piece."""
    T = len(spect)
    starts = chunk_starts(T, chunk_size, border_size, avoid_short_end)
    padded = zeropad(spect, border_size, border_size)  # frame t lives at row t + border_size
    chunks = [padded[s + border_size : min(s + chunk_size, T + border_size) + border_size] for s in starts.tolist()]
    return chunks, starts


def aggregate_prediction(pred_chunks: list, starts: list, full_size: int, chunk_size: int, border_size: int,
                         overlap_mode: str, device: str | torch.device) -> tuple[torch.Tensor, torch.Tensor]:
    """Piece-level logits from chunk-level ones (reference inference.py:138-185): every chunk loses border_size frames
    on both sides, overlaps go to the earlier ("keep_first") or later ("keep_last") chunk, frames no chunk covers
    stay at -1000.  Every frame is written once, from the chunk that owns it."""
    if overlap_mode not in ("keep_first", "keep_last"):
        raise ValueError("overlap_mode must be 'keep_first' or 'keep_last'")
    beat = torch.full((full_size,), -1000.0, device=device)
    downbeat = torch.full((full_size,), -1000.0, device=device)
    starts = [int(s) for s in starts]
    spans = [(s + border_size, s + len(p["beat"]) - border_size) for s, p in zip(starts, pred_chunks)]
    order = range(len(spans)) if overlap_mode == "keep_first" else range(len(spans) - 1, -1, -1)
    claimed_lo, claimed_hi = None, None  # frames already owned: one interval, chunks are visited in order
    for i in order:
        lo, hi = max(spans[i][0], 0), min(spans[i][1], full_size)
        if claimed_lo is not None:
            if overlap_mode == "keep_first":
                lo = max(lo, claimed_hi)
            else:
                hi = min(hi, claimed_lo)
        if hi > lo:
            off = lo - starts[i]
            beat[lo:hi] = pred_chunks[i]["beat"][off : off + hi - lo]
            downbeat[lo:hi] = pred_chunks[i]["downbeat"][off : off + hi - lo]
            claimed_lo = lo if claimed_lo is None else min(claimed_lo, lo)
            claimed_hi = hi if claimed_hi is None else max(claimed_hi, hi)
    return beat, downbeat


def engine_chunking(chunk_size: int, border_size: int, overlap_mode: str, max_chunk_size: int = BT_CHUNK) -> tuple:
    """The `chunking` argument of Engine.spect2frames_cat / audio2frames_cat for split_predict_aggregate's values: the
    checked triple.  ``ValueError`` for values the CUDA path cannot run (engine.chunking_struct; chunk_size up to the
    model's max_chunk_size)."""
    chunking_struct(chunk_size, border_size, overlap_mode, max_chunk_size)
    return int(chunk_size), int(border_size), overlap_mode


def _plan_groups(n_samples, sr: int, chunking: tuple):
    """Groups of consecutive clips for the pipeline: the padded frames of GROUP_CHUNKS 1500-frame chunks each, so that
    a group of long chunks fits one wave's frame budget (bt_set_wave_chunks)."""
    return plan_groups([padded_frames(n, sr, *chunking[:2]) for n in n_samples], GROUP_CHUNKS * BT_CHUNK, GROUP_CLIPS)


def split_predict_aggregate(spect: torch.Tensor, chunk_size: int, border_size: int, overlap_mode: str,
                            model) -> dict:
    """Reference inference.py:188-230: chunk the piece, run `model` on every chunk, stitch.  A ``BeatThisB200`` model
    runs as ONE call of the CUDA path for every chunk_size up to its max_chunk_size (1500 unless loaded with more),
    border_size with 0 <= 2 * border_size < chunk_size and overlap_mode (all chunks batched, chunking and stitching
    inside the kernels; other values raise ``ValueError``); any other model goes chunk by chunk through the functions
    above.  With border_size 0 and chunk_size >= the piece's length the piece runs as one sequence."""
    if isinstance(model, BeatThisB200):
        chunking = engine_chunking(chunk_size, border_size, overlap_mode, model.max_chunk_size)
        spect = torch.as_tensor(spect, dtype=torch.float32, device=model.device).contiguous()
        beat, down = model.engine.spect2frames_cat(spect, [0, spect.shape[0]], chunking)
        return {"beat": beat, "downbeat": down}
    chunks, starts = split_piece(spect, chunk_size, border_size=border_size, avoid_short_end=True)
    preds = []
    for chunk in chunks:
        out = model(chunk.unsqueeze(0))
        preds.append({"beat": out["beat"][0], "downbeat": out["downbeat"][0]})
    beat, down = aggregate_prediction(preds, starts, spect.shape[0], chunk_size, border_size, overlap_mode, spect.device)
    return {"beat": beat, "downbeat": down}


class Spect2Frames:
    """Framewise beat / downbeat logits from a spectrogram (reference inference.py:233-257)."""

    def __init__(self, checkpoint_path="final0", device="cuda", float16=False, max_chunk_size=BT_CHUNK):
        """max_chunk_size: the longest chunk_size spects2frames / frames_batch take (load_model)."""
        super().__init__()
        self.device = torch.device(device)
        self.float16 = float16
        self.model = load_model(checkpoint_path, self.device, float16, max_chunk_size=max_chunk_size)
        self.device = self.model.device

    def spect2frames(self, spect):
        spect = torch.as_tensor(spect, dtype=torch.float32, device=self.device).contiguous()
        if spect.ndim != 2 or spect.shape[1] != 128:
            raise ValueError(f"Expected a (time, 128) spectrogram, got shape {tuple(spect.shape)}")
        beat, down = self.model.engine.spect2frames_cat(spect, [0, spect.shape[0]])
        return beat, down

    def spects2frames(self, spects, chunk_size: int = 1500, border_size: int = 6, overlap_mode: str = "keep_first"):
        """Batched variant: list of [T_i,128] tensors -> list of (beat, downbeat), every piece cut and stitched as
        split_predict_aggregate(spect, chunk_size, border_size, overlap_mode, model) does, all in one call."""
        chunking = engine_chunking(chunk_size, border_size, overlap_mode, self.model.max_chunk_size)
        spects = [torch.as_tensor(s, dtype=torch.float32, device=self.device) for s in spects]
        fo = _lib.offsets(s.shape[0] for s in spects)
        beat, down = self.model.engine.spect2frames_cat(torch.cat(spects).contiguous(), fo, chunking)
        return [(beat[fo[i] : fo[i + 1]], down[fo[i] : fo[i + 1]]) for i in range(len(spects))]

    def __call__(self, spect):
        return self.spect2frames(spect)


def _soxr_resample(signal, sr):
    """The reference's own host resampler (inference.py:274-275), when the package is installed."""
    try:
        import soxr
    except ImportError as e:
        raise RuntimeError("resampler='soxr' needs the `soxr` package; the default resampler='device' does not") from e
    return soxr.resample(signal, in_rate=sr, out_rate=22050)


class Audio2Frames(Spect2Frames):
    """Framewise logits from an audio signal (reference inference.py:260-281).

    Audio that is not at 22.05 kHz is resampled on the device (`resampler="device"`, a Kaiser-windowed-sinc
    polyphase FIR designed to soxr-HQ-like targets, see preprocessing.resample_filter_bank) or, with
    `resampler="soxr"`, by the reference's own host library when it is installed."""

    _want = "frames"

    def __init__(self, checkpoint_path="final0", device="cuda", float16=False, resampler="device",
                 max_chunk_size=BT_CHUNK):
        super().__init__(checkpoint_path, device, float16, max_chunk_size)
        self._init_front(resampler)

    def _init_front(self, resampler="device"):
        if resampler not in ("device", "soxr"):
            raise ValueError("resampler must be 'device' or 'soxr'")
        self.resampler = resampler
        self.spect = LogMelSpect(device=self.device, _engine=self.model.engine)
        self._pipe = None

    @classmethod
    def from_model(cls, model: BeatThisB200, **kw):
        """Wrap an already loaded model (e.g. one whose weights arrived by broadcast, distributed.py)."""
        self = cls.__new__(cls)
        self.model, self.device, self.float16 = model, model.device, model.float16
        self._init_front(kw.pop("resampler", "device"))
        self._init_post(**kw)
        return self

    def _init_post(self):
        pass

    @property
    def pipeline(self) -> BeatPipeline:
        if self._pipe is None:
            self._pipe = BeatPipeline(self.model.engine)
        return self._pipe

    # ---- one clip (the reference's call signatures) ---------------------------------------------------
    def _prepare(self, signals, sr):
        arrays = [as_signal_array(s) for s in signals]
        if int(sr) != 22050 and self.resampler == "soxr":  # the reference's order: mono mix, then soxr (inference.py:270-275)
            arrays = [np.ascontiguousarray(_soxr_resample(a if a.ndim == 1 else a.mean(1), sr)) for a in arrays]
            sr = 22050
        return arrays, int(sr)

    def signal2spect(self, signal, sr):
        arrays, sr = self._prepare([signal], sr)
        n = arrays[0].shape[0]
        host = torch.empty(max(n, 1), dtype=torch.float32, pin_memory=True)
        so = self.pipeline.stage_signals(arrays, host)
        audio = host[:n].to(self.device)
        if sr != 22050:
            audio, so = self.model.engine.resample_cat(audio, so, sr)
        spect, _ = self.model.engine.logmel_cat(audio, so)
        return spect

    def __call__(self, signal, sr):
        (beat, down), = Audio2Frames.batch(self, [signal], sr)
        return beat, down

    # ---- many clips ---------------------------------------------------------------------------------------
    def _run_groups(self, arrays, sr, want, chunking=DEFAULT_CHUNKING):
        """Generator over groups: (first index, last index + 1, pipeline result)."""
        pipe = self.pipeline
        groups = _plan_groups([a.shape[0] for a in arrays], sr, chunking)
        try:
            results = pipe.run(len(groups),
                               lambda g: pipe.submit_signals(arrays[groups[g][0] : groups[g][1]], sr, want, chunking))
            for (lo, hi), res in zip(groups, results):
                yield lo, hi, res
        finally:
            pipe.drain()

    def batch(self, signals, sr=22050):
        """list of signals (1-D or (time, channels) arrays, `sr` Hz) -> list of (beat_logits, downbeat_logits) device
        tensors; staging, copies and kernels of consecutive groups of clips overlap."""
        return self._frames_batch(signals, sr)

    def _frames_batch(self, signals, sr, chunking=DEFAULT_CHUNKING):
        """batch() with the `chunking` argument of Engine.audio2frames_cat."""
        arrays, sr = self._prepare(signals, sr)
        out = [None] * len(arrays)
        for lo, hi, (beat, down, fo) in self._run_groups(arrays, sr, "frames", chunking):
            for i in range(lo, hi):
                out[i] = (beat[fo[i - lo] : fo[i - lo + 1]], down[fo[i - lo] : fo[i - lo + 1]])
        return out

    def frames_from_device(self, audio: torch.Tensor, sample_offsets):
        """Audio already on the device (flat mono fp32 tensor at 22.05 kHz + offsets)."""
        return self.model.engine.audio2frames_cat(audio, list(sample_offsets))


class Audio2Beats(Audio2Frames):
    """Beat / downbeat positions in seconds from an audio signal (reference
    inference.py:284-303)."""

    def __init__(self, checkpoint_path="final0", device="cuda", float16=False, dbn=False, resampler="device",
                 dbn_impl="auto", max_chunk_size=BT_CHUNK):
        super().__init__(checkpoint_path, device, float16, resampler, max_chunk_size)
        self._init_post(dbn, dbn_impl)

    def _init_post(self, dbn=False, dbn_impl="auto"):
        """dbn_impl (with dbn=True): "auto" (madmom if installed, else the host C++ tracker), "madmom", "native" (the
        host C++ tracker) or "device" (the same tracker on the GPU, see Postprocessor)."""
        self.frames2beats = Postprocessor(type="dbn" if dbn else "minimal", engine=self.model.engine, dbn_impl=dbn_impl)

    def __call__(self, signal, sr):
        return Audio2Beats.batch(self, [signal], sr)[0]

    def _finish(self, res):
        """pipeline result of one group -> list of (beat_times, downbeat_times)."""
        if self.frames2beats.type == "minimal" or self.frames2beats.on_device:
            return res
        import time

        beat_h, down_h, fo = res
        t0 = time.perf_counter()
        out = self.frames2beats.batch_host(beat_h, down_h, fo)
        st = self.pipeline.stats
        st["post_s"] = st.get("post_s", 0.0) + time.perf_counter() - t0
        return out

    @property
    def pipeline(self) -> BeatPipeline:
        pipe = super().pipeline
        if self.frames2beats.on_device:
            pipe.dbn_params = self.frames2beats.dbn_params
        return pipe

    @property
    def _want_beats(self):
        if self.frames2beats.type == "minimal":
            return "beats"
        return "dbn_device" if self.frames2beats.on_device else "logits_host"

    def batch(self, signals, sr=22050):
        """list of signals -> list of (beat_times, downbeat_times) numpy float64 arrays.  With the host DBN, the host
        Viterbi of group g runs while the GPU works on group g+1; the device DBN runs on the compute stream after the
        forward pass of its group, like the peak picker."""
        arrays, sr = self._prepare(signals, sr)
        out = [None] * len(arrays)
        if self.frames2beats.type == "minimal" or self.frames2beats.on_device:
            for lo, hi, res in self._run_groups(arrays, sr, self._want_beats):
                out[lo:hi] = res
            return out
        # DBN: the host Viterbi of a group runs on a worker thread (numpy and the C++ tracker release the GIL), so the
        # calling thread is free to stage and enqueue the next groups
        from concurrent.futures import ThreadPoolExecutor

        with ThreadPoolExecutor(max_workers=1) as post:
            pending = [(lo, hi, post.submit(self._finish, res)) for lo, hi, res in self._run_groups(arrays, sr, "logits_host")]
            for lo, hi, fut in pending:
                out[lo:hi] = fut.result()
        return out


class File2Beats(Audio2Beats):
    def __call__(self, audio_path):
        signal, sr = load_audio(audio_path)
        return super().__call__(signal, sr)

    def batch(self, audio_paths, on_error: str = "raise"):
        """Many files per call.  WAV files are read, mixed to mono and cast by the native host threads straight into
        the pinned staging ring (no numpy round trip); FLAC files (with a known length) are staged as frame bytes and
        decoded and mixed on the device (bt_flac_decode), and so are MP3 files (bt_mp3_decode) and Ogg Vorbis files
        (bt_vorbis_decode); other containers go through load_audio.  Files of equal container and sample rate share
        groups.  on_error: "raise", or "skip" (a file that cannot be loaded or processed yields None instead of
        aborting the call -- the behaviour of the reference's per-file loop, cli.py:185-190); a FLAC, MP3 or Ogg Vorbis
        file with a malformed frame or packet raises RuntimeError naming it, or yields None."""
        if on_error not in ("raise", "skip"):
            raise ValueError("on_error must be 'raise' or 'skip'")
        paths = [str(p) for p in audio_paths]
        out = [None] * len(paths)
        kinds, bad = _native_groups(paths, raise_short=on_error == "raise")
        pipe = self.pipeline
        want = self._want_beats
        for (kind, sr), (idx, infos) in kinds.items():
            groups = _plan_groups([_n_samples(info) for info in infos], sr, DEFAULT_CHUNKING)

            def submit(g, idx=idx, infos=infos, groups=groups, sr=sr, kind=kind):
                lo, hi = groups[g]
                _SUBMIT[kind](pipe)([paths[i] for i in idx[lo:hi]], infos[lo:hi], sr, want)

            try:
                for (lo, hi), res in zip(groups, pipe.run(len(groups), submit)):
                    status = pipe.last_status
                    for j, (k, r) in enumerate(zip(idx[lo:hi], self._finish(res))):
                        if status is not None and status[j] != 0:
                            if on_error == "raise":
                                raise RuntimeError(f'Could not decode "{paths[k]}": malformed {_NAME[kind]}')
                            r = None
                        out[k] = r
            except Exception:
                pipe.drain()
                if on_error == "raise":
                    raise
                for i in idx:  # isolate the failure: one file at a time
                    if out[i] is None:
                        try:
                            out[i] = File2Beats.__call__(self, paths[i])
                        except Exception:
                            out[i] = None
        native = bad.union(*(idx for idx, _ in kinds.values()))
        rest = [i for i in range(len(paths)) if i not in native]
        loaded = {}
        for i in rest:
            try:
                loaded[i] = load_audio(paths[i])
            except Exception:
                if on_error == "raise":
                    raise
        for sr in sorted({s for _, s in loaded.values()}):
            idx = [i for i in loaded if loaded[i][1] == sr]
            try:
                res = Audio2Beats.batch(self, [loaded[i][0] for i in idx], sr)
            except Exception:
                if on_error == "raise":
                    raise
                res = []
                for i in idx:
                    try:
                        res.append(Audio2Beats.__call__(self, *loaded[i]))
                    except Exception:
                        res.append(None)
            for i, r in zip(idx, res):
                out[i] = r
        return out


    def frames_batch(self, audio_paths, chunk_size: int = 1500, border_size: int = 6, overlap_mode: str = "keep_first"):
        """Framewise (beat, downbeat) logits of many files as device tensors, through the groups and kernels of batch()
        up to the post-processor: frames2beats.batch_cat of them gives batch()'s beats.  Every piece is cut and
        stitched as split_predict_aggregate(spect, chunk_size, border_size, overlap_mode, model) does (chunk_size up to
        the model's max_chunk_size).  Errors raise."""
        chunking = engine_chunking(chunk_size, border_size, overlap_mode, self.model.max_chunk_size)
        paths = [str(p) for p in audio_paths]
        out = [None] * len(paths)
        kinds, _ = _native_groups(paths, raise_short=True)
        pipe = self.pipeline
        for (kind, sr), (idx, infos) in kinds.items():
            groups = _plan_groups([_n_samples(info) for info in infos], sr, chunking)

            def submit(g, idx=idx, infos=infos, groups=groups, sr=sr, kind=kind):
                lo, hi = groups[g]
                _SUBMIT[kind](pipe)([paths[i] for i in idx[lo:hi]], infos[lo:hi], sr, "frames", chunking)

            try:
                for (lo, hi), (beat, down, fo) in zip(groups, pipe.run(len(groups), submit)):
                    status = pipe.last_status
                    for j, k in enumerate(idx[lo:hi]):
                        if status is not None and status[j] != 0:
                            raise RuntimeError(f'Could not decode "{paths[k]}": malformed {_NAME[kind]}')
                        out[k] = (beat[fo[j] : fo[j + 1]], down[fo[j] : fo[j + 1]])
            finally:
                pipe.drain()
        native = set().union(*(idx for idx, _ in kinds.values()))
        loaded = {i: load_audio(paths[i]) for i in range(len(paths)) if i not in native}
        for sr in sorted({s for _, s in loaded.values()}):
            idx = [i for i in loaded if loaded[i][1] == sr]
            for i, r in zip(idx, Audio2Frames._frames_batch(self, [loaded[i][0] for i in idx], sr, chunking)):
                out[i] = r
        return out


def _n_samples(info) -> int:
    if isinstance(info, _lib.bt_wav_info):
        return int(info.frames)
    return int(info.n_samples) if isinstance(info, (_lib.bt_mp3_info, _lib.bt_vorbis_info)) else int(info.total_samples)


# the BeatPipeline route and the error-message name of each native container
_SUBMIT = {"wav": lambda p: p.submit_wavs, "flac": lambda p: p.submit_flacs, "mp3": lambda p: p.submit_mp3s,
           "vorbis": lambda p: p.submit_vorbis}
_NAME = {"flac": "FLAC frames", "mp3": "MP3 frames", "vorbis": "Ogg Vorbis packets"}


def _native_groups(paths, raise_short: bool):
    """The files the native readers take, by (container, sample rate) in sorted order: ({("wav" | "flac" | "mp3" | "vorbis", sr):
    ([index, ...], [probe info, ...])}, set of indices of files too short to run).  A clip needs more than 512 samples at 22.05 kHz (reflect padding
    of the STFT): a shorter one raises ValueError under raise_short, else it is marked bad (not retried through
    load_audio).  A FLAC file whose STREAMINFO leaves the length unknown goes to load_audio."""
    kinds, bad = {}, set()
    for i, (kind, info) in enumerate(_lib.probe_audio(paths)):
        if kind is None or (kind == "flac" and info.total_samples == 0):
            continue
        n = _n_samples(info)
        if n * 22050 // max(1, info.sample_rate) <= 512:
            if raise_short:
                raise ValueError(f'"{paths[i]}" is too short ({n} samples)')
            bad.add(i)
            continue
        idx, infos = kinds.setdefault((kind, int(info.sample_rate)), ([], []))
        idx.append(i)
        infos.append(info)
    return dict(sorted(kinds.items())), bad


class File2File(File2Beats):
    def __call__(self, audio_path, output_path):
        beats, downbeats = File2Beats.__call__(self, audio_path)
        save_beat_tsv(beats, downbeats, output_path)
