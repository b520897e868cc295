"""Beat and downbeat accuracy on annotated pieces: the evaluation half of the reference's
``launch_scripts/compute_paper_metrics.py`` without Lightning or mir_eval.

* ``beat_metrics`` scores any tracker's output: mir_eval.beat's F-measure, Cemgil and continuity at their defaults, for
  many (estimates, references) sets in one ``bt_beat_metrics`` launch (one H2D copy, one kernel, one D2H copy).
* ``evaluate`` runs a model over annotated pieces (audio files or stored spectrograms) through the batched inference
  path, restricts the truth to the piece (``prepare_annotations``, dataset.py:536-547) and scores beats and downbeats
  in one metric launch.  Its summary keys are the reference's (``_compute_metrics_target``, pl_module.py:131-160).
  With ``losses=True`` (``--losses``) it adds the test losses of the checkpoint's loss pair (``piece_losses``).
  Truth, losses and post-processing use the frame rate of the predictions: the checkpoint's ``fps`` hyper-parameter
  (50 when absent, as the reference's ``PLBeatThis``), or ``fps=`` / ``--fps``.
* ``python -m beat_this_b200.evaluate`` is the command line counterpart of compute_paper_metrics.py.

    python -m beat_this_b200.evaluate --models final0.ckpt --data data          # prepared dataset layout
    python -m beat_this_b200.evaluate --models final0.ckpt --audio songs/ --annotations beats/
    python -m beat_this_b200.evaluate --models fold*.ckpt --data data --datasplit val --aggregation-type k-fold
"""
from __future__ import annotations

import argparse
import json
import sys
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np
import torch

from . import _lib
from .engine import Engine

FIELDS = ("n_ref", "n_est", "matches", "P", "R", "F", "cemgil", "cemgil_max", "CMLc", "CMLt", "AMLc", "AMLt")
SUMMARY_KEYS = tuple(f"{k}_{t}" for t in ("beat", "downbeat") for k in ("F-measure", "Cemgil", "CMLt", "AMLt"))
LOSS_KEYS = ("test_loss_beat", "test_loss_downbeat", "test_loss")
FPS = 50

_engine = Engine.shared  # _engine(device), the name earlier versions offered


def check_times(times, what="beat times") -> np.ndarray:
    """1-D float64 array of finite, non-negative, non-decreasing times, or ValueError (mir_eval.beat.validate)."""
    t = np.asarray(times, dtype=np.float64)
    if t.ndim != 1:
        raise ValueError(f"{what} must be a 1-D array, got shape {t.shape}")
    if not np.all(np.isfinite(t)):
        raise ValueError(f"{what} must be finite")
    if t.size and t.min() < 0:
        raise ValueError(f"{what} must not be negative")
    if np.any(np.diff(t) < 0):
        raise ValueError(f"{what} must be in increasing order")
    return t


def load_beat_annotations(path):
    """A ``.beats`` file (one time per line, optionally a tab and the position in the bar, 1 = downbeat; reference
    dataset.py:117-123) -> (beats, downbeats, has_downbeats).  One column: no downbeats.  ValueError for times that
    are unsorted, negative or not finite."""
    text = Path(path).read_text()
    rows = [line.split() for line in text.splitlines() if line.strip()]
    ncol = {len(r) for r in rows}
    if len(ncol) > 1 or ncol - {1, 2}:
        raise ValueError(f"{path}: expected one or two columns on every line")
    a = np.array(rows, dtype=np.float64).reshape(len(rows), -1)
    beats = check_times(a[:, 0] if len(rows) else np.zeros(0), f"{path}: beat times")
    if a.shape[1] == 2:
        return beats, beats[a[:, 1].astype(int) == 1], True
    return beats, np.zeros(0), False


def beat_metrics(estimates, references, min_beat_time=5.0, f_window=0.07, cemgil_sigma=0.04, phase_threshold=0.175,
                 period_threshold=0.175, device="cuda") -> np.ndarray:
    """Score estimates[i] against references[i] (host arrays of times in seconds) for every i: a float64 array
    [n, 12] with the columns FIELDS (the contract of bt_beat_metrics, include/beatthis.h).  Inputs are checked with
    check_times first."""
    if len(estimates) != len(references):
        raise ValueError("need one reference array per estimate array")
    est = [check_times(e, f"estimates[{i}]") for i, e in enumerate(estimates)]
    ref = [check_times(r, f"references[{i}]") for i, r in enumerate(references)]
    n = len(est)
    if n == 0:
        return np.zeros((0, len(FIELDS)))
    eng = Engine.shared(device)
    offs = _lib.offsets(len(a) for a in est + ref)
    host = torch.empty(max(offs[-1], 1), dtype=torch.float64).pin_memory()
    if offs[-1]:
        host[: offs[-1]].numpy()[:] = np.concatenate(est + ref)
    packed = host.to(eng.device, non_blocking=True)  # estimates of every set, then references: one copy
    out = torch.empty((n, len(FIELDS)), dtype=torch.float64, device=eng.device)
    p = _lib.bt_beat_metric_params(min_beat_time, f_window, cemgil_sigma, phase_threshold, period_threshold)
    eng.beat_metrics(packed, offs, p, out)
    return out.cpu().numpy()


# ---- pieces and the model run ------------------------------------------------------------------------------------
@dataclass
class Piece:
    """One annotated piece: audio (a file path) or spect (a [T, 128] log-mel spectrogram), and its truth."""
    name: str
    beats: np.ndarray
    downbeats: np.ndarray
    has_downbeats: bool = True
    dataset: str = ""
    audio: str | None = None
    spect: np.ndarray | None = None


@dataclass
class EvalResult:
    pieces: list  # Piece, in input order
    metrics: dict  # key -> float64 array over pieces: SUMMARY_KEYS, then every FIELDS column as <field>_<beat|downbeat>
    predictions: list  # (beats, downbeats) per piece
    summary: dict = field(default_factory=dict)  # SUMMARY_KEYS -> mean over pieces

    def dataset_summary(self) -> dict:
        """SUMMARY_KEYS -> {dataset: mean over its pieces} (compute_paper_metrics.py's per-dataset table)."""
        ds = np.asarray([p.dataset for p in self.pieces])
        return {k: {d: float(np.mean(self.metrics[k][ds == d])) for d in np.unique(ds)} for k in SUMMARY_KEYS}


def horizon(times: np.ndarray, T: int, fps: float = FPS) -> np.ndarray:
    """Annotations inside a piece of T spectrogram frames at `fps` frames per second: times in [0, T / fps)
    (prepare_annotations with start_frame = 0, dataset.py:536-547)."""
    return times[(times >= 0) & (times < T / fps)]


def _frames_of_audio(runner, path) -> int:
    """Spectrogram length of an audio file as the inference path computes it (after resampling to 22.05 kHz)."""
    from . import preprocessing as P
    from .preprocessing import load_audio

    infos, ok = _lib.wav_probe([path])
    if ok[0]:
        n, sr = int(infos[0].frames), int(infos[0].sample_rate)
    else:
        sig, sr = load_audio(path)
        n = len(sig)
    if int(sr) != 22050:
        n = P.resampled_length(n, *P.resample_ratio(sr))
    return 1 + n // 441


def _predict(runner, pieces, group=64, logits=False, post=None):
    """(beats, downbeats) and spectrogram length of every piece through the batched inference path; with `logits`,
    also every piece's (beat, downbeat) logits on the device (audio then goes through the frames path and the
    runner's post-processor, which gives the same beats), else None.  post: the post-processor of the spectrogram
    pieces' logits (default: the runner's)."""
    post = runner.frames2beats if post is None else post
    preds, frames, frame_logits = [None] * len(pieces), [0] * len(pieces), [None] * len(pieces)
    audio = [i for i, p in enumerate(pieces) if p.audio is not None]
    if audio and logits:
        out = runner.frames_batch([pieces[i].audio for i in audio])
        fo = _lib.offsets(len(b) for b, _ in out)
        beat = torch.cat([b for b, _ in out]).contiguous()
        down = torch.cat([d for _, d in out]).contiguous()
        for i, r, o in zip(audio, runner.frames2beats.batch_cat(beat, down, fo), out):
            preds[i], frames[i], frame_logits[i] = r, len(o[0]), o
    elif audio:
        res = runner.batch([pieces[i].audio for i in audio])
        for i, r in zip(audio, res):
            preds[i] = r
            frames[i] = _frames_of_audio(runner, pieces[i].audio)
    spect = [i for i, p in enumerate(pieces) if p.audio is None]
    for g in range(0, len(spect), group):
        idx = spect[g : g + group]
        out = runner.spects2frames([np.asarray(pieces[i].spect, dtype=np.float32) for i in idx])
        fo = _lib.offsets(b.shape[0] for b, _ in out)
        beat = torch.cat([b for b, _ in out]).contiguous()
        down = torch.cat([d for _, d in out]).contiguous()
        for i, r, a, b, o in zip(idx, post.batch_cat(beat, down, fo), fo[:-1], fo[1:], out):
            preds[i], frames[i] = r, b - a
            if logits:
                frame_logits[i] = o
    return preds, frames, frame_logits


def framewise_truth(times, T: int, fps: float = FPS) -> np.ndarray:
    """prepare_annotations(item, 0, T, fps)'s framewise truth (reference dataset.py:512-534) as fp32: 1 at the frames
    np.round(time * fps) (half to even) inside [0, T), 0 elsewhere."""
    f = np.round(np.asarray(times, dtype=np.float64) * fps).astype(np.int64)
    out = np.zeros(T, dtype=np.float32)
    out[f[(f >= 0) & (f < T)]] = 1
    return out


def piece_losses(runner, pieces, logits, fps: float = FPS) -> dict:
    """The reference's test losses (test_step, pl_module.py:99-114,224-229) of every piece: the checkpoint's loss pair
    (loss_from_hparams) on the full-piece logits against the framewise truth at `fps`, the downbeat mask 0 for pieces
    without downbeat annotations.  All beat rows in one bt_beat_loss call, all downbeat rows in another."""
    from .loss import beat_loss_rows, loss_from_hparams, loss_spec

    dev = runner.model.device
    fo = _lib.offsets(len(b) for b, _ in logits)
    out = {}
    for t, (target, module) in enumerate(zip(("beat", "downbeat"), loss_from_hparams(runner.model.checkpoint_hparams))):
        x = torch.cat([lg[t] for lg in logits]).contiguous()
        truth = [framewise_truth(p.beats if t == 0 else p.downbeats, len(lg[t]), fps) for p, lg in zip(pieces, logits)]
        y = torch.from_numpy(np.concatenate(truth)).to(dev)
        keep = [1.0 if t == 0 or p.has_downbeats else 0.0 for p in pieces]
        m = torch.from_numpy(np.repeat(np.asarray(keep, np.float32), np.diff(fo))).to(dev)
        rows, _ = beat_loss_rows(x, y, m, fo, *loss_spec(module))
        out[f"test_loss_{target}"] = rows.cpu().numpy()
    out["test_loss"] = out["test_loss_beat"] + out["test_loss_downbeat"]
    return out


def make_runner(model, device="cuda", float16=True, dbn=False, dbn_impl="auto"):
    """A File2Beats for a checkpoint (path, short name or loaded dict) or an already loaded BeatThisB200."""
    from .inference import BeatThisB200, File2Beats, load_model

    if not isinstance(model, BeatThisB200):
        model = load_model(model, device, float16)
    return File2Beats.from_model(model, dbn=dbn, dbn_impl=dbn_impl)


def evaluate(model_or_runner, items=None, min_beat_time=5.0, device="cuda", float16=True, dbn=False, dbn_impl="auto",
             losses=False, fps=None, data=None, datasplit=None, datamodule_hparams=None):
    """Predict every Piece of `items` with the model (a File2Beats / Audio2Beats runner, a BeatThisB200 or a checkpoint;
    float16 / dbn / dbn_impl apply when a runner has to be built) and score it against its annotations: truth cut to
    [0, T / fps) for a spectrogram of T frames, beats and downbeats of all pieces in one bt_beat_metrics launch.
    fps: the frame rate of the model's predictions (None: the checkpoint's ``fps`` hyper-parameter, 50 when absent).
    The logits of stored spectrograms are post-processed at that rate; audio files go through the inference
    classes' 50 fps front end, so audio pieces with another fps are a ValueError.
    "Cemgil_<target>" is the reference's mean of mir_eval's (cemgil, cemgil_max) pair (pl_module.py:157-160); both
    parts stay available as cemgil_<target> and cemgil_max_<target>.  Pieces without downbeat annotations score 0 on
    the downbeat keys, as in the reference.  With `losses`, metrics also hold every piece's test_loss_beat,
    test_loss_downbeat and test_loss (piece_losses), and summary their means.
    datasplit ("train", "val" or "test"): instead of `items`, the full pieces of that split of the prepared dataset
    `data` (split_pieces) under `datamodule_hparams`, by default the checkpoint's datamodule_hyper_parameters when
    model_or_runner is a checkpoint (else BeatDataModule's defaults)."""
    from .postprocessor import Postprocessor, check_fps

    if datasplit is not None:
        if items is not None or data is None:
            raise ValueError("datasplit selects the pieces of `data`: give data and no items")
        if datamodule_hparams is None and isinstance(model_or_runner, (str, Path, dict)):
            from .inference import load_checkpoint

            ckpt = model_or_runner if isinstance(model_or_runner, dict) else load_checkpoint(model_or_runner, "cpu")
            datamodule_hparams = ckpt.get("datamodule_hyper_parameters", {})
        items = split_pieces(data, datasplit, datamodule_hparams)
    elif items is None:
        raise ValueError("evaluate needs items, or data and a datasplit")
    runner = model_or_runner
    if not hasattr(runner, "frames2beats"):
        runner = make_runner(runner, device, float16, dbn, dbn_impl)
    if fps is None:
        fps = runner.model.checkpoint_hparams.get("fps", FPS)
    check_fps(fps)
    pieces = list(items)
    post = runner.frames2beats
    if fps != post.fps:
        audio = [p.name for p in pieces if p.audio is not None]
        if audio:
            raise ValueError(f"{audio[0]}: audio is analysed at {post.fps} fps by the inference front end, not at the "
                             f"model's {fps}; evaluate stored spectrograms at that rate instead")
        post = Postprocessor(post.type, fps, engine=runner.model.engine, dbn_impl=post.dbn_impl)
    preds, frames, logits = _predict(runner, pieces, logits=losses, post=post)
    est, ref = [], []
    for target in (0, 1):
        for p, pr, T in zip(pieces, preds, frames):
            truth = check_times(p.beats if target == 0 else p.downbeats, f"{p.name}: truth")
            ref.append(horizon(truth, T, fps))
            est.append(pr[target])
    rows = beat_metrics(est, ref, min_beat_time=min_beat_time, device=runner.model.device)
    n = len(pieces)
    metrics = {}
    for t, target in enumerate(("beat", "downbeat")):
        part = rows[t * n : (t + 1) * n]
        col = {f: part[:, j] for j, f in enumerate(FIELDS)}
        metrics[f"F-measure_{target}"] = col["F"]
        metrics[f"Cemgil_{target}"] = (col["cemgil"] + col["cemgil_max"]) / 2
        metrics[f"CMLt_{target}"] = col["CMLt"]
        metrics[f"AMLt_{target}"] = col["AMLt"]
    for t, target in enumerate(("beat", "downbeat")):
        for j, f in enumerate(FIELDS):
            metrics[f"{f}_{target}"] = rows[t * n : (t + 1) * n, j]
    metrics = {k: metrics[k] for k in (*SUMMARY_KEYS, *[k for k in metrics if k not in SUMMARY_KEYS])}
    keys = SUMMARY_KEYS
    if losses and n:
        metrics.update(piece_losses(runner, pieces, logits, fps))
        keys = (*SUMMARY_KEYS, *LOSS_KEYS)
    summary = {k: float(np.mean(metrics[k])) if n else float("nan") for k in keys}
    return EvalResult(pieces, metrics, preds, summary)


# ---- data discovery ------------------------------------------------------------------------------------------------
def dataset_name(dataset: str, stem: str) -> str:
    """The reference's grouping name: rwc pieces are split by subsection (dataset.py:135-137)."""
    return "rwc_" + stem.split("_", 2)[1] if dataset == "rwc" else dataset


def discover_data(data_dir, items_file=None, names=None) -> list:
    """Pieces of the reference's prepared layout: DIR/annotations/<dataset>/annotations/beats/<stem>.beats with the
    spectrogram in DIR/audio/spectrograms/<dataset>.npz (key <stem>/track) or .../<dataset>/<stem>/track.npy
    (float16 as stored, cast to fp32).  <dataset>/info.json's has_downbeats is honoured when present: false drops the
    downbeat truth, true skips a piece whose file has one column (as the reference's dataset does).  items_file:
    lines "dataset/stem" restricting the set; names: the same as a list.  Bundles are read through
    dataset.Bundle (memory-mapped, float16 members only)."""
    from .dataset import Bundle

    root = Path(data_dir)
    ann = root / "annotations"
    if names is not None:
        names = list(names)
    elif items_file is not None:
        names = [ln.strip() for ln in Path(items_file).read_text().splitlines() if ln.strip()]
    else:
        names = [f"{d.name}/{f.stem}" for d in sorted(p for p in ann.iterdir() if p.is_dir())
                 for f in sorted((d / "annotations" / "beats").glob("*.beats"))]
    infos, bundles, pieces = {}, {}, []
    for name in names:
        dataset, stem = name.split("/", 1)
        if dataset not in infos:
            info = ann / dataset / "info.json"
            infos[dataset] = json.loads(info.read_text()) if info.exists() else {}
            npz = root / "audio" / "spectrograms" / f"{dataset}.npz"
            bundles[dataset] = Bundle(npz) if npz.exists() else None
        beats, downbeats, has_down = load_beat_annotations(ann / dataset / "annotations" / "beats" / f"{stem}.beats")
        declared = infos[dataset].get("has_downbeats")
        if declared and not has_down:
            print(f"Skipping {name} because it has 1 columns but downbeat is supposed to be there.")
            continue
        if declared is False:
            downbeats, has_down = np.zeros(0), False
        bundle = bundles[dataset]
        if bundle is not None and f"{stem}/track" in bundle:
            spect = bundle[f"{stem}/track"]
        else:
            spect = np.load(root / "audio" / "spectrograms" / dataset / stem / "track.npy")
        pieces.append(Piece(f"{name}/track.npy", beats, downbeats, has_down, dataset_name(dataset, stem),
                            spect=np.asarray(spect, dtype=np.float32)))
    return pieces


def split_pieces(data_dir, datasplit, datamodule_hparams=None) -> list:
    """discover_data's pieces for one split ("train", "val" or "test") of a prepared dataset under a checkpoint's
    datamodule hyper-parameters (test_dataset, fold, hung_data, no_val; dataset.split_items), always full pieces, as
    compute_paper_metrics.datamodule_setup selects them (:159-171)."""
    from .dataset import split_items

    return discover_data(data_dir, names=split_items(data_dir, datasplit, datamodule_hparams))


def discover_audio(paths, annotations_dir) -> list:
    """Audio files (directories are searched recursively) paired with annotations_dir/<stem>.beats; the dataset of a
    piece is the name of its directory."""
    files = []
    for p in map(Path, paths):
        files += sorted(f for f in p.rglob("*") if f.is_file() and f.suffix != ".beats") if p.is_dir() else [p]
    pieces = []
    for f in files:
        beats, downbeats, has_down = load_beat_annotations(Path(annotations_dir) / f"{f.stem}.beats")
        pieces.append(Piece(str(f), beats, downbeats, has_down, f.parent.name, audio=str(f)))
    return pieces


def write_predictions(fn, result: EvalResult) -> None:
    """{piece: [[time, beat number], ...]} as compute_paper_metrics.py's write_predictions (:228-235) writes it."""
    from .utils import infer_beat_numbers

    np.savez(fn, **{p.name: np.vstack([b, infer_beat_numbers(b, d)]).T for p, (b, d) in zip(result.pieces, result.predictions)})


# ---- command line ------------------------------------------------------------------------------------------------
def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m beat_this_b200.evaluate",
                                 description="Beat and downbeat accuracy of one or more checkpoints on annotated pieces.")
    add = ap.add_argument
    add("--models", nargs="+", required=True, help="checkpoint files or names")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="prepared dataset directory (annotations/ and audio/spectrograms/)")
    src.add_argument("--audio", nargs="+", help="audio files or directories (with --annotations)")
    add("--annotations", help="directory of <stem>.beats files for --audio")
    pick = ap.add_mutually_exclusive_group()
    pick.add_argument("--items", help="file of 'dataset/stem' lines restricting --data")
    pick.add_argument("--datasplit", choices=["train", "val", "test"], default=None,
                      help="score the pieces of this split of --data under each checkpoint's datamodule "
                           "hyper-parameters (default: every annotated piece)")
    add("--gpu", type=int, default=0)
    add("--eval-trim-beats", metavar="SECONDS", type=float, default=None,
        help="skip beats before this time (default: the checkpoint's eval_trim_beats, else 5)")
    add("--dbn", default=None, action=argparse.BooleanOptionalAction,
        help="DBN post-processing (default: the checkpoint's use_dbn)")
    add("--dbn-impl", default="auto", choices=["auto", "madmom", "native", "device"], help="DBN decoder [%(default)s]")
    add("--float16", default=True, action=argparse.BooleanOptionalAction,
        help="16-bit kernels, as the reference evaluates with precision='16-mixed' [on]")
    add("--aggregation-type", default="mean-std", choices=["mean-std", "k-fold"],
        help="summary over several models: mean and deviation of their summaries, or k-fold (each model on its own "
             "split, per-piece metrics concatenated) [%(default)s]")
    add("--dump-predictions", metavar="FILENAME", default=None, help="write the predictions to this .npz file")
    add("--losses", action="store_true",
        help="also report the test losses of the checkpoint's loss_type (test_loss_beat, test_loss_downbeat, test_loss)")
    add("--fps", type=float, default=None,
        help="frame rate of the model's predictions, for the truth and the post-processing (default: the checkpoint's "
             "fps, else 50)")
    return ap


def _print_single(result: EvalResult) -> None:
    print("Metrics")
    for k, v in result.summary.items():
        print(f"{k}: {v}")
    print("Dataset metrics")
    for k, v in result.dataset_summary().items():
        print(k)
        for d, value in v.items():
            print(f"{d}: {value}")
        print("------")


def _print_mean_std(summaries: list) -> None:
    print("Metrics")
    for k in summaries[0]:
        vals = [s[k] for s in summaries]
        print(f"{k}: {round(float(np.mean(vals)), 3)} +- {round(float(np.std(vals)), 3)}")


def _print_k_fold(result: EvalResult) -> None:
    print("Dataset metrics")
    for k, v in result.dataset_summary().items():
        print(k)
        for d, value in v.items():
            print(f"{d}: {round(value, 3)}")
        print("------")


def concat_results(results: list) -> EvalResult:
    """The k-fold aggregate of several results (compute_paper_metrics.py:127-137): pieces, per-piece metrics and
    predictions concatenated in order; ValueError when a piece appears twice."""
    pieces = [p for r in results for p in r.pieces]
    names = [p.name for p in pieces]
    if len(set(names)) != len(names):
        raise ValueError("There are repeated pieces in the folds")
    metrics = {k: np.concatenate([r.metrics[k] for r in results]) for k in results[0].metrics}
    summary = {k: float(np.mean(metrics[k])) if pieces else float("nan") for k in results[0].summary}
    return EvalResult(pieces, metrics, [p for r in results for p in r.predictions], summary)


def run(models, data=None, audio=None, annotations=None, items=None, gpu=0, eval_trim_beats=None, dbn=None,
        dbn_impl="auto", float16=True, aggregation_type="mean-std", dump_predictions=None, losses=False, fps=None,
        datasplit=None) -> int:
    from .inference import load_checkpoint

    if audio is not None and annotations is None:
        raise SystemExit("--audio needs --annotations")
    if datasplit is not None and (data is None or items is not None):
        raise SystemExit("--datasplit needs --data and excludes --items")
    if aggregation_type not in ("mean-std", "k-fold"):
        raise ValueError(f"Unknown aggregation type {aggregation_type}")
    k_fold = len(models) > 1 and aggregation_type == "k-fold"
    if len(models) > 1 and dump_predictions and not k_fold:
        print("cannot dump predictions when doing inference for multiple models")
        return 1
    pieces = None
    if datasplit is None:
        pieces = discover_data(data, items) if data is not None else discover_audio(audio, annotations)
    summaries, results = [], []
    for i, m in enumerate(models):
        if len(models) == 1:
            print("Single model prediction for", m)
        elif k_fold:
            print(f"Model {i + 1}/{len(models)}")
        ckpt = load_checkpoint(m, "cpu")
        if datasplit is not None and (pieces is None or k_fold):
            # k-fold: every checkpoint on its own split; otherwise the first checkpoint's split for all
            pieces = split_pieces(data, datasplit, ckpt.get("datamodule_hyper_parameters", {}))
        hp = ckpt.get("hyper_parameters", {})
        trim = eval_trim_beats if eval_trim_beats is not None else float(hp.get("eval_trim_beats", 5))
        use_dbn = dbn if dbn is not None else bool(hp.get("use_dbn", False))
        rate = fps if fps is not None else hp.get("fps", FPS)
        runner = make_runner(ckpt, f"cuda:{gpu}", float16, use_dbn, dbn_impl)
        result = evaluate(runner, pieces, min_beat_time=trim, losses=losses, fps=rate)
        summaries.append(result.summary)
        results.append(result)
        if len(models) == 1:
            _print_single(result)
            if dump_predictions:
                write_predictions(dump_predictions, result)
    if k_fold:
        result = concat_results(results)
        _print_k_fold(result)
        if dump_predictions:
            write_predictions(dump_predictions, result)
    elif len(models) > 1:
        _print_mean_std(summaries)
    return 0


def main(argv=None) -> int:
    return run(**vars(build_parser().parse_args(argv)))


if __name__ == "__main__":
    sys.exit(main())
