"""Training batches of the reference's prepared data, assembled on the GPU: the reference's ``BeatTrackingDataset`` and
``BeatDataModule`` (beat_this/dataset/dataset.py, dataset/augment.py) without Lightning or worker processes.

* ``train_val_items`` / ``test_items`` / ``split_items``: the item lists of ``BeatDataModule.setup`` (dataset.py:305-446)
  from the split files and a checkpoint's ``datamodule_hyper_parameters``.
* ``Bundle``: memory-mapped float16 members of an uncompressed ``.npz`` (what ``prepare`` and the reference's
  preprocessing write), zero-copy views and frame counts read from the ``.npy`` headers.
* ``BeatTrackingDataset``: the reference's constructor, item loading, oversampling and positive weights; ``draw``
  takes one item's random draws in the reference's order and returns where its excerpt comes from.
* ``TrainingBatches``: shuffled batches with ``default_collate``'s keys, staged through pinned memory in one
  host->device copy and assembled by one ``bt_train_batch`` launch (gather, zero and permute masks, frame targets,
  padding mask).

The random draws are the reference's calls on a numpy legacy RNG (the ``np.random`` module unless a ``RandomState`` is
given): with ``np.random.seed(s)`` and the same index sequence, the batches equal the reference's items bitwise.
"""
from __future__ import annotations

import io
import json
import re
import zipfile
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch

from . import _lib
from .augment import precomputed_augmentation_filenames, shift_filename, stretch_annotations, stretch_filename
from .engine import Engine

N_BINS = 128
AUGMENTATIONS = ("mask", "pitch", "tempo")
MASK_KINDS = ("permute", "zero")
# the training datasets of Hung et al., "Modeling beats and downbeats with a time-frequency transformer" (dataset.py:357)
HUNG_DATA = re.compile("^(hainsworth/|ballroom/|hjdb/|beatles/|rwc/rwc_popular|simac/|smc/|harmonix/|).*$")


# ---- split files ---------------------------------------------------------------------------------------------------
def _read_split(path) -> list:
    """(piece, part) rows of a tab-separated split file, blank lines skipped; parts stay strings."""
    rows = []
    for line in Path(path).read_text().splitlines():
        if line.strip():
            piece, part = line.split("\t")[:2]
            rows.append((piece, part.strip()))
    return rows


def train_val_items(data_dir, test_dataset="gtzan", fold=None, hung_data=False, no_val=False, **_) -> tuple:
    """(train_items, val_items) as ``BeatDataModule.setup("fit")`` forms them (dataset.py:313-364): every dataset
    directory under DIR/annotations with the split file (``8-folds.split`` for a fold, else ``single.split``) except
    ``test_dataset``; fold f validates on part f and trains on the rest, the single split on "val" and "train";
    ``no_val`` adds the validation items to training, ``hung_data`` keeps only the training items of Hung et al.'s
    datasets.  Both lists sorted.  Other keyword arguments (a checkpoint's remaining datamodule hyper-parameters) are
    ignored."""
    ann = Path(data_dir) / "annotations"
    split_file = "8-folds.split" if fold is not None else "single.split"
    train, val = [], []
    for d in ann.iterdir():
        if not d.is_dir() or not (d / split_file).exists() or d.name == test_dataset:
            continue
        for piece, part in _read_split(d / split_file):
            if fold is not None:
                (val if part == str(fold) else train).append(f"{d.name}/{piece}")
            elif part in ("val", "train"):
                (val if part == "val" else train).append(f"{d.name}/{piece}")
    if no_val:
        train += val
    if hung_data:
        train = [item for item in train if HUNG_DATA.match(item)]
    return sorted(train), sorted(val)


def test_items(data_dir, test_dataset="gtzan", **_) -> list:
    """``BeatDataModule.setup("test")``'s items (dataset.py:404-411): every ``.beats`` file of the test dataset, sorted."""
    beats = Path(data_dir) / "annotations" / test_dataset / "annotations" / "beats"
    return sorted(f"{test_dataset}/{f.stem}" for f in beats.glob("*.beats"))


def split_items(data_dir, datasplit, hparams=None) -> list:
    """The items of one split ("train", "val" or "test") under the datamodule hyper-parameters `hparams` (a checkpoint's
    ``datamodule_hyper_parameters``; missing keys take BeatDataModule's defaults), as the reference's predict stage
    selects them (dataset.py:426-446)."""
    hp = dict(hparams or {})
    hp.pop("data_dir", None)  # a Lightning checkpoint records the directory it was trained from; data_dir wins
    if datasplit == "test":
        return test_items(data_dir, **hp)
    if datasplit not in ("train", "val"):
        raise ValueError(f"datasplit must be 'train', 'val' or 'test', got {datasplit!r}")
    train, val = train_val_items(data_dir, **hp)
    return train if datasplit == "train" else val


# ---- bundles ---------------------------------------------------------------------------------------------------------
def _check_spect(a, name):
    if a.dtype != np.float16:
        raise ValueError(f"{name}: spectrograms must be float16 (as prepare and the reference's preprocessing write "
                         f"them), got {a.dtype}")
    return a


class Bundle:
    """The uncompressed ``.npy`` members of an ``.npz`` file, memory-mapped: ``bundle[name]`` is a read-only view of
    member ``name`` (without ``.npy``), ``bundle.frames(name)`` its first dimension from the header alone.  Compressed
    members are not listed, as in the reference's MemmappedNpzFile.  Members must be float16 (ValueError)."""

    def __init__(self, path):
        self.path = str(path)
        with zipfile.ZipFile(path) as z:
            self._members = {i.filename[:-4]: (i.header_offset, i.file_size) for i in z.infolist()
                             if i.filename.endswith(".npy") and i.compress_type == zipfile.ZIP_STORED}
        self.mmap = np.memmap(path, mode="r")
        self._headers = {}

    @property
    def files(self) -> list:
        return list(self._members)

    def __contains__(self, name) -> bool:
        return name in self._members

    def _header(self, name):
        """(data offset, shape, fortran order, dtype) of a member."""
        if name not in self._headers:
            off, size = self._members[name]
            fn_len, extra_len = np.frombuffer(self.mmap[off + 26 : off + 30], "<u2")  # local file header
            start = off + 30 + int(fn_len) + int(extra_len)
            f = io.BytesIO(self.mmap[start : start + min(size, 1 << 16)].tobytes())
            version = np.lib.format.read_magic(f)
            read = np.lib.format.read_array_header_1_0 if version == (1, 0) else np.lib.format.read_array_header_2_0
            shape, fortran, dtype = read(f)
            if dtype != np.float16:
                raise ValueError(f"{self.path}: member {name} is {dtype}; spectrograms must be float16 (as prepare and "
                                 "the reference's preprocessing write them)")
            self._headers[name] = (start + f.tell(), shape, fortran, dtype)
        return self._headers[name]

    def frames(self, name) -> int:
        return int(self._header(name)[1][0])

    def __getitem__(self, name) -> np.ndarray:
        start, shape, fortran, dtype = self._header(name)
        n = int(np.prod(shape)) * dtype.itemsize
        return self.mmap[start : start + n].view(dtype).reshape(shape, order="F" if fortran else "C")


# ---- mask augmentation as a row map ---------------------------------------------------------------------------------
def mask_row_map(n, mask, fps, rng=np.random) -> np.ndarray:
    """``augment_mask_`` (augment.py:129-201) applied to the int32 row indices 0..n-1 of an excerpt of n frames instead
    of to its spectrogram, with the same draws in the same order: zeroed rows become -1, permuted rows move.  The result
    says where every row of the masked excerpt comes from, overlapping and repeated masks included.  As in the
    reference, a mask start never reaches the last possible position (randint(0, n - length)), a mask that is not
    shorter than the excerpt raises ValueError (numpy's randint), and a permute mask of `length` rows is cut into at most
    length + 1 parts (empty parts allowed)."""
    m = np.arange(n, dtype=np.int32)
    count = rng.randint(mask["min_count"], mask["max_count"] + 1)
    lo, hi = int(mask["min_len"] * fps), int(mask["max_len"] * fps)
    for _ in range(count):
        length = rng.randint(lo, hi + 1)
        start = rng.randint(0, n - length)
        seg = m[start : start + length]
        if mask["kind"] == "zero":
            seg[:] = -1
        elif mask["kind"] == "permute":
            parts = min(rng.randint(mask["min_parts"], mask["max_parts"] + 1), length + 1)
            bounds = [0, *np.sort(rng.choice(length, parts - 1, replace=False)).tolist(), length]
            seg[:] = np.concatenate([seg[bounds[k] : bounds[k + 1]] for k in rng.permutation(parts)])
        else:
            raise ValueError(f"Unsupported mask operation: {mask['kind']}")
    return m


# ---- the dataset -------------------------------------------------------------------------------------------------------
@dataclass
class Excerpt:
    """One item's draws: rows [start, start + n) of `spect` (the chosen variant, memory-mapped) through `row_map`
    (None: identity), sorted beat and downbeat frames in [0, n), and the rest of the reference's item."""
    spect: np.ndarray
    spect_path: str
    dataset: str
    start: int
    n: int
    row_map: np.ndarray | None
    beat_frames: np.ndarray
    downbeat_frames: np.ndarray
    downbeat_mask: bool
    truth_orig_beat: bytes
    truth_orig_downbeat: bytes


class BeatTrackingDataset:
    """The reference's ``BeatTrackingDataset`` (dataset.py:23-244) over the prepared layout of `data_folder`
    (annotations/<dataset>/..., audio/spectrograms/<dataset>.npz or <dataset>/<stem>/<variant>.npy).  Items are loaded
    in order; an item missing a variant ``augmentations`` needs, or with one column in a dataset whose info.json
    declares downbeats, is skipped with the reference's message; with ``length_based_oversampling_factor`` (and a
    train_length) each item repeats round(factor * frames / train_length) times, at least once.  Augmentation keys
    other than "mask", "pitch" and "tempo" are a ValueError, as in BeatDataModule."""

    def __init__(self, item_names, data_folder, spect_fps=50, train_length=1500, deterministic=False, augmentations={},
                 length_based_oversampling_factor=0):
        if not set(augmentations).issubset(AUGMENTATIONS):
            raise ValueError(f"Unsupported augmentations: {augmentations.keys()}")
        if "mask" in augmentations and augmentations["mask"].get("kind") not in MASK_KINDS:
            raise ValueError(f"Unsupported mask operation: {augmentations['mask'].get('kind')}")
        root = Path(data_folder)
        self.spect_basepath = root / "audio" / "spectrograms"
        self.annotation_basepath = root / "annotations"
        self.fps = spect_fps
        self.train_length = train_length
        self.deterministic = deterministic
        self.augmentations = augmentations
        self.length_based_oversampling_factor = length_based_oversampling_factor
        datasets = sorted({name.split("/", 1)[0] for name in item_names})
        self.dataset_info = {d: json.loads((self.annotation_basepath / d / "info.json").read_text()) for d in datasets}
        self.spects = {}
        for d in datasets:
            npz = self.spect_basepath / f"{d}.npz"
            if npz.exists():
                self.spects[d] = Bundle(npz)
        self._variants = precomputed_augmentation_filenames(augmentations)
        items = [it for it in map(self._load_item, item_names) if it is not None]
        if length_based_oversampling_factor and train_length is not None:
            over = []
            for it in items:
                k = int(np.round(length_based_oversampling_factor * self._frames(it["spect_path"]) / train_length))
                over += [it] * max(k, 1)
            print(f"Training set oversampled from {len(items)} to {len(over)} excerpts.")
            items = over
        self.items = items

    def _load_item(self, name):
        dataset, stem = name.split("/", 1)
        bundle = self.spects.get(dataset, ())
        for fn in self._variants:
            if f"{stem}/{fn[:-4]}" not in bundle and not (self.spect_basepath / name / fn).exists():
                print(f"Skipping {name} because not all necessary spectrograms are there.")
                return None
        ann = np.loadtxt(self.annotation_basepath / dataset / "annotations" / "beats" / f"{stem}.beats")
        if ann.ndim == 2:
            beat_time, beat_value = ann[:, 0], ann[:, 1].astype(int)
        else:
            beat_time, beat_value = ann, np.zeros_like(ann, dtype=np.int32)
        has_down = self.dataset_info[dataset]["has_downbeats"]
        if has_down and ann.ndim != 2:
            print(f"Skipping {name} because it has {ann.ndim} columns but downbeat is supposed to be there.")
            return None
        if dataset == "rwc":
            dataset = "rwc_" + stem.split("_", 2)[1]
        return {"spect_path": Path(name) / "track.npy", "beat_time": beat_time, "beat_value": beat_value,
                "downbeat_mask": has_down, "dataset": dataset}

    def _source(self, spect_path):
        """(bundle, member) or (None, loose .npy path) of a spect_path."""
        dataset, rest = str(spect_path).split("/", 1)
        b = self.spects.get(dataset)
        if b is not None and rest[:-4] in b:
            return b, rest[:-4]
        return None, self.spect_basepath / spect_path

    def _spect(self, spect_path) -> np.ndarray:
        b, key = self._source(spect_path)
        a = b[key] if b is not None else _check_spect(np.load(key, mmap_mode="r"), str(key))
        if a.ndim != 2 or a.shape[1] != N_BINS:
            raise ValueError(f"{spect_path}: expected [frames, {N_BINS}] spectrogram, got {a.shape}")
        return a

    def _frames(self, spect_path) -> int:
        b, key = self._source(spect_path)
        return b.frames(key) if b is not None else len(self._spect(spect_path))

    def __len__(self) -> int:
        return len(self.items)

    def get_frame_count(self, index) -> int:
        return self._frames(self.items[index]["spect_path"])

    def get_beat_count(self, index) -> int:
        return len(self.items[index]["beat_time"])

    def get_downbeat_count(self, index) -> int:
        return int((self.items[index]["beat_value"] == 1).sum())

    def positive_weights(self, widen_target_mask=3) -> dict:
        """``BeatDataModule.get_train_positive_weights`` (dataset.py:473-509) over this dataset's (oversampled) items:
        round((frames - positives * (2 w + 1)) / positives) for beats, and for downbeats over the items with
        downbeat annotations."""
        frames = frames_db = beats = downs = 0
        for it in self.items:
            f = self._frames(it["spect_path"])
            frames += f
            beats += len(it["beat_value"])
            if it["downbeat_mask"]:
                frames_db += f
                downs += int((it["beat_value"] == 1).sum())
        w = widen_target_mask * 2 + 1
        return {"beat": int(np.round((frames - beats * w) / beats)),
                "downbeat": int(np.round((frames_db - downs * w) / downs))}

    def _pitchtempo(self, item, rng):
        """augment_pitchtempo (augment.py:5-57): with both kinds one randint(2) picks pitch (0) or tempo."""
        aug = self.augmentations
        kind = ("pitch" if rng.randint(2) == 0 else "tempo") if "pitch" in aug and "tempo" in aug else \
            "pitch" if "pitch" in aug else "tempo" if "tempo" in aug else None
        if kind == "pitch":
            return shift_filename(item, rng.randint(aug["pitch"]["min"], aug["pitch"]["max"] + 1))
        if kind == "tempo":
            t = aug["tempo"]
            p = rng.choice(np.arange(t["min"], t["max"] + 1, t["stride"]))
            return stretch_annotations(stretch_filename(item, p), p)
        return item

    def draw(self, index, rng=None) -> Excerpt:
        """The random draws of ``__getitem__(index)`` (dataset.py:169-241) in the reference's order -- pitch or tempo
        variant, excerpt start, mask -- on `rng` (default: the np.random module).  Quirks kept:
        the start of a piece longer than train_length is randint(0, longer), which never picks the last start, or
        longer // 2 when deterministic; beat frames are round(time * fps) (numpy's half to even) of the times after a
        tempo variant divided them by 1 + p / 100, and frames outside [0, n) are dropped; truth_orig_* filters the
        times (not the frames) to [start / fps, end / fps) and shifts them by start / fps."""
        rng = np.random if rng is None else rng
        item = self._pitchtempo(self.items[index], rng)
        spect = self._spect(item["spect_path"])
        T = len(spect)
        longer = T - self.train_length if self.train_length is not None else 0
        if longer > 0:
            start = longer // 2 if self.deterministic else int(rng.randint(0, longer))
            end = start + self.train_length
        else:
            start, end = 0, T
        n = end - start
        row_map = mask_row_map(n, self.augmentations["mask"], self.fps, rng) if "mask" in self.augmentations else None
        # prepare_annotations (dataset.py:512-556)
        times, values = item["beat_time"], item["beat_value"]
        frames = (times * self.fps).round().astype(int) - start
        lo = np.searchsorted(frames, 0)
        hi = lo + np.searchsorted(frames[lo:], n)
        beat = frames[lo:hi]
        down = beat[values[lo:hi] == 1]
        lo_t, hi_t = start / self.fps, end / self.fps
        orig_down = times[item["beat_value"] == 1]
        return Excerpt(spect, str(item["spect_path"]), item["dataset"], start, n, row_map,
                       beat.astype(np.int32), down.astype(np.int32), bool(item["downbeat_mask"]),
                       (times[(times >= lo_t) & (times < hi_t)] - lo_t).tobytes(),
                       (orig_down[(orig_down >= lo_t) & (orig_down < hi_t)] - lo_t).tobytes())


# ---- batches ---------------------------------------------------------------------------------------------------------
train_batch = Engine.train_batch  # train_batch(engine, rows, ...), the name earlier versions offered


@dataclass
class _Staged:
    """One batch on its way: its draws, frame length L, window row offsets, and the pinned buffer (slot) its windows
    are being copied into by `copies`."""
    excerpts: list
    length: int
    rows: list
    slot: int
    copies: list


class TrainingBatches:
    """Batches of ``dataset`` as the reference's train loader (``DataLoader(shuffle=True, drop_last=True)`` with
    ``default_collate``) forms them, assembled on `device`:

    * order: ``torch.randperm`` of a generator seeded with `seed` (a random seed when None) per pass, as RandomSampler;
      without `shuffle`, 0..n-1.  ``len`` is the number of batches.
    * ``batch(indices)``: the batch of those items; their draws run in order on `rng` (default: the np.random module).
    * a batch is a dict: ``spect`` [B, L, 128] float16, ``truth_beat``, ``truth_downbeat``, ``padding_mask`` [B, L]
      bool, all on the device; ``downbeat_mask`` [B] bool and ``start_frame`` [B] int64 on the host; ``spect_path``
      and ``dataset`` lists of str; ``truth_orig_beat`` / ``truth_orig_downbeat`` lists of float64 ``bytes``.
      L is the dataset's train_length; a dataset with train_length None gives full pieces and needs batch_size 1.

    Each item's window (min(L, frames - start) rows of its memory-mapped variant) is copied by host threads into one
    pinned buffer, which goes to the device in one copy on a copy stream; one ``bt_train_batch`` launch on the current
    stream then gathers the rows through the mask row maps and writes the targets.  While a batch is consumed, the
    next one's draws are taken and its windows copied and uploaded (two pinned buffers and two device buffers
    alternate).

    ``shard`` (data-parallel training; None: every batch): a function of the batch index that says whether this rank
    assembles the batch.  Iteration then yields None for the batches it does not, after taking their items' draws all
    the same, in order, so that every rank's random state follows the one-process run's."""

    def __init__(self, dataset: BeatTrackingDataset, batch_size=8, shuffle=True, drop_last=True, seed=None,
                 device="cuda", rng=None, threads=8, shard=None):
        if batch_size < 1:
            raise ValueError("batch_size must be positive")
        if dataset.train_length is None and batch_size != 1:
            raise ValueError("a dataset of full pieces (train_length=None) needs batch_size=1")
        self.dataset, self.batch_size, self.shuffle, self.drop_last = dataset, batch_size, shuffle, drop_last
        self.rng, self.shard = rng, shard
        self.engine = Engine.shared(device)
        self.device = self.engine.device
        if seed is None:
            seed = int(torch.empty((), dtype=torch.int64).random_().item())
        self.generator = torch.Generator().manual_seed(seed)
        self._pool = ThreadPoolExecutor(max_workers=threads)
        self._copy_stream = torch.cuda.Stream(self.device)
        self._host = [None, None]  # pinned uint16 windows
        self._dev = [None, None]  # device copies of them
        self._uploaded = [None, None]  # event: the H2D copy out of host[k] is done
        self._consumed = [None, None]  # event: the kernel reading dev[k] is done
        self._next = 0

    def __len__(self) -> int:
        n = len(self.dataset)
        return n // self.batch_size if self.drop_last else -(-n // self.batch_size)

    def _order(self) -> list:
        n = len(self.dataset)
        return torch.randperm(n, generator=self.generator).tolist() if self.shuffle else list(range(n))

    def __iter__(self):
        order = self._order()
        chunks = [order[i : i + self.batch_size] for i in range(0, len(order), self.batch_size)]
        if self.drop_last and chunks and len(chunks[-1]) < self.batch_size:
            chunks.pop()
        own = self.shard or (lambda k: True)
        staged = self._stage(chunks[0], own(0)) if chunks else None
        for k in range(len(chunks)):
            out = None if staged is None else self._launch(staged)
            staged = self._stage(chunks[k + 1], own(k + 1)) if k + 1 < len(chunks) else None
            yield out

    def batch(self, indices) -> dict:
        return self._launch(self._stage(list(indices)))

    # -- staging
    def _stage(self, indices, own: bool = True) -> _Staged | None:
        ex = [self.dataset.draw(int(i), self.rng) for i in indices]
        if not own:  # drawn for the random state; another rank assembles the batch
            return None
        length = self.dataset.train_length if self.dataset.train_length is not None else ex[0].n
        rows = _lib.offsets(e.n for e in ex)
        slot = self._next
        self._next ^= 1
        if self._uploaded[slot] is not None:
            self._uploaded[slot].synchronize()  # the pinned buffer's previous upload has left it
        need = max(rows[-1], 1) * N_BINS
        if self._host[slot] is None or self._host[slot].numel() < need:
            self._host[slot] = torch.empty(need, dtype=torch.int16, pin_memory=True)
        host = self._host[slot].numpy().view(np.uint16)
        copies = [self._pool.submit(self._copy_window, host, a, e) for a, e in zip(rows[:-1], ex)]
        return _Staged(ex, length, rows, slot, copies)

    @staticmethod
    def _copy_window(host, row, e):
        dst = host[row * N_BINS : (row + e.n) * N_BINS].reshape(e.n, N_BINS)
        dst[:] = e.spect[e.start : e.start + e.n].view(np.uint16)

    def _launch(self, s: _Staged) -> dict:
        for f in s.copies:
            f.result()
        ex, rows, slot, L = s.excerpts, s.rows, s.slot, s.length
        B = len(ex)
        total = rows[-1]
        compute = torch.cuda.current_stream(self.device)
        need = max(total, 1) * N_BINS
        if self._dev[slot] is None or self._dev[slot].numel() < need:
            self._dev[slot] = torch.empty(need, dtype=torch.int16, device=self.device)
            self._copy_stream.wait_stream(compute)  # the new block may be one the current stream's pending work freed
        dev = self._dev[slot]
        with torch.cuda.stream(self._copy_stream):
            if self._consumed[slot] is not None:
                self._copy_stream.wait_event(self._consumed[slot])  # the last kernel reading dev[slot] is done
            dev[: total * N_BINS].copy_(self._host[slot][: total * N_BINS], non_blocking=True)
            self._uploaded[slot] = torch.cuda.Event()
            self._uploaded[slot].record(self._copy_stream)
        compute.wait_event(self._uploaded[slot])
        maps = None
        if any(e.row_map is not None for e in ex):
            maps = np.concatenate([e.row_map if e.row_map is not None else np.arange(e.n, dtype=np.int32) for e in ex])
        beat_off = _lib.offsets(len(e.beat_frames) for e in ex)
        down_off = _lib.offsets(len(e.downbeat_frames) for e in ex)
        beats = np.concatenate([e.beat_frames for e in ex] + [np.zeros(1, np.int32)])
        downs = np.concatenate([e.downbeat_frames for e in ex] + [np.zeros(1, np.int32)])
        spect = torch.empty((B, L, N_BINS), dtype=torch.float16, device=self.device)
        tb, td, pm = (torch.empty((B, L), dtype=torch.bool, device=self.device) for _ in range(3))
        self.engine.train_batch(dev, rows, L, maps, beats, beat_off, downs, down_off, spect, tb, td, pm)
        self._consumed[slot] = torch.cuda.Event()
        self._consumed[slot].record(compute)
        return {
            "spect": spect,
            "spect_path": [e.spect_path for e in ex],
            "dataset": [e.dataset for e in ex],
            "start_frame": torch.tensor([e.start for e in ex], dtype=torch.int64),
            "truth_beat": tb,
            "truth_downbeat": td,
            "downbeat_mask": torch.tensor([e.downbeat_mask for e in ex], dtype=torch.bool),
            "padding_mask": pm,
            "truth_orig_beat": [e.truth_orig_beat for e in ex],
            "truth_orig_downbeat": [e.truth_orig_downbeat for e in ex],
        }
