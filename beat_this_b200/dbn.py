"""Host dynamic-Bayesian-network post-processor: stand-in for madmom's ``DBNDownBeatTrackingProcessor`` as the
reference configures it (model/postprocessor.py:29-37: beats_per_bar=[3, 4], min_bpm=55, max_bpm=215, fps=50,
transition_lambda=100; madmom defaults observation_lambda=16, threshold=0.05, correct=True, num_tempi=60).

madmom is a third-party package that is not installable offline, so this is a RESTATEMENT of its published
algorithm (F. Krebs, S. Boeck, G. Widmer, "An Efficient State-Space Model for Joint Tempo and Meter Tracking",
ISMIR 2015; S. Boeck et al., "Joint Beat and Downbeat Tracking with Recurrent Neural Networks", ISMIR 2016):
parity with madmom is UNPINNED (madmom is not installable offline); tests check the Viterbi decoder against a brute-force
dense decoder and the tracker on synthetic activations.

State space: for every beat of the bar and every tempo (beat interval of i frames, i = round(60 fps / max_bpm) ..
round(60 fps / min_bpm)) the i positions inside that beat.  A state advances by one position per frame with
probability 1; at a beat boundary the interval may change with probability ~ exp(-lambda |i_new / i_old - 1|)
(normalised over the new intervals).  Observation: states in the first 1/observation_lambda of a beat emit the
beat (downbeat for the first beat of the bar) activation, all others (1 - sum(act)) / (observation_lambda - 1).
One HMM per bar length is decoded with Viterbi, the more probable path wins.
"""
from __future__ import annotations

import numpy as np

from . import _lib

_LIB = False


def _native():
    """The shared library if it is built (the decoder itself needs no GPU): whether to use it or the numpy twins."""
    global _LIB
    if _LIB is False:
        try:
            _LIB = _lib.load()
        except Exception:
            _LIB = None
    return _LIB


class _BarModel:
    """State space + transition + observation model for one bar length (vectorised for Viterbi)."""

    def __init__(self, beats, min_interval, max_interval, num_tempi, transition_lambda, observation_lambda):
        intervals = np.arange(np.round(min_interval), np.round(max_interval) + 1)
        if num_tempi is not None and num_tempi < len(intervals):  # log-spaced tempi, as few as requested
            n_log = num_tempi
            intervals = []
            while len(intervals) < num_tempi:
                intervals = np.unique(np.round(np.logspace(np.log2(min_interval), np.log2(max_interval), n_log, base=2)))
                n_log += 1
        self.intervals = np.asarray(intervals, dtype=np.int64)
        self.beats = int(beats)
        n_int = len(self.intervals)
        per_beat = int(self.intervals.sum())
        self.num_states = per_beat * self.beats
        first = np.cumsum(np.r_[0, self.intervals[:-1]])
        last = np.cumsum(self.intervals) - 1
        pos = np.concatenate([np.linspace(0, 1, i, endpoint=False) for i in self.intervals])
        self.positions = np.concatenate([pos + b for b in range(self.beats)])
        self.first_states = np.stack([first + b * per_beat for b in range(self.beats)])  # [beats, n_int]
        self.last_states = np.stack([last + b * per_beat for b in range(self.beats)])
        # tempo change at a beat boundary: from interval (rows) to interval (cols)
        ratio = self.intervals[None, :].astype(np.float64) / self.intervals[:, None].astype(np.float64)
        prob = np.exp(-transition_lambda * np.abs(ratio - 1.0))
        prob[prob <= np.spacing(1.0)] = 0.0
        prob /= prob.sum(1, keepdims=True)
        with np.errstate(divide="ignore"):
            self.log_tempo = np.log(prob)  # [from, to], -inf where impossible
        # what a state observes: 0 no beat, 1 beat, 2 downbeat
        border = 1.0 / observation_lambda
        self.pointers = np.zeros(self.num_states, dtype=np.int64)
        self.pointers[self.positions % 1 < border] = 1
        self.pointers[self.positions < border] = 2
        self.observation_lambda = observation_lambda
        self._is_first = np.zeros(self.num_states, dtype=bool)
        self._is_first[self.first_states.ravel()] = True
        self._n_int = n_int

    def log_densities(self, act):
        d = np.empty((len(act), 3))
        with np.errstate(divide="ignore", invalid="ignore"):
            d[:, 0] = np.log((1.0 - act.sum(1)) / (self.observation_lambda - 1))
            d[:, 1] = np.log(act[:, 0])
            d[:, 2] = np.log(act[:, 1])
        return d

    def viterbi(self, act):
        """Most probable state path and its log-probability (uniform initial distribution): the C++ decoder of the
        shared library (bt_dbn_viterbi, csrc/dbn_host.cpp -- madmom's is Cython), or `viterbi_numpy` when the
        library has not been built (both are host code and are tested against each other)."""
        if _native() is None:
            return self.viterbi_numpy(act)
        return _lib.dbn_viterbi(self.log_densities(act), self.beats, self.intervals, self.log_tempo, self.pointers)

    def viterbi_numpy(self, act):
        T, S = len(act), self.num_states
        dens = self.log_densities(act)
        v = np.full(S, -np.log(S))
        # back pointers are only ambiguous for the first states of a beat: which tempo we came from
        back = np.empty((T, self.beats, self._n_int), dtype=np.int16)
        not_first = ~self._is_first
        for t in range(T):
            new = np.empty(S)
            new[1:][not_first[1:]] = v[:-1][not_first[1:]]  # same tempo: position p-1 -> p
            for b in range(self.beats):
                cand = v[self.last_states[b - 1]][:, None] + self.log_tempo  # [from, to]
                arg = cand.argmax(0)
                back[t, b] = arg
                new[self.first_states[b]] = cand[arg, np.arange(self._n_int)]
            v = new + dens[t, self.pointers]
        state = int(v.argmax())
        logp = float(v[state])
        path = np.empty(T, dtype=np.int64)
        # which beat / tempo slot a first state belongs to
        slot = {int(s): (b, k) for b in range(self.beats) for k, s in enumerate(self.first_states[b])}
        for t in range(T - 1, -1, -1):
            path[t] = state
            if state in slot:
                b, k = slot[state]
                state = int(self.last_states[b - 1][back[t, b, k]])
            else:
                state -= 1
        return path, logp


class DBNDownBeatTracker:
    def __init__(self, beats_per_bar=(3, 4), min_bpm=55.0, max_bpm=215.0, num_tempi=60, transition_lambda=100,
                 observation_lambda=16, threshold=0.05, correct=True, fps=50):
        self.fps = float(fps)
        self.threshold = threshold
        self.correct = correct
        self.params = dict(beats_per_bar=[int(b) for b in np.atleast_1d(beats_per_bar)], min_bpm=float(min_bpm),
                           max_bpm=float(max_bpm), num_tempi=int(num_tempi or 0), transition_lambda=float(transition_lambda),
                           observation_lambda=float(observation_lambda))
        min_interval = 60.0 * fps / max_bpm
        max_interval = 60.0 * fps / min_bpm
        self.models = [_BarModel(b, min_interval, max_interval, num_tempi, transition_lambda, observation_lambda)
                       for b in np.atleast_1d(beats_per_bar)]

    @property
    def track_params(self) -> dict:
        """Every tracker parameter of bt_dbn_track / bt_dbn_track_device: `params` plus threshold, correct and fps."""
        return dict(self.params, threshold=float(self.threshold or 0.0), correct=bool(self.correct), fps=self.fps)

    def __call__(self, activations):
        """activations [T, 2] = (beat-but-not-downbeat, downbeat) probabilities -> [[time_s, beat_number], ...]."""
        if _native() is not None:
            return self.batch([activations])[0]
        return self.track_numpy(activations)

    def batch(self, activations_list, n_threads: int = 0):
        """Many pieces at once on the C++ tracker of the shared library (bt_dbn_track: model construction, Viterbi
        and peak correction in C++, one host thread per piece); `track_numpy` is its numpy twin."""
        if _native() is None:
            return [self.track_numpy(a) for a in activations_list]
        acts = [np.ascontiguousarray(a, dtype=np.float64).reshape(-1, 2) for a in activations_list]
        fo = _lib.offsets(len(a) for a in acts)
        cat = np.concatenate(acts) if acts else np.zeros((0, 2))
        return self.batch_cat(cat, fo, n_threads)

    def batch_cat(self, activations: np.ndarray, frame_offsets, n_threads: int = 0):
        """Same, for pieces that already sit back to back in one [total_frames, 2] float64 array."""
        fo = np.ascontiguousarray(frame_offsets, dtype=np.int64)
        n = len(fo) - 1
        if _native() is None:
            return [self.track_numpy(activations[fo[i] : fo[i + 1]]) for i in range(n)]
        times, numbers, counts = _lib.dbn_track(activations, fo, self.track_params, n_threads)
        out = []
        for i in range(n):
            a, k = int(fo[i]), int(counts[i])
            out.append(np.stack((times[a : a + k], numbers[a : a + k].astype(np.float64)), axis=1) if k else np.empty((0, 2)))
        return out

    def track_numpy(self, activations):
        act = np.asarray(activations, dtype=np.float64)
        first = 0
        if self.threshold:  # only decode between the first and the last frame that exceeds the threshold
            idx = np.nonzero(act >= self.threshold)[0]
            if idx.any():
                first = max(first, int(idx.min()))
                act = act[first : min(len(act), int(idx.max()) + 1)]
            else:
                act = act[:0]
        if not act.any():
            return np.empty((0, 2))
        results = [m.viterbi(act) for m in self.models]
        best = int(np.argmax([r[1] for r in results]))
        path, model = results[best][0], self.models[best]
        beat_numbers = model.positions[path].astype(int) + 1
        if self.correct:  # move every beat to the strongest activation inside its beat region
            beats = []
            in_beat = model.pointers[path] >= 1
            idx = np.nonzero(np.diff(in_beat.astype(int)))[0] + 1
            if in_beat[0]:
                idx = np.r_[0, idx]
            if in_beat[-1]:
                idx = np.r_[idx, in_beat.size]
            if idx.any():
                for left, right in idx.reshape((-1, 2)):
                    beats.append(int(np.argmax(act[left:right])) // 2 + left)
            beats = np.asarray(beats, dtype=int)
        else:
            beats = np.nonzero(np.diff(beat_numbers))[0] + 1
        return np.vstack(((beats + first) / self.fps, beat_numbers[beats])).T
