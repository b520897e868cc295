"""Float64 numpy restatement of the loss contract of include/beatthis.h (bt_beat_loss, bt_beat_loss_backward): what the
kernels in csrc/kernels_loss.cu and the reference's beat_this/model/loss.py compute, written out frame by frame; and
the cases of the reference's outputs the CPU and GPU loss tests share."""
import os

import numpy as np

from conftest import GOLDEN

MASKED_BCE, SHIFT_TOLERANT, SPLIT_SHIFT_TOLERANT = 0, 1, 2
FPS = 50


def softplus(z):
    return np.log1p(np.exp(-np.abs(z))) + np.maximum(z, 0.0)


def bce(x, y, p):
    """binary_cross_entropy_with_logits with pos_weight p, elementwise."""
    return (1 - y) * x + (1 + (p - 1) * y) * softplus(-x)


def bce_grad(x, y, p):
    return (p * y + 1 - y) / (1 + np.exp(-x)) - p * y


def _windows(a, r):
    """[len - 2r, 2r + 1] view: row c is a[c .. c + 2r] (centre c + r)."""
    return np.lib.stride_tricks.sliding_window_view(a, 2 * r + 1)


def row_terms(x, y, m, kind, t, p):
    """One row -> (terms over the scored frames, d(sum of terms)/dx over every frame)."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    m = np.ones_like(x) if m is None else np.asarray(m, np.float64)
    n = len(x)
    grad = np.zeros(n)
    if kind == MASKED_BCE:
        return m * bce(x, y, p), m * bce_grad(x, y, p)
    if n < 4 * t + 1:
        raise ValueError("row shorter than 4t + 1")
    c = np.arange(2 * t, n - 2 * t)
    wx = _windows(x, t)[c - t]  # x[c - t .. c + t]
    arg = np.argmax(wx, axis=1)  # first maximum
    xs = wx[np.arange(len(c)), arg]
    ys = _windows(y, 2 * t)[c - 2 * t].max(axis=1)
    yc, mc = y[c], m[c]
    if kind == SHIFT_TOLERANT:
        w = (yc + (1 - ys)) * mc
        terms, g = w * bce(xs, yc, p), w * bce_grad(xs, yc, p)
    elif kind == SPLIT_SHIFT_TOLERANT:
        terms = yc * mc * bce(xs, yc, p) + (1 - ys) * mc * bce(xs, ys, p)
        g = yc * mc * bce_grad(xs, yc, p) + (1 - ys) * mc * bce_grad(xs, ys, p)
    else:
        raise ValueError(f"unknown kind {kind}")
    np.add.at(grad, c - t + arg, g)  # ascending windows; the first maximum of each wins
    return terms, grad


def loss_rows(preds, targets, mask, offsets, kind, t, p, grad_mean=1.0):
    """Concatenated rows -> (per-row losses, mean over all rows' scored frames, d(mean)/d preds * grad_mean)."""
    rows, total, n_scored, grads = [], 0.0, 0, []
    for a, b in zip(offsets[:-1], offsets[1:]):
        terms, g = row_terms(preds[a:b], targets[a:b], None if mask is None else mask[a:b], kind, t, p)
        rows.append(terms.sum() / len(terms))
        total += terms.sum()
        n_scored += len(terms)
        grads.append(g)
    grad = np.concatenate(grads) * (grad_mean / n_scored) if grads else np.zeros(0)
    return np.asarray(rows), total / n_scored, grad


def framewise_truth(times, T, fps=FPS):
    """prepare_annotations(item, 0, T, fps)'s framewise truth (reference dataset.py:512-534): frames round(time * fps),
    half to even, kept in [0, T), set to 1."""
    f = np.round(np.asarray(times, np.float64) * fps).astype(np.int64)
    f = f[(f >= 0) & (f < T)]
    out = np.zeros(T, np.float32)
    out[f] = 1
    return out


# ---- the cases of the unmodified reference's outputs (tests/golden/loss.npz, oracle/make_golden_loss.py)
GOLD = np.load(os.path.join(GOLDEN, "loss.npz"))
CASES = range(int(GOLD["n"]))


def fixture_case(k):
    """(preds, targets, mask or None, row offsets, kind, tolerance, pos_weight, reference loss, reference grad), the
    mask broadcast to the predictions' shape and every array flattened into rows of T frames."""
    kind, t, pw, has_mask = GOLD[f"spec{k}"]
    x = GOLD[f"preds{k}"]
    m = np.broadcast_to(GOLD[f"mask{k}"], x.shape).astype(np.float32).ravel() if has_mask else None
    T = x.shape[-1]
    off = (np.arange(x.size // T + 1) * T).tolist()
    return (x.ravel(), GOLD[f"targets{k}"].ravel(), m, off, int(kind), int(t), float(pw), float(GOLD[f"loss{k}"]),
            GOLD[f"grad{k}"].ravel())


# torch's fp32 gradient form cancels when p y is close to (p y + 1 - y) sigmoid(x) (soft targets, p = 4.5): the fixture
# itself is then off by up to ~2e-6 of max |g| (1.7e-6 in case 61)
GRAD_TOL = 2e-6
