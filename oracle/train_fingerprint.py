"""Compact fingerprints of gradient tensors, shared by oracle/make_golden_train_grads.py and the tests that read its
fixture: per tensor the sum, the L2 norm and the dot products with three seeded standard-normal vectors (float64)."""
from __future__ import annotations

import numpy as np

N_DOTS = 3


def probes(n: int, index: int) -> np.ndarray:
    """[N_DOTS, n] float64 probe vectors of table entry `index`."""
    return np.random.default_rng(7000 + index).standard_normal((N_DOTS, n))


def fingerprint(g: np.ndarray, index: int) -> np.ndarray:
    """[sum, norm, dot_0, dot_1, dot_2] of gradient g (any shape) of table entry `index`, in float64."""
    v = np.asarray(g, dtype=np.float64).reshape(-1)
    return np.concatenate([[v.sum(), np.linalg.norm(v)], probes(v.size, index) @ v])


def bounds(ref: np.ndarray, n: int, index: int, rel: float) -> np.ndarray:
    """What |fingerprint(g) - ref| may be when ||g - g_ref|| <= rel ||g_ref||: by Cauchy-Schwarz, rel ||g_ref|| times
    sqrt(n) for the sum, 1 for the norm and the probe's norm for each dot product."""
    norm = ref[1]
    return rel * norm * np.concatenate([[np.sqrt(n), 1.0], np.linalg.norm(probes(n, index), axis=1)])
