"""A float64 restatement of bt_adamw_step (include/beatthis.h) and its elementwise error bound.

The scalars are derived as the library derives them (double, then rounded to fp32); the element ops are then taken
exactly in float64 from the same fp32 inputs.  The kernel rounds each op to fp32 (or fuses a multiply-add), so with
u = 2^-24 its results may differ from the restatement by at most, to first order:
  m: 2u (|g - m| + |m'|)                    (g - m, the lerp's product and sum; |1 - beta1|, |beta1| <= 1)
  v: 3u (beta2 v + (1 - beta2) g^2 + v')    (two products and a sum; every term >= 0)
  den = sqrt(v') / c2 + eps: (sqrt(v') / c2) (rel(v') / 2 + 2u) + u den
  p: u |p decay| + |s| (|q| (err(den) / den + 2u) + err(m) / den) + u |p'|    with q = m' / den, s the step size
The bound used is twice that, plus the smallest normal fp32 for results near zero."""
from __future__ import annotations

import numpy as np

from numerics import U, f32

TINY = float(np.finfo(np.float32).tiny)


def scalars(lr, beta1, beta2, eps, weight_decay, step) -> dict:
    """The fp32 scalars of one entry, derived in double as torch's foreach path does in Python."""
    bc1 = 1.0 - beta1 ** float(step)
    bc2 = 1.0 - beta2 ** float(step)
    return dict(decay=f32(1.0 - lr * weight_decay), decay_on=weight_decay != 0, w1=f32(1.0 - beta1),
                beta2=f32(beta2), w2=f32(1.0 - beta2), c2=f32(bc2 ** 0.5), eps=f32(eps), s=f32(lr / bc1 * -1.0))


def adamw(p, g, m, v, **hp):
    """(p', m', v') in float64 and their bounds (ep, em, ev) from fp32 arrays p, g, m, v and the hyperparameters
    lr, beta1, beta2, eps, weight_decay, step."""
    k = scalars(**hp)
    p, g, m, v = (np.asarray(a, dtype=np.float64) for a in (p, g, m, v))
    p1 = p * k["decay"] if k["decay_on"] else p
    d = g - m
    w1 = k["w1"]
    m1 = m + w1 * d if abs(w1) < 0.5 else g - d * float(np.float32(1.0 - np.float32(w1)))
    v1 = v * k["beta2"] + k["w2"] * g * g
    s = np.sqrt(v1) / k["c2"]
    den = s + k["eps"]
    q = m1 / den
    p2 = p1 + k["s"] * q
    em = 2 * U * (np.abs(d) + np.abs(m1))
    ev = 3 * U * (k["beta2"] * v + k["w2"] * g * g + v1)
    rel_v = np.divide(ev, v1, out=np.zeros_like(v1), where=v1 > 0)
    eden = s * (rel_v / 2 + 2 * U) + U * den
    eq = np.abs(q) * (eden / den + 2 * U) + em / den
    ep = (U * np.abs(p1) if k["decay_on"] else 0.0) + abs(k["s"]) * eq + U * np.abs(p2)
    return (p2, m1, v1), tuple(2 * e + TINY for e in (ep, em, ev))
