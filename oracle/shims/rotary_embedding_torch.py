"""Import shim so the UNMODIFIED reference can be imported in this
container, where `rotary_embedding_torch` (pinned 0.6.4 in the reference's
requirements.txt:6) is not installed and there is no network.

TEST INFRASTRUCTURE ONLY (used by oracle/make_golden.py). It restates the published
lucidrains rotary-embedding-torch 0.6.x behaviour for the one call the reference makes
(`rotate_queries_or_keys`, reference beat_this/model/roformer.py:121-123) with the
constructor the reference uses (`RotaryEmbedding(head_dim)`, beat_tracker.py:52):

  freqs  = 1 / theta^(arange(0, dim, 2)/dim), theta=10000       -> nn.Parameter [dim/2]
  angle  = repeat(pos[:,None] * freqs, '... n -> ... (n r)', r=2)  (adjacent pairs share a freq)
  out    = t*cos(angle) + rotate_half(t)*sin(angle),  rotate_half: (x0,x1)->(-x1,x0) on
           interleaved pairs;  pos = arange(seq_len) along dim -2; fp32 math.

PARITY UNPINNED for this third-party piece: the package itself is absent, so the
restatement cannot be executed against it here.
"""
import torch
from torch import nn


def _rotate_half(x):
    x = x.reshape(*x.shape[:-1], -1, 2)
    x1, x2 = x.unbind(dim=-1)
    return torch.stack((-x2, x1), dim=-1).reshape(*x.shape[:-2], -1)


class RotaryEmbedding(nn.Module):
    def __init__(self, dim, theta=10000):
        super().__init__()
        freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: (dim // 2)].float() / dim))
        self.freqs = nn.Parameter(freqs, requires_grad=False)

    def rotate_queries_or_keys(self, t, seq_dim=-2):
        n = t.shape[seq_dim]
        pos = torch.arange(n, device=t.device, dtype=torch.float32)
        ang = pos[:, None] * self.freqs.float()[None, :]
        ang = ang.repeat_interleave(2, dim=-1)  # [n, dim]
        with torch.autocast(t.device.type, enabled=False):
            tf = t.float()
            out = tf * ang.cos() + _rotate_half(tf) * ang.sin()
        return out.type(t.dtype)
