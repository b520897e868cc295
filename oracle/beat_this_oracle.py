"""CPU oracle: a functional (module-free) restatement of the reference Audio->Beats path.

TEST INFRASTRUCTURE ONLY.  Nothing in the product package (beat_this_b200/) imports this
file; it is used by tests/, __graft_entry__.smoke() and the cpu_baseline / reference legs
of bench.py as the *checker* and the timed CPU baseline.

Every function cites the reference file:line (relative to the reference's source tree) it restates.
Floating point (fp32 by default, like the reference's CPU path); plain torch CPU ops.

Pinning: oracle/make_golden.py imports the UNMODIFIED reference (through the import shims
in oracle/shims/) and checks this restatement against it on seeded inputs and synthetic
checkpoints, then writes tests/golden/*.npz from the reference's own outputs.  The
reference's own tests hold no golden vectors (tests/test_inference.py asserts types only).
Third-party arithmetic not in the reference's source tree and not installed here stays
"parity unpinned": rotary_embedding_torch 0.6.4 (RoPE; restated from its published
semantics, see oracle/shims/rotary_embedding_torch.py), soxr 0.3.7 (resampler; not
exercised: all inputs are 22.05 kHz), madmom (DBN; host, optional).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

SR = 22050
N_FFT = 1024
HOP = 441
N_MELS = 128
CHUNK = 1500
BORDER = 6
FPS = 50

# --------------------------------------------------------------------------------------
# log-mel  (reference beat_this/preprocessing.py:27-59; torchaudio functional.py:54-145,
# 425-587 and transforms/_transforms.py MelSpectrogram/MelScale)
# --------------------------------------------------------------------------------------


def _hz_to_mel_slaney(freq: float) -> float:
    # torchaudio functional.py:425-456
    f_sp = 200.0 / 3
    mels = freq / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = math.log(6.4) / 27.0
    if freq >= min_log_hz:
        mels = min_log_mel + math.log(freq / min_log_hz) / logstep
    return mels


def mel_filterbank(n_freqs=N_FFT // 2 + 1, f_min=30.0, f_max=11000.0, n_mels=N_MELS, sr=SR):
    """fb[n_freqs, n_mels] fp32, slaney scale, norm=None (torchaudio functional.py:459-587)."""
    all_freqs = torch.linspace(0, sr // 2, n_freqs)
    m_pts = torch.linspace(_hz_to_mel_slaney(f_min), _hz_to_mel_slaney(f_max), n_mels + 2)
    f_sp = 200.0 / 3
    freqs = f_sp * m_pts
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = math.log(6.4) / 27.0
    log_t = m_pts >= min_log_mel
    freqs[log_t] = min_log_hz * torch.exp(logstep * (m_pts[log_t] - min_log_mel))
    f_pts = freqs
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.max(torch.zeros(1), torch.min(down, up))


def logmel(x: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """x [L] -> [1 + L//441, 128].  preprocessing.py:56-59 -> torch.stft(center=True, reflect,
    periodic hann(1024), normalized=True) -> abs -> @fb -> log1p(1000*)."""
    x = x.to(dtype)
    xp = F.pad(x[None, None], (N_FFT // 2, N_FFT // 2), mode="reflect")[0, 0]
    frames = xp.unfold(0, N_FFT, HOP)  # [T, 1024]
    win = torch.hann_window(N_FFT, periodic=True, dtype=dtype)
    spec = torch.fft.rfft(frames * win, dim=-1)  # [T, 513]
    mag = spec.abs() * (1.0 / math.sqrt(N_FFT))
    mel = mag @ mel_filterbank().to(dtype)
    return torch.log1p(1000.0 * mel)


def signal2spect(signal: np.ndarray, sr: int) -> torch.Tensor:
    """inference.py:269-277 (mono mix in numpy f64, cast fp32, log-mel).  sr must be 22050
    (the soxr branch, inference.py:274-275, is third-party and not restated)."""
    signal = np.asarray(signal)
    if signal.ndim == 2:
        signal = signal.mean(1)
    elif signal.ndim != 1:
        raise ValueError(f"Expected 1D or 2D signal, got shape {signal.shape}")
    if sr != SR:
        raise NotImplementedError("oracle covers 22.05 kHz input only (soxr is third-party)")
    return logmel(torch.tensor(signal, dtype=torch.float32))


# --------------------------------------------------------------------------------------
# chunking / aggregation  (inference.py:90-185)
# --------------------------------------------------------------------------------------


def split_starts(T: int, chunk: int = CHUNK, border: int = BORDER) -> np.ndarray:
    """inference.py:119-125 with avoid_short_end=True."""
    starts = np.arange(-border, T - border, chunk - 2 * border)
    if T > chunk - 2 * border:
        starts[-1] = T - (chunk - border)
    return starts


def split_piece(spect: torch.Tensor, chunk: int = CHUNK, border: int = BORDER):
    """inference.py:100-135."""
    T = len(spect)
    starts = split_starts(T, chunk, border)
    chunks = []
    for s in starts:
        s = int(s)
        piece = spect[max(s, 0) : min(s + chunk, T)]
        left = max(0, -s)
        right = max(0, min(border, s + chunk - T))
        chunks.append(F.pad(piece, (0, 0, left, right)))
    return chunks, starts


def aggregate(pred_chunks, starts, T, chunk=CHUNK, border=BORDER):
    """inference.py:138-185, overlap_mode='keep_first'.  pred_chunks: list of (beat, downbeat)."""
    beat = torch.full((T,), -1000.0)
    down = torch.full((T,), -1000.0)
    for s, (b, d) in reversed(list(zip(starts, pred_chunks))):
        s = int(s)
        beat[s + border : s + chunk - border] = b[border:-border]
        down[s + border : s + chunk - border] = d[border:-border]
    return beat, down


# --------------------------------------------------------------------------------------
# model  (beat_this/model/beat_tracker.py, roformer.py)
# --------------------------------------------------------------------------------------


def rmsnorm(x, gamma):
    """roformer.py:22-32: F.normalize(x, dim=-1) * sqrt(dim) * gamma (eps 1e-12 on the norm)."""
    n = x.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    return x / n * math.sqrt(x.shape[-1]) * gamma


def rope(t, freqs):
    """rotary_embedding_torch 0.6.x rotate_queries_or_keys (roformer.py:121-123): interleaved
    pairs, angle = pos * freqs[i] for pair i, pos = 0..n-1 along dim -2."""
    n = t.shape[-2]
    pos = torch.arange(n, dtype=torch.float32)
    ang = (pos[:, None] * freqs[None, :].float()).repeat_interleave(2, dim=-1)
    t2 = t.reshape(*t.shape[:-1], -1, 2)
    rot = torch.stack((-t2[..., 1], t2[..., 0]), dim=-1).reshape(t.shape)
    return t * ang.cos() + rot * ang.sin()


def pre_attention(x, sd, p, heads):
    """roformer.py:114-125: the attention's inputs on x [S, n, dim]: roped q and k, v [S, h, n, d] and the gate
    logits [S, n, h] (before the sigmoid)."""
    xn = rmsnorm(x, sd[p + ".norm.gamma"])
    qkv = xn @ sd[p + ".to_qkv.weight"].T
    S, n, _ = x.shape
    qkv = qkv.view(S, n, 3, heads, -1).permute(2, 0, 3, 1, 4)  # (qkv) S h n d
    q, k, v = qkv[0], qkv[1], qkv[2]
    freqs = sd.get(p + ".rotary_embed.freqs")
    if freqs is None:
        d = q.shape[-1]
        freqs = 1.0 / (10000 ** (torch.arange(0, d, 2).float() / d))
    q, k = rope(q, freqs), rope(k, freqs)
    gates = xn @ sd[p + ".to_gates.weight"].T + sd[p + ".to_gates.bias"]  # [S, n, h]
    return q, k, v, gates


def attention(x, sd, p, heads, explicit=False):
    """roformer.py:114-132 (+ Attend :73-80).  x [S, n, dim] -> [S, n, dim] (no residual)."""
    q, k, v, gates = pre_attention(x, sd, p, heads)
    S, n, _ = x.shape
    if explicit:
        s = (q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
        out = torch.softmax(s, dim=-1) @ v
    else:
        out = F.scaled_dot_product_attention(q, k, v)
    out = out * gates.permute(0, 2, 1).unsqueeze(-1).sigmoid()
    out = out.permute(0, 2, 1, 3).reshape(S, n, -1)
    return out @ sd[p + ".to_out.0.weight"].T


def feedforward(x, sd, p):
    """roformer.py:38-61: RMSNorm -> Linear -> GELU(erf) -> Linear."""
    h = rmsnorm(x, sd[p + ".net.0.gamma"])
    h = F.gelu(h @ sd[p + ".net.1.weight"].T + sd[p + ".net.1.bias"])
    return h @ sd[p + ".net.4.weight"].T + sd[p + ".net.4.bias"]


def batchnorm(x, sd, p, dim):
    """eval-mode BatchNorm (beat_tracker.py:113,123,165), eps 1e-5, channel axis `dim`."""
    shape = [1] * x.ndim
    shape[dim] = -1
    scale = sd[p + ".weight"] / torch.sqrt(sd[p + ".running_var"] + 1e-5)
    shift = sd[p + ".bias"] - sd[p + ".running_mean"] * scale
    return x * scale.view(shape) + shift.view(shape)


def forward(sd: dict, x: torch.Tensor, taps: dict | None = None, explicit=False, sum_head=True):
    """BeatThis.forward (beat_tracker.py:188-192) on x [B, L, 128] -> (beat[B,L], downbeat[B,L]).
    `taps`, when given, collects intermediates in [B, F, L, C] (frontend) / [B, L, D] layout."""
    B, L, _ = x.shape

    def tap(name, val):
        if taps is not None:
            taps[name] = val.detach().clone()

    # stem: beat_tracker.py:108-126
    h = batchnorm(x.transpose(1, 2), sd, "frontend.stem.bn1d", 1)[:, None]  # [B,1,128,L]
    h = F.conv2d(h, sd["frontend.stem.conv2d.weight"], stride=(4, 1), padding=(0, 1))
    h = F.gelu(batchnorm(h, sd, "frontend.stem.bn2d", 1))  # [B,32,32,L]
    tap("stem", h.permute(0, 2, 3, 1))
    # frontend blocks: beat_tracker.py:128-168, PartialFTTransformer :290-301
    for i in range(3):
        p = f"frontend.blocks.{i}"
        if (p + ".partial.attnF.to_qkv.weight") in sd:
            C, Fq = h.shape[1], h.shape[2]
            heads = C // 32
            z = h.permute(0, 3, 2, 1).reshape(B * L, Fq, C)
            z = z + attention(z, sd, p + ".partial.attnF", heads, explicit)
            tap(f"b{i}.attnF", z.view(B, L, Fq, C).permute(0, 2, 1, 3))
            z = z + feedforward(z, sd, p + ".partial.ffF")
            tap(f"b{i}.ffF", z.view(B, L, Fq, C).permute(0, 2, 1, 3))
            z = z.view(B, L, Fq, C).permute(0, 2, 1, 3).reshape(B * Fq, L, C)
            z = z + attention(z, sd, p + ".partial.attnT", heads, explicit)
            tap(f"b{i}.attnT", z.view(B, Fq, L, C))
            z = z + feedforward(z, sd, p + ".partial.ffT")
            tap(f"b{i}.ffT", z.view(B, Fq, L, C))
            h = z.view(B, Fq, L, C).permute(0, 3, 1, 2)
        h = F.conv2d(h, sd[p + ".conv2d.weight"], stride=(2, 1), padding=(0, 1))
        h = F.gelu(batchnorm(h, sd, p + ".norm", 1))
        tap(f"b{i}.conv", h.permute(0, 2, 3, 1))
    # concat + linear: beat_tracker.py:76-77  ("b c f t -> b t (c f)")
    h = h.permute(0, 3, 1, 2).reshape(B, L, -1)
    h = h @ sd["frontend.linear.weight"].T + sd["frontend.linear.bias"]
    tap("frontend", h)
    # transformer: roformer.py:176-181
    D = h.shape[-1]
    n_layers = 1 + max(
        int(k.split(".")[2]) for k in sd if k.startswith("transformer_blocks.layers.")
    )
    for l in range(n_layers):
        p = f"transformer_blocks.layers.{l}"
        h = attention(h, sd, p + ".0", D // 32, explicit) + h
        tap(f"l{l}.attn", h)
        h = feedforward(h, sd, p + ".1") + h
        tap(f"l{l}.ff", h)
    h = rmsnorm(h, sd["transformer_blocks.norm.gamma"])
    # SumHead: beat_tracker.py:315-330 (beat = beat + downbeat in fp32); Head: beat_tracker.py:333-346
    o = h @ sd["task_heads.beat_downbeat_lin.weight"].T + sd["task_heads.beat_downbeat_lin.bias"]
    beat = o[..., 0] + o[..., 1] if sum_head else o[..., 0]
    down = o[..., 1]
    return beat, down


def strip_prefix(state_dict: dict) -> dict:
    """inference.py:83 / utils.py:105-111 ('model.' and '_orig_mod.' prefixes)."""
    return {k.replace("model.", "").replace("_orig_mod.", ""): v for k, v in state_dict.items()}


@torch.inference_mode()
def spect2frames(sd: dict, spect: torch.Tensor, batch_chunks: bool = True, sum_head: bool = True):
    """Spect2Frames.spect2frames (inference.py:244-254): chunk 1500 / border 6 / keep_first."""
    chunks, starts = split_piece(spect)
    if batch_chunks and len({len(c) for c in chunks}) == 1:
        b, d = forward(sd, torch.stack(chunks), sum_head=sum_head)
        preds = list(zip(b, d))
    else:
        preds = []
        for c in chunks:
            b, d = forward(sd, c[None], sum_head=sum_head)
            preds.append((b[0], d[0]))
    return aggregate(preds, starts, len(spect))


# --------------------------------------------------------------------------------------
# minimal postprocessor  (beat_this/model/postprocessor.py:85-136, 176-197)
# --------------------------------------------------------------------------------------


def deduplicate_peaks(peaks, width=1) -> np.ndarray:
    """postprocessor.py:176-197 (running-mean merge, python floats = float64)."""
    result = []
    it = iter(int(p) for p in peaks)
    try:
        p = next(it)
    except StopIteration:
        return np.array(result)
    c = 1
    for p2 in it:
        if p2 - p <= width:
            c += 1
            p += (p2 - p) / c
        else:
            result.append(p)
            p = p2
            c = 1
    result.append(p)
    return np.array(result)


def postp_minimal(beat: torch.Tensor, downbeat: torch.Tensor, fps: int = FPS):
    """postprocessor.py:85-136 for one un-padded piece: peak = (x == maxpool7(x)) & (x > 0)."""
    out = []
    for x in (beat, downbeat):
        x = x.float()[None]
        peaks = (x == F.max_pool1d(x, 7, 1, 3)) & (x > 0)
        frames = torch.nonzero(peaks[0]).numpy()[:, 0]
        out.append(deduplicate_peaks(frames, 1) / fps)
    beat_time, down_time = out
    if len(beat_time) > 0:
        for i, d in enumerate(down_time):
            down_time[i] = beat_time[np.argmin(np.abs(beat_time - d))]
    return beat_time, np.unique(down_time)


def audio2beats(sd: dict, signal: np.ndarray, sr: int = SR):
    """Audio2Beats.__call__ (inference.py:301-303) with the minimal postprocessor."""
    b, d = spect2frames(sd, signal2spect(signal, sr))
    return postp_minimal(b, d)


def resample_direct_terms(x, sr_in: int, sr_out: int, n):
    """The terms of the direct form at the output indices n: (samples [len(n), 2 half + 1], weights [len(n), 2 half + 1])
    with y[n] = sum(samples * weights, 1) -- the input samples j = floor(n M / L) - half .. floor(n M / L) + half
    (zeros outside the clip) and their weights s h(s (n M / L - j)), half = ceil(Z / s) + 1.  The phase n M / L - j
    is an exact integer plus (n M mod L) / L, so it is rounded once however long the clip is."""
    import math

    import numpy as np

    from beat_this_b200 import preprocessing as P

    x = np.asarray(x, dtype=np.float64)
    g = math.gcd(int(sr_in), int(sr_out))
    L, M = sr_out // g, sr_in // g
    s = min(1.0, L / M)
    half = int(math.ceil(P.RESAMPLE_ZERO_CROSSINGS / s)) + 1
    q, r = np.divmod(np.asarray(n, dtype=np.int64) * M, L)
    off = np.arange(-half, half + 1)
    j = q[:, None] + off[None, :]
    ok = (j >= 0) & (j < len(x))
    xv = np.where(ok, x[np.clip(j, 0, max(len(x) - 1, 0))] if len(x) else 0.0, 0.0)
    t = (r / L)[:, None] - off[None, :]
    return xv, s * P.resample_kernel(s * t)


def resample_direct(x, sr_in: int, sr_out: int = 22050):
    """Float64 direct-form evaluation of the resampler DEFINITION in beat_this_b200/preprocessing.py
    (stand-in for soxr.resample, reference inference.py:274-275; parity with soxr unpinned): every output
    sample sums the continuous Kaiser-windowed sinc over the input samples in its support -- no polyphase
    bank, so the bank construction and the kernel indexing are checked independently."""
    import math

    import numpy as np

    g = math.gcd(int(sr_in), int(sr_out))
    L, M = sr_out // g, sr_in // g
    n_out = (2 * len(x) * L + M) // (2 * M)
    y = np.zeros(n_out)
    for n0 in range(0, n_out, 4096):
        xv, w = resample_direct_terms(x, sr_in, sr_out, np.arange(n0, min(n_out, n0 + 4096)))
        y[n0 : n0 + len(xv)] = (xv * w).sum(1)
    return y
