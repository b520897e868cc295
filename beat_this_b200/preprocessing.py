"""Audio loading and the log-mel frontend (mirror of reference beat_this/preprocessing.py).

``LogMelSpect`` keeps the reference's constructor and call signature (preprocessing.py:27-59).  At the
reference defaults it runs the model path's fused sm_90a kernel (frame -> Hann -> 1024-point FFT -> |.| ->
128-band slaney mel -> log1p(1000 x)) through ``bt_logmel``; any other analysis parameters run the general kernel
through ``bt_logmel_config`` on the tables ``MelTables`` builds.
``load_audio`` (preprocessing.py:6-24) walks the reference's decoder chain (torchaudio, soundfile, madmom -- whichever
is installed), then the native FLAC, MP3 and Ogg Vorbis decoders (``bt_flac_decode``, ``bt_mp3_decode``,
``bt_vorbis_decode`` on the current CUDA device) and then two dependency-free WAV readers; the batched File2Beats path
reads WAV, FLAC, MP3 and Ogg Vorbis files natively (``bt_stage_wav_files``, ``bt_flac_decode``, ``bt_mp3_decode``,
``bt_vorbis_decode``) and only falls back to this function for other containers.
"""
from __future__ import annotations

import math
import numbers
import wave

import numpy as np
import torch

SAMPLE_RATE = 22050
N_FFT = 1024
HOP = 441
N_MELS = 128
F_MIN = 30.0
F_MAX = 11000.0


def _decode_torchaudio(path, dtype):
    import torchaudio

    waveform, sr = torchaudio.load(str(path), channels_first=False)
    return np.asanyarray(waveform.squeeze().numpy(), dtype=dtype), int(sr)


def _decode_soundfile(path, dtype):
    import soundfile

    wav, sr = soundfile.read(str(path), dtype=dtype)
    return wav, int(sr)


def _decode_madmom(path, dtype):
    import madmom.io

    wav, sr = madmom.io.load_audio_file(str(path), dtype=dtype)
    return wav, int(sr)


def _decode_wav_scipy(path, dtype):
    from scipy.io import wavfile

    sr, data = wavfile.read(str(path))
    full_scale = {np.dtype(np.int16): 32768.0, np.dtype(np.int32): 2147483648.0}
    if data.dtype in full_scale:
        wav = data.astype(dtype) / full_scale[data.dtype]
    elif data.dtype == np.uint8:
        wav = (data.astype(dtype) - 128.0) / 128.0
    else:
        wav = data.astype(dtype)
    return wav, int(sr)


def _decode_wav_stdlib(path, dtype):
    with wave.open(str(path), "rb") as w:
        sr, nch, width = w.getframerate(), w.getnchannels(), w.getsampwidth()
        raw = np.frombuffer(w.readframes(w.getnframes()), dtype=np.uint8)
    if width == 1:
        wav = (raw.astype(dtype) - 128.0) / 128.0
    else:  # little-endian signed PCM of `width` bytes: assemble in int64, sign-extend
        b = raw.reshape(-1, width).astype(np.int64)
        v = sum(b[:, k] << (8 * k) for k in range(width))
        v = np.where(v >= 1 << (8 * width - 1), v - (1 << (8 * width)), v)
        wav = v.astype(dtype) / float(1 << (8 * width - 1))
    return (wav.reshape(-1, nch) if nch > 1 else wav), int(sr)


def _decode_flac_native(path, dtype):
    """A FLAC file decoded on the current CUDA device (bt_flac_decode): value / 2^(bits-1) in float64, [time] or
    [time, channels], as soundfile returns it."""
    import ctypes

    from . import _lib

    info = _lib.bt_flac_info()
    code = _lib.load().bt_flac_probe(str(path).encode(), ctypes.byref(info))
    if code != 0:
        raise ValueError("not a FLAC stream" if code == -6 else "cannot read the file")
    if not torch.cuda.is_available():
        raise RuntimeError("no CUDA device to decode FLAC on")
    from .engine import Engine

    fo, status_at, bo, total = _lib.flac_layout([info])
    host = np.zeros(max(total, 1), dtype=np.uint8)
    nf, ns, status = _lib.stage_flac_files([path], [info], host.ctypes.data, 1)
    if status[0] != 0:
        raise RuntimeError("malformed FLAC frames")
    n, ch = ns[0], info.channels
    dev = torch.device("cuda", torch.cuda.current_device())
    buf = torch.from_numpy(host).to(dev)
    out = torch.empty(max(n * ch, 1), dtype=torch.float64, device=dev)
    Engine.shared(dev).flac_decode(buf, _lib.flac_streams([info], nf, ns, [0]), _lib.BT_FLAC_CHANNELS_F64, out,
                                   status_at)
    if int(buf[status_at : status_at + 4].view(torch.int32).item()) != 0:
        raise RuntimeError("malformed FLAC frame")
    wav = out[: n * ch].cpu().numpy()
    return (wav.reshape(n, ch) if ch > 1 else wav).astype(dtype, copy=False), int(info.sample_rate)


def _decode_mp3_native(path, dtype):
    """An MPEG-1 Layer III file decoded on the current CUDA device (bt_mp3_decode): float64 samples, [time] or
    [time, channels], as torchaudio returns them cast to float64."""
    import ctypes

    from . import _lib

    info = _lib.bt_mp3_info()
    code = _lib.load().bt_mp3_probe(str(path).encode(), ctypes.byref(info))
    if code != 0:
        raise ValueError("not an MPEG-1 Layer III stream" if code == -6 else "cannot read the file")
    if not torch.cuda.is_available():
        raise RuntimeError("no CUDA device to decode MP3 on")
    from .engine import Engine

    fo, status_at, bo, total = _lib.mp3_layout([info])
    host = np.zeros(max(total, 1), dtype=np.uint8)
    nf, mb, status = _lib.stage_mp3_files([path], [info], host.ctypes.data, 1)
    if status[0] != 0:
        raise RuntimeError("malformed MP3 frames")
    n, ch = info.n_samples, info.channels
    dev = torch.device("cuda", torch.cuda.current_device())
    buf = torch.from_numpy(host).to(dev)
    out = torch.empty(max(n * ch, 1), dtype=torch.float64, device=dev)
    Engine.shared(dev).mp3_decode(buf, _lib.mp3_streams([info], nf, mb, [0]), _lib.BT_MP3_CHANNELS_F64, out, status_at)
    if int(buf[status_at : status_at + 4].view(torch.int32).item()) != 0:
        raise RuntimeError("malformed MP3 frames")
    wav = out[: n * ch].cpu().numpy()
    return (wav.reshape(n, ch) if ch > 1 else wav).astype(dtype, copy=False), int(info.sample_rate)


def _decode_vorbis_native(path, dtype):
    """An Ogg Vorbis file decoded on the current CUDA device (bt_vorbis_decode): float64 samples, [time] or
    [time, channels]."""
    import ctypes

    from . import _lib

    info = _lib.bt_vorbis_info()
    code = _lib.load().bt_vorbis_probe(str(path).encode(), ctypes.byref(info))
    if code != 0:
        raise ValueError("not an Ogg Vorbis stream" if code == -6 else "cannot read the file")
    if not torch.cuda.is_available():
        raise RuntimeError("no CUDA device to decode Ogg Vorbis on")
    from .engine import Engine

    fo, status_at, bo, total = _lib.vorbis_layout([info])
    host = np.zeros(max(total, 1), dtype=np.uint8)
    npk, pb, bs, status = _lib.stage_vorbis_files([path], [info], host.ctypes.data, 1)
    if status[0] != 0:
        raise RuntimeError("malformed Ogg Vorbis packets")
    n, ch = info.n_samples, info.channels
    dev = torch.device("cuda", torch.cuda.current_device())
    buf = torch.from_numpy(host).to(dev)
    out = torch.empty(max(n * ch, 1), dtype=torch.float64, device=dev)
    Engine.shared(dev).vorbis_decode(buf, _lib.vorbis_streams([info], npk, pb, bs, [0]), _lib.BT_VORBIS_CHANNELS_F64,
                                     out, status_at)
    if int(buf[status_at : status_at + 4].view(torch.int32).item()) != 0:
        raise RuntimeError("malformed Ogg Vorbis packets")
    wav = out[: n * ch].cpu().numpy()
    return (wav.reshape(n, ch) if ch > 1 else wav).astype(dtype, copy=False), int(info.sample_rate)


# tried in this order; the first three are the reference's chain (preprocessing.py:6-24), the rest need nothing beyond
# this package, scipy and the standard library and keep FLAC and WAV input working where none of those packages has a
# decoder
AUDIO_BACKENDS = (("torchaudio", _decode_torchaudio), ("soundfile", _decode_soundfile), ("madmom", _decode_madmom),
                  ("native FLAC", _decode_flac_native), ("native MP3", _decode_mp3_native),
                  ("native Ogg Vorbis", _decode_vorbis_native),
                  ("scipy.io.wavfile", _decode_wav_scipy),
                  ("wave", _decode_wav_stdlib))


def load_audio(path, dtype="float64"):
    """(waveform [time] or [time, channels] in [-1, 1), sample rate) like reference preprocessing.py:6-24: torchaudio,
    then soundfile, then madmom (each only if it is installed and can decode the file), then two WAV-only readers."""
    tried = []
    for name, decode in AUDIO_BACKENDS:
        try:
            return decode(path, dtype)
        except Exception as e:  # missing package, missing codec, unreadable file: next backend
            tried.append(f"{name}: {type(e).__name__}" + (f" ({e})" if name.startswith("native") else ""))
    raise RuntimeError(f'Could not load audio from "{path}". Without torchaudio, soundfile or madmom, FLAC, MP3 '
                       "(MPEG-1 Layer III) and Ogg Vorbis (all on a CUDA device) and WAV are the formats read. (" + "; ".join(tried)
                       + ")")


# ------------------------------------------------------------------------------------------
# constants of the fused log-mel kernel
# ------------------------------------------------------------------------------------------


def _hz_to_mel(freq: float, mel_scale: str = "slaney") -> float:
    if mel_scale == "htk":
        return 2595.0 * math.log10(1.0 + (freq / 700.0))
    f_sp = 200.0 / 3
    mels = freq / f_sp
    min_log_hz = 1000.0
    if freq >= min_log_hz:
        mels = min_log_hz / f_sp + math.log(freq / min_log_hz) / (math.log(6.4) / 27.0)
    return mels


def mel_filterbank(n_freqs=N_FFT // 2 + 1, f_min=F_MIN, f_max=F_MAX, n_mels=N_MELS, sample_rate=SAMPLE_RATE,
                   mel_scale="slaney"):
    """torchaudio.functional.melscale_fbanks(norm=None) restated with the same fp32 torch ops, so that the
    coefficients are bit-identical to what the reference's MelSpectrogram holds (reference preprocessing.py:43-53)
    for either mel scale, any sample rate (the grid tops out at the integer ``sample_rate // 2``) and any band count.
    ``ValueError`` for a mel_scale other than "slaney" / "htk", as torchaudio."""
    if mel_scale not in ("slaney", "htk"):
        raise ValueError('mel_scale should be one of "htk" or "slaney".')
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_pts = torch.linspace(_hz_to_mel(f_min, mel_scale), _hz_to_mel(f_max, mel_scale), n_mels + 2)
    if mel_scale == "htk":
        f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    else:
        f_sp = 200.0 / 3
        f_pts = f_sp * m_pts
        min_log_hz = 1000.0
        min_log_mel = min_log_hz / f_sp
        logstep = math.log(6.4) / 27.0
        log_t = m_pts >= min_log_mel
        f_pts[log_t] = min_log_hz * torch.exp(logstep * (m_pts[log_t] - min_log_mel))
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.max(torch.zeros(1), torch.min(down, up))  # [n_freqs, n_mels]


def filterbank_csr(fb: np.ndarray):
    """[n_freqs, n_mels] filterbank -> (start bin [n_mels], pointers [n_mels + 1], weights): band m is the run
    w[ptr[m]:ptr[m+1]] on the bins from start[m] on, from its first to its last non-zero bin (an all-zero band is
    an empty run at bin 0)."""
    starts, ptr, w = [], [0], []
    for m in range(fb.shape[1]):
        nz = np.nonzero(fb[:, m])[0]
        if len(nz) == 0:
            starts.append(0)
        else:
            lo, hi = int(nz[0]), int(nz[-1]) + 1
            starts.append(lo)
            w.extend(fb[lo:hi, m].tolist())
        ptr.append(len(w))
    return np.asarray(starts, np.int32), np.asarray(ptr, np.int32), np.asarray(w, np.float32)


def fft_twiddles(n_fft: int) -> np.ndarray:
    """e^{-2 pi i j / n_fft} for j < n_fft / 2 as interleaved (re, im) fp32, computed in float64."""
    k = np.arange(n_fft // 2, dtype=np.float64)
    tw = np.stack([np.cos(2 * np.pi * k / n_fft), -np.sin(2 * np.pi * k / n_fft)], axis=1)
    return tw.astype(np.float32).reshape(-1)


def mel_constants() -> dict:
    """Window, FFT twiddles and the filterbank in CSR form (each mel band is one contiguous
    run of FFT bins) as packed parameters ``mel.*``."""
    starts, ptr, w = filterbank_csr(mel_filterbank().numpy())  # [513, 128]
    return {
        "mel.window": torch.hann_window(N_FFT, periodic=True).numpy(),
        "mel.twiddle": fft_twiddles(N_FFT),
        "mel.fb_start": starts.astype(np.float32),
        "mel.fb_ptr": ptr.astype(np.float32),
        "mel.fb_w": w,
    }


MEL_N_FFT_RANGE = (64, 8192)
MEL_MAX_BANDS = 1024


def mel_norm_mode(normalized) -> int:
    """torchaudio's `normalized` (_get_spec_norms) as bt_mel_config.norm_mode: "frame_length" scales the STFT by
    n_fft^-1/2, True or "window" divides it by sqrt(sum window^2), False leaves it."""
    from ._lib import BT_MEL_NORM_FRAME_LENGTH, BT_MEL_NORM_NONE, BT_MEL_NORM_WINDOW

    if isinstance(normalized, str):
        if normalized not in ("frame_length", "window"):
            raise ValueError(f"Invalid normalized parameter: {normalized}")
        return BT_MEL_NORM_FRAME_LENGTH if normalized == "frame_length" else BT_MEL_NORM_WINDOW
    if isinstance(normalized, bool):
        return BT_MEL_NORM_WINDOW if normalized else BT_MEL_NORM_NONE
    raise TypeError("Input type not supported")


class MelTables:
    """Host-side constants of one bt_logmel_config analysis (include/beatthis.h): the config struct, the periodic
    Hann window, the FFT twiddles and the filterbank in CSR form.  ``to(device)`` gives the device copies the call
    takes.  Raises what the contract names for arguments outside it."""

    def __init__(self, sample_rate, n_fft, hop_length, f_min, f_max, n_mels, mel_scale, normalized, power,
                 log_multiplier):
        from ._lib import bt_mel_config

        norm_mode = mel_norm_mode(normalized)
        if mel_scale not in ("slaney", "htk"):
            raise ValueError('mel_scale should be one of "htk" or "slaney".')
        if power is None:
            raise NotImplementedError("complex output (power=None) is not implemented")
        lo, hi = MEL_N_FFT_RANGE
        n_fft_ok = isinstance(n_fft, numbers.Integral) and lo <= n_fft <= hi and n_fft & (n_fft - 1) == 0
        if not (n_fft_ok and isinstance(hop_length, numbers.Integral) and hop_length >= 1
                and isinstance(n_mels, numbers.Integral)
                and 1 <= n_mels <= MEL_MAX_BANDS and math.isfinite(power) and power > 0
                and math.isfinite(log_multiplier)):
            raise NotImplementedError(
                f"the log-mel kernels take a power-of-two n_fft in [{lo}, {hi}], hop_length >= 1, 1 <= n_mels <= "
                f"{MEL_MAX_BANDS}, a finite power > 0 and a finite log_multiplier (got n_fft={n_fft}, "
                f"hop_length={hop_length}, n_mels={n_mels}, power={power}, log_multiplier={log_multiplier})")
        f_max = f_max if f_max is not None else float(sample_rate // 2)
        if f_min > f_max:
            raise ValueError(f"Require f_min: {f_min} <= f_max: {f_max}")
        n_fft, hop_length, n_mels = int(n_fft), int(hop_length), int(n_mels)
        self.n_fft, self.hop_length, self.n_mels = n_fft, hop_length, n_mels
        self.config = bt_mel_config(n_fft, hop_length, n_mels, norm_mode, float(power), float(log_multiplier))
        self.fb = mel_filterbank(n_fft // 2 + 1, f_min, f_max, n_mels, sample_rate, mel_scale)
        self.fb_start, self.fb_ptr, self.fb_w = filterbank_csr(self.fb.numpy())
        self.window = torch.hann_window(n_fft, periodic=True)
        self.twiddle = fft_twiddles(n_fft)

    def to(self, device) -> dict:
        """Device tensors of the tables (fb_w holds at least one element, so that its pointer is never null)."""
        fb_w = self.fb_w if len(self.fb_w) else np.zeros(1, np.float32)
        return {
            "window": self.window.to(device),
            "twiddle": torch.from_numpy(self.twiddle).to(device),
            "fb_start": torch.from_numpy(self.fb_start).to(device),
            "fb_ptr": torch.from_numpy(self.fb_ptr).to(device),
            "fb_w": torch.from_numpy(fb_w).to(device),
        }


# ------------------------------------------------------------------------------------------------
# Resampler constants (device stand-in for ``soxr.resample(signal, in_rate=sr, out_rate=22050)``,
# reference inference.py:274-275).  soxr is a third-party C library that is absent offline, so this
# is a *restated published method* (band-limited interpolation with a Kaiser-windowed sinc, J. O.
# Smith, "Digital Audio Resampling"), designed to soxr's documented HQ targets: flat (+-1e-5 dB) to
# 0.93 of the output Nyquist, <= -124 dB from the Nyquist on.  Parity with soxr itself is UNPINNED
# (DESIGN.md section 2); the CUDA kernel is checked against a float64 direct-form evaluation.
#   y[n] = sum_j x[j] * g * h(s * (n*M/L - j)),  h(t) = rho * sinc(rho t) * kaiser_beta(t / Z), |t| <= Z
#   L/M = sr_out/sr_in in lowest terms, s = g = min(1, L/M)
RESAMPLE_ZERO_CROSSINGS = 94
RESAMPLE_BETA = 12.8
RESAMPLE_ROLLOFF = 0.9565


def resample_ratio(sr_in: int, sr_out: int = SAMPLE_RATE):
    """(L, M) with sr_out / sr_in = L / M in lowest terms."""
    sr_in, sr_out = int(sr_in), int(sr_out)
    if sr_in <= 0 or sr_out <= 0:
        raise ValueError("sample rates must be positive integers")
    g = math.gcd(sr_in, sr_out)
    return sr_out // g, sr_in // g


def resampled_length(n: int, L: int, M: int) -> int:
    """Number of output samples for n input samples: round-half-up of n * L / M."""
    return (2 * n * L + M) // (2 * M)


def resample_kernel(t):
    """h(t) of the header comment, float64, t in units of output-band zero crossings."""
    t = np.asarray(t, dtype=np.float64)
    u = np.clip(1.0 - (t / RESAMPLE_ZERO_CROSSINGS) ** 2, 0.0, None)
    w = np.i0(RESAMPLE_BETA * np.sqrt(u)) / np.i0(RESAMPLE_BETA)
    h = RESAMPLE_ROLLOFF * np.sinc(RESAMPLE_ROLLOFF * t) * w
    return np.where(np.abs(t) <= RESAMPLE_ZERO_CROSSINGS, h, 0.0)


def resample_filter_bank(sr_in: int, sr_out: int = SAMPLE_RATE):
    """Polyphase bank for the device kernel: (coef float32 [L, K], L, M, K).  Output n reads the K input
    samples q - K/2 + 1 + k (k = 0..K-1, q = floor(n M / L)) with the row phase = (n M) mod L."""
    L, M = resample_ratio(sr_in, sr_out)
    s = min(1.0, L / M)
    K = 2 * int(math.ceil(RESAMPLE_ZERO_CROSSINGS / s))
    if L * K > (1 << 26):
        raise ValueError(f"resampling {sr_in} -> {sr_out} Hz needs a {L} x {K} polyphase bank; use a rate with a "
                         "larger common divisor with the target rate")
    phase = np.arange(L, dtype=np.float64)[:, None] / L
    k = np.arange(K, dtype=np.float64)[None, :]
    coef = s * resample_kernel(s * (phase + (K // 2 - 1) - k))
    return coef.astype(np.float32), L, M, K


class LogMelSpect(torch.nn.Module):
    """Drop-in for the reference class (preprocessing.py:27-59) with every one of its analysis parameters
    (contract: ``bt_logmel_config`` in include/beatthis.h).  The reference defaults run the model path's fused
    kernel (``bt_logmel``); any other parameters run the general kernel (``bt_logmel_config``) on tables built here.
    ``_general=True`` sends the defaults through the general kernel too (for tests)."""

    DEFAULTS = (22050, 1024, 441, 30, 11000, 128, "slaney", "frame_length", 1, 1000)

    def __init__(
        self,
        sample_rate=22050,
        n_fft=1024,
        hop_length=441,
        f_min=30,
        f_max=11000,
        n_mels=128,
        mel_scale="slaney",
        normalized="frame_length",
        power=1,
        log_multiplier=1000,
        device="cuda",
        _engine=None,
        _general=False,
    ):
        super().__init__()
        from .engine import Engine

        given = (sample_rate, n_fft, hop_length, f_min, f_max, n_mels, mel_scale, normalized, power, log_multiplier)
        self.tables = MelTables(*given)
        if given == self.DEFAULTS and not _general:
            self.tables = None
            self.engine = _engine if _engine is not None else Engine.mel_only(device)
        else:
            self.engine = _engine if _engine is not None else Engine(None, None, device)
            self.device_tables = self.tables.to(self.engine.device)

    def forward(self, x):
        """Input is a waveform as a monodimensional array of shape T,
        output is a 2D log mel spectrogram of shape (F, n_mels)."""
        return self.batch([x])[0]

    def batch(self, signals):
        """Many 1-D signals in one kernel launch: a list of [1 + len_i // hop_length, n_mels] spectrograms."""
        if self.tables is None:
            return self.engine.logmel(signals)
        return self.engine.logmel_config(signals, self.tables, self.device_tables)
