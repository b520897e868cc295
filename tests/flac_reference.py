"""A FLAC encoder written from RFC 9639 for the decoder's tests: its input integers are the oracle.

It can emit every feature the decoder takes -- 4 to 32 bits per sample, 1 to 8 channels and the four channel
assignments, CONSTANT / VERBATIM / FIXED (orders 0-4) / LPC (orders 1-32) subframes, wasted bits, both Rice methods
at every partition order with escaped partitions, fixed and variable block sizes (odd sizes coded in 8 or 16 bits, a
short last block), every sample-rate code, a total-samples field of 0, extra metadata blocks, an ID3v2 prefix and frames
whose data holds false sync codes that pass CRC-8.  Nothing in it is taken from another implementation, and no file
written by libFLAC is checked here (none exists on the machines these tests run on): parity with libFLAC-written files
is unpinned.

The conventions that a misreading shared by this encoder and the decoder would hide, to check against the RFC:
  - zigzag fold of residuals: e >= 0 -> 2e, e < 0 -> -2e - 1 (section 9.2.7.1);
  - side = left - right (9.1.3); left/side carries left and side, side/right side and right;
  - mid/side: mid = (left + right) >> 1 (floor), rebuilt as (mid << 1) | (side & 1);
  - LPC: prediction = (sum_j c[j] * s[i - 1 - j]) >> shift, arithmetic shift, c[0] on the newest sample (9.2.6);
  - the first residual partition holds (block size >> partition order) - predictor order residuals (9.2.7).
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field

import numpy as np

RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10,
              96000: 11}
BITS_CODES = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6, 32: 7}
ASSIGNMENTS = {"left_side": 8, "side_right": 9, "mid_side": 10}


# ---- CRCs -----------------------------------------------------------------------------------------------------------
def _table(poly: int, width: int) -> np.ndarray:
    top, mask = 1 << (width - 1), (1 << width) - 1
    t = np.zeros(256, dtype=np.int64)
    for b in range(256):
        c = b << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) & mask if c & top else (c << 1) & mask
        t[b] = c
    return t


CRC8 = _table(0x07, 8)
CRC16 = _table(0x8005, 16)


def crc8(data: bytes) -> int:
    c = 0
    for b in data:
        c = int(CRC8[c ^ b])
    return c


def crc16_many(frames: list) -> list:
    """CRC-16 of every byte string of `frames`, vectorised across them."""
    n = len(frames)
    lens = np.array([len(f) for f in frames], dtype=np.int64)
    buf = np.zeros((n, int(lens.max()) if n else 0), dtype=np.int64)
    for i, f in enumerate(frames):
        buf[i, : len(f)] = np.frombuffer(f, dtype=np.uint8)
    crc = np.zeros(n, dtype=np.int64)
    for j in range(buf.shape[1]):
        live = lens > j
        nxt = ((crc << 8) & 0xFFFF) ^ CRC16[((crc >> 8) ^ buf[:, j]) & 0xFF]
        crc = np.where(live, nxt, crc)
    return [int(c) for c in crc]


# ---- bits -----------------------------------------------------------------------------------------------------------
class BitWriter:
    """MSB-first bits, collected as 0/1 arrays and packed once."""

    def __init__(self):
        self.chunks = []
        self.n = 0

    def bits(self, values, width: int):
        """Each value as `width` bits, two's complement (width <= 63)."""
        v = np.asarray(values, dtype=np.int64).reshape(-1)
        if width == 0 or v.size == 0:
            return
        u = v.astype(np.uint64) & np.uint64((1 << width) - 1)
        shifts = np.arange(width - 1, -1, -1, dtype=np.uint64)
        self._add(((u[:, None] >> shifts) & np.uint64(1)).astype(np.uint8).reshape(-1))

    def unary(self, q: int):
        self._add(np.r_[np.zeros(q, dtype=np.uint8), np.uint8(1)])

    def rice(self, values, k: int):
        """Zigzag-folded values: q = u >> k zeros, a one, then the k low bits of u."""
        v = np.asarray(values, dtype=np.int64)
        u = np.where(v >= 0, 2 * v, -2 * v - 1).astype(np.uint64)
        q = (u >> np.uint64(k)).astype(np.int64)
        lens = q + 1 + k
        out = np.zeros(int(lens.sum()), dtype=np.uint8)
        starts = np.cumsum(lens) - lens
        out[starts + q] = 1
        for j in range(k):
            out[starts + q + 1 + j] = ((u >> np.uint64(k - 1 - j)) & np.uint64(1)).astype(np.uint8)
        self._add(out)

    def _add(self, a):
        self.chunks.append(a)
        self.n += a.size

    def pad(self):
        if self.n % 8:
            self._add(np.zeros(8 - self.n % 8, dtype=np.uint8))

    def tobytes(self) -> bytes:
        self.pad()
        return np.packbits(np.concatenate(self.chunks)).tobytes() if self.chunks else b""


def coded_number(v: int) -> bytes:
    """The UTF-8-like coding of frame and sample numbers (9.1.5): 1 byte below 2^7, else a lead byte of n ones and a
    zero, then n - 1 bytes 10xxxxxx; up to 7 bytes (36 bits, lead 0xFE)."""
    if v < 0x80:
        return bytes([v])
    for n, cap in ((2, 11), (3, 16), (4, 21), (5, 26), (6, 31), (7, 36)):
        if v < 1 << cap:
            tail = [0x80 | ((v >> (6 * k)) & 0x3F) for k in range(n - 2, -1, -1)]
            lead = (0xFF << (8 - n)) & 0xFF | (v >> (6 * (n - 1)))
            return bytes([lead & 0xFF] + tail)
    raise ValueError("number needs more than 36 bits")


# ---- subframes ------------------------------------------------------------------------------------------------------
@dataclass
class Subframe:
    """How one channel of a frame is coded.  kind: constant | verbatim | fixed | lpc; method: 0 (4-bit Rice
    parameters) or 1 (5-bit); porder: partition order (clipped to what the block allows); escape: escape every
    other partition (the odd ones); wasted: code the common trailing zero bits as wasted bits."""
    kind: str = "lpc"
    order: int = 8
    precision: int = 12
    method: int = 0
    porder: int = 4
    escape: bool = False
    wasted: bool = True


def _trailing_zeros(x) -> int:
    nz = x[x != 0]
    if nz.size == 0:
        return 0
    w = 0
    while w < 32 and np.all((nz >> w) & 1 == 0):
        w += 1
    return w


def _lpc_coefs(x, order: int, precision: int):
    """Quantised LPC coefficients (any coefficients give an exact code; these are a least-squares fit) and shift."""
    xf = x.astype(np.float64)
    if len(x) <= order or not np.any(xf):
        c = np.zeros(order)
    else:
        A = np.stack([xf[order - 1 - j : len(x) - 1 - j] for j in range(order)], axis=1)
        c = np.linalg.lstsq(A, xf[order:], rcond=None)[0]
    cmax = np.abs(c).max() if np.any(c) else 1.0
    lim = (1 << (precision - 1)) - 1
    shift = int(np.clip(precision - 2 - int(np.ceil(np.log2(max(cmax, 1e-9)))), 0, 15))
    q = np.clip(np.round(c * (1 << shift)), -lim - 1, lim).astype(np.int64)
    return q, shift


def _residual_lpc(x, q, shift: int):
    order = len(q)
    pred = np.zeros(len(x) - order, dtype=np.int64)
    for j in range(order):
        pred += q[j] * x[order - 1 - j : len(x) - 1 - j]
    return x[order:] - (pred >> shift)


def _write_residual(w: BitWriter, e, bs: int, order: int, sf: Subframe):
    porder = sf.porder
    while porder > 0 and ((bs % (1 << porder)) or (bs >> porder) < order):
        porder -= 1
    w.bits(sf.method, 2)
    w.bits(porder, 4)
    psize, pos = bs >> porder, 0
    pbits = 5 if sf.method else 4
    kmax = (1 << pbits) - 2
    for p in range(1 << porder):
        n = psize - (order if p == 0 else 0)
        part = e[pos : pos + n]
        pos += n
        need = int(max(int(np.abs(part).max()).bit_length() + 1, 1)) if n and np.any(part) else 0
        if sf.escape and p % 2 == 1 and need <= 31:
            w.bits((1 << pbits) - 1, pbits)
            w.bits(need, 5)
            w.bits(part, need)
            continue
        u = np.where(part >= 0, 2 * part, -2 * part - 1) if n else np.zeros(1, dtype=np.int64)
        mean = float(np.mean(u)) if n else 0.0
        k = int(np.clip(int(np.floor(np.log2(mean))) if mean >= 1 else 0, 0, kmax))
        w.bits(k, pbits)
        w.rice(part, k)


def write_subframe(w: BitWriter, x, ss: int, sf: Subframe):
    """Channel samples x (int64) of `ss` bits as one subframe."""
    bs = len(x)
    wasted = _trailing_zeros(x) if sf.wasted else 0
    if wasted >= ss:
        wasted = 0
    y = x >> wasted
    s = ss - wasted
    kind = sf.kind
    if kind in ("fixed", "lpc") and sf.order > bs:  # a block shorter than the predictor goes verbatim
        kind = "verbatim"
    if kind == "constant" and not np.all(x == x[0]):
        raise ValueError("a CONSTANT subframe needs a constant channel")
    type_code = {"constant": 0, "verbatim": 1}.get(kind)
    if kind == "fixed":
        type_code = 8 + sf.order
    elif kind == "lpc":
        type_code = 31 + sf.order
    w.bits(0, 1)
    w.bits(type_code, 6)
    if wasted:
        w.bits(1, 1)
        w.unary(wasted - 1)
    else:
        w.bits(0, 1)
    if kind == "constant":
        w.bits(y[0], s)
    elif kind == "verbatim":
        w.bits(y, s)
    elif kind == "fixed":
        order = sf.order
        w.bits(y[:order], s)
        _write_residual(w, np.diff(y, order) if order else y.copy(), bs, order, sf)
    else:
        order = sf.order
        q, shift = _lpc_coefs(y, order, sf.precision)
        w.bits(y[:order], s)
        w.bits(sf.precision - 1, 4)
        w.bits(shift, 5)
        w.bits(q, sf.precision)
        _write_residual(w, _residual_lpc(y, q, shift), bs, order, sf)


# ---- frames and streams ---------------------------------------------------------------------------------------------
@dataclass
class FrameStyle:
    """How one frame is coded.  assignment: independent | left_side | side_right | mid_side (two channels);
    subframes: one Subframe for every channel, or a list per channel; bs_code: auto | 8bit | 16bit; rate_code: auto |
    streaminfo | khz | hz | tens; bits_code: auto | streaminfo; verbatim_payload: bytes a mono 16-bit frame carries as
    its VERBATIM samples (a false sync code, say)."""
    assignment: str = "independent"
    subframes: object = field(default_factory=Subframe)
    bs_code: str = "auto"
    rate_code: str = "auto"
    bits_code: str = "auto"


def _bs_code(bs: int, how: str):
    if how == "auto":
        if bs == 192:
            return 1, b""
        for k in range(4):
            if bs == 576 << k:
                return 2 + k, b""
        for k in range(8):
            if bs == 256 << k:
                return 8 + k, b""
        how = "8bit" if bs <= 256 else "16bit"
    if how == "8bit":
        return 6, bytes([bs - 1])
    return 7, (bs - 1).to_bytes(2, "big")


def _rate_code(rate: int, how: str):
    if how == "auto":
        if rate in RATE_CODES:
            return RATE_CODES[rate], b""
        how = "khz" if rate % 1000 == 0 and rate <= 255000 else "hz" if rate < 65536 else "tens"
    if how == "streaminfo":
        return 0, b""
    if how == "khz":
        return 12, bytes([rate // 1000])
    if how == "hz":
        return 13, rate.to_bytes(2, "big")
    return 14, (rate // 10).to_bytes(2, "big")


def frame_header(number: int, bs: int, rate: int, channels: int, bits: int, style: FrameStyle, variable: bool) -> bytes:
    bc, bs_tail = _bs_code(bs, style.bs_code)
    rc, rate_tail = _rate_code(rate, style.rate_code)
    ch = channels - 1 if style.assignment == "independent" else ASSIGNMENTS[style.assignment]
    sz = BITS_CODES.get(bits, 0) if style.bits_code == "auto" else 0
    h = bytes([0xFF, 0xF8 | int(variable), (bc << 4) | rc, (ch << 4) | (sz << 1)]) + coded_number(number) + bs_tail + \
        rate_tail
    return h + bytes([crc8(h)])


def encode_frame_body(x, bits: int, style: FrameStyle) -> bytes:
    """Subframes of block x [bs, channels] after the header, padded to a byte."""
    ch = x.shape[1]
    sfs = style.subframes if isinstance(style.subframes, (list, tuple)) else [style.subframes] * ch
    a = style.assignment
    if a == "independent":
        chans, sizes = [x[:, c] for c in range(ch)], [bits] * ch
    else:
        L, R = x[:, 0], x[:, 1]
        side = L - R
        if a == "left_side":
            chans, sizes = [L, side], [bits, bits + 1]
        elif a == "side_right":
            chans, sizes = [side, R], [bits + 1, bits]
        else:
            chans, sizes = [(L + R) >> 1, side], [bits, bits + 1]
    w = BitWriter()
    for c, (y, s) in enumerate(zip(chans, sizes)):
        write_subframe(w, y.astype(np.int64), s, sfs[c])
    return w.tobytes()


def streaminfo(x, rate: int, bits: int, blocks, total_zero: bool, frame_sizes) -> bytes:
    T, ch = x.shape
    body = blocks[:-1] if len(blocks) > 1 else blocks
    w = BitWriter()
    w.bits(min(body), 16)
    w.bits(max(blocks), 16)
    w.bits(min(frame_sizes), 24)
    w.bits(max(frame_sizes), 24)
    w.bits(rate, 20)
    w.bits(ch - 1, 3)
    w.bits(bits - 1, 5)
    w.bits(0 if total_zero else T, 36)
    return w.tobytes() + md5_of(x, bits)


def md5_of(x, bits: int) -> bytes:
    """STREAMINFO's MD5: the samples interleaved, each little-endian signed in ceil(bits / 8) bytes (9.2 of
    STREAMINFO)."""
    nb = (bits + 7) // 8
    b = np.ascontiguousarray(x, dtype="<i8").view(np.uint8).reshape(-1, 8)[:, :nb]
    return hashlib.md5(b.tobytes()).digest()


def metadata_block(kind: int, body: bytes, last: bool) -> bytes:
    return bytes([(0x80 if last else 0) | kind]) + len(body).to_bytes(3, "big") + body


def id3v2(size: int = 37) -> bytes:
    s = [(size >> 21) & 0x7F, (size >> 14) & 0x7F, (size >> 7) & 0x7F, size & 0x7F]
    return b"ID3" + bytes([4, 0, 0]) + bytes(s) + bytes(size)


@dataclass
class Stream:
    data: bytes            # the file
    samples: np.ndarray    # [T, channels] int64: the oracle
    frames: list           # (offset from the first frame, first sample, bytes, block size) per frame
    frames_offset: int     # byte offset of the first frame in the file


def encode(x, rate: int, bits: int, blocks=4096, style=None, variable: bool = False, total_zero: bool = False,
           extra_metadata: bool = False, id3: bool = False, false_syncs: bool = False) -> Stream:
    """A FLAC file of the integers x ([T] or [T, channels], each within `bits` bits).  blocks: a fixed block size (the
    last block is what remains) or the list of block sizes (variable: a variable-block-size stream, numbered by
    sample); style: a FrameStyle, or a function of the frame index giving one; false_syncs: every frame of a mono
    16-bit stream is followed by a VERBATIM frame whose samples hold a frame header that passes CRC-8 but does not
    continue the stream."""
    x = np.asarray(x, dtype=np.int64)
    if x.ndim == 1:
        x = x[:, None]
    T, ch = x.shape
    if isinstance(blocks, int):
        blocks = [blocks] * (T // blocks) + ([T % blocks] if T % blocks else [])
    assert sum(blocks) == T
    style_of = style if callable(style) else (lambda i, s=style or FrameStyle(): s)
    bodies, first = [], 0
    for i, bs in enumerate(blocks):
        st = style_of(i)
        if false_syncs and i % 2 == 1:
            st = FrameStyle(subframes=Subframe(kind="verbatim", wasted=False), rate_code=st.rate_code)
        head = frame_header(first if variable else i, bs, rate, ch, bits, st, variable)
        bodies.append(head + encode_frame_body(x[first : first + bs], bits, st))
        first += bs
    frames = [b + c.to_bytes(2, "big") for b, c in zip(bodies, crc16_many(bodies))]
    meta = [metadata_block(0, streaminfo(x, rate, bits, blocks, total_zero, [len(f) for f in frames]), False)]
    if extra_metadata:
        meta += [metadata_block(1, bytes(100), False),                                   # PADDING
                 metadata_block(2, b"test" + bytes(12), False),                          # APPLICATION
                 metadata_block(3, bytes(18), False),                                    # SEEKTABLE (one point)
                 metadata_block(4, (4).to_bytes(4, "little") + b"test" + bytes(4), False),  # VORBIS_COMMENT
                 metadata_block(6, bytes(32), False)]                                    # PICTURE (empty fields)
    meta[-1] = bytes([meta[-1][0] | 0x80]) + meta[-1][1:]
    prefix = (id3v2() if id3 else b"") + b"fLaC" + b"".join(meta)
    table, off, first = [], 0, 0
    for f, bs in zip(frames, blocks):
        table.append((off, first, len(f), bs))
        off += len(f)
        first += bs
    return Stream(prefix + b"".join(frames), x, table, len(prefix))


def false_sync_samples(bs: int, channels: int, bits: int, rate: int) -> np.ndarray:
    """16-bit mono samples whose big-endian bytes are a frame header (frame number 12345, so it continues nothing)
    that passes CRC-8, repeated: a VERBATIM subframe of them puts false sync codes at byte boundaries."""
    h = frame_header(12345, 4096, rate, channels, bits, FrameStyle(), False)
    h = h + bytes(len(h) % 2)
    words = np.frombuffer(h, dtype=">i2").astype(np.int64)
    return np.resize(words, bs)


def wav_twin(x, rate: int, bits: int) -> bytes:
    """A PCM WAV file of the same samples: 8, 16, 24 or 32 bits as they are; 12 or 20 bits shifted into a 16- or
    24-bit container; 4 bits into 8 (unsigned)."""
    x = np.asarray(x, dtype=np.int64)
    if x.ndim == 1:
        x = x[:, None]
    container = 8 if bits <= 8 else 16 if bits <= 16 else 24 if bits <= 24 else 32
    v = x << (container - bits)
    nb = container // 8
    if nb == 1:
        raw = (v + 128).astype(np.uint8).tobytes()
    else:
        raw = np.ascontiguousarray(v, dtype="<i8").view(np.uint8).reshape(-1, 8)[:, :nb].tobytes()
    ch = x.shape[1]
    fmt = (1).to_bytes(2, "little") + ch.to_bytes(2, "little") + rate.to_bytes(4, "little") + \
        (rate * ch * nb).to_bytes(4, "little") + (ch * nb).to_bytes(2, "little") + container.to_bytes(2, "little")
    body = b"WAVE" + b"fmt " + len(fmt).to_bytes(4, "little") + fmt + b"data" + len(raw).to_bytes(4, "little") + raw
    return b"RIFF" + len(body).to_bytes(4, "little") + body
