"""Ogg Vorbis written from the Vorbis I specification (Xiph.Org), for the tests of native Ogg Vorbis input.

Three parts:
- Ogg pages: a writer (CRC-32 with polynomial 0x04C11DB7, lacing, packets spanning pages, granule positions) and a
  reader;
- a float64 Vorbis I decoder, the oracle for bt_vorbis_decode: codeword assignment by the specification's rule,
  floor1, residues 0 / 1 / 2, inverse square-polar coupling, the IMDCT, the power-complementary window, overlap-add and
  the granule-position trims;
- an encoder built from the analysis side: the MDCT under the Vorbis window, a floor1 fit, VQ quantisation of the
  residue with cascades, square-polar coupling, and a setup-header writer with chosen codebooks.

No real Vorbis file, encoder or library is used; parity with libvorbis output is not pinned."""
from __future__ import annotations

import dataclasses
import struct

import numpy as np

# ------------------------------------------------------------------------------------------------ bits, CRC, Ogg pages


class BitWriter:
    """LSB first within each byte, as Vorbis packs its fields."""

    def __init__(self):
        self.bits = []

    def write(self, value: int, n: int):
        for i in range(n):
            self.bits.append((value >> i) & 1)

    def code(self, code: int, length: int):  # a codeword, its first bit the most significant
        for i in range(length - 1, -1, -1):
            self.bits.append((code >> i) & 1)

    def bytes(self) -> bytes:
        out = bytearray((len(self.bits) + 7) // 8)
        for i, b in enumerate(self.bits):
            out[i >> 3] |= b << (i & 7)
        return bytes(out)


class EndOfPacket(Exception):
    pass


class BitReader:
    def __init__(self, data: bytes):
        self.data, self.pos = data, 0

    def bit(self) -> int:
        if self.pos >= 8 * len(self.data):
            raise EndOfPacket
        b = (self.data[self.pos >> 3] >> (self.pos & 7)) & 1
        self.pos += 1
        return b

    def read(self, n: int) -> int:
        if self.pos + n > 8 * len(self.data):
            self.pos = 8 * len(self.data)
            raise EndOfPacket
        return sum(self.bit() << i for i in range(n))


def ogg_crc(data: bytes) -> int:
    crc = 0
    for b in data:
        crc ^= b << 24
        for _ in range(8):
            crc = ((crc << 1) ^ 0x04C11DB7) if crc & 0x80000000 else crc << 1
            crc &= 0xFFFFFFFF
    return crc


def page(body_segments, flags: int, granule: int, serial: int, seq: int, body: bytes) -> bytes:
    head = b"OggS" + bytes([0, flags]) + struct.pack("<qII", granule, serial, seq) + b"\0\0\0\0"
    head += bytes([len(body_segments)]) + bytes(body_segments)
    crc = ogg_crc(head + body)
    return head[:22] + struct.pack("<I", crc) + head[26:] + body


def ogg_stream(packets, granules, serial=0x1234, page_bytes=4000, packets_per_page=None, seq0=0,
               header_pages=True) -> bytes:
    """Pages of a logical stream holding `packets` (bytes); granules[k]: the granule position after packet k (-1
    where none).  The identification header gets its own page and the comment and setup headers end their page
    (header_pages); audio pages close after packets_per_page packets or when about page_bytes are filled, so packets
    span pages.  The last page carries the end-of-stream flag."""
    pages, seq = [], seq0
    segs, body, cont, gran, count = [], b"", False, -1, 0

    def flush(last=False, next_cont=False):
        nonlocal segs, body, cont, gran, seq, count
        flags = (1 if cont else 0) | (2 if seq == seq0 else 0) | (4 if last else 0)
        pages.append(page(segs, flags, gran, serial, seq, body))
        seq += 1
        segs, body, gran, count, cont = [], b"", -1, 0, next_cont

    for k, p in enumerate(packets):
        rest = p
        while True:
            if len(segs) == 255:
                flush(next_cont=True)
            take = min(255, len(rest))
            segs.append(take)
            body += rest[:take]
            rest = rest[take:]
            if take < 255:
                break
            if not rest:  # a packet of 255 k bytes ends with a 0 lacing value
                if len(segs) == 255:
                    flush(next_cont=True)
                segs.append(0)
                break
            if len(body) >= page_bytes:
                flush(next_cont=True)
        gran = granules[k]
        count += 1
        last = k == len(packets) - 1
        boundary = (header_pages and k in (0, 2)) or last or len(body) >= page_bytes or (
            packets_per_page is not None and count >= packets_per_page)
        if boundary:
            flush(last)
    return b"".join(pages)


def read_pages(data: bytes):
    """[(header_type, granule, serial, seq, [packet pieces as (bytes, completes)])] of a file's complete pages."""
    out, pos = [], 0
    while pos + 27 <= len(data) and data[pos:pos + 4] == b"OggS":
        nseg = data[pos + 26]
        laces = data[pos + 27:pos + 27 + nseg]
        body_at = pos + 27 + nseg
        size = sum(laces)
        if body_at + size > len(data) or len(laces) < nseg:
            break
        flags = data[pos + 5]
        granule, serial, seq = struct.unpack("<qII", data[pos + 6:pos + 22])
        pieces, at, cur = [], body_at, b""
        for lace in laces:
            cur += data[at:at + lace]
            at += lace
            if lace < 255:
                pieces.append((cur, True))
                cur = b""
        if laces and laces[-1] == 255:
            pieces.append((cur, False))
        out.append((flags, granule, serial, seq, pieces))
        pos = body_at + size
    return out


# ------------------------------------------------------------------------------------------------ codebooks


def float32_pack(x: float) -> int:
    """The specification's float32 packing of x (a 21-bit mantissa, exponent bias 788), exact for the values used."""
    if x == 0:
        return 0
    sign = 0x80000000 if x < 0 else 0
    m, e = abs(x), 0
    while m < (1 << 20):
        m *= 2
        e -= 1
    while m >= (1 << 21):
        m /= 2
        e += 1
    assert m == int(m), x
    return sign | ((e + 788) << 21) | int(m)


def float32_unpack(x: int) -> float:
    mantissa = x & 0x1FFFFF
    exponent = (x & 0x7FE00000) >> 21
    return float(np.ldexp(-mantissa if x & 0x80000000 else mantissa, exponent - 788))


def lookup1_values(entries: int, dim: int) -> int:
    r = 0
    while (r + 1) ** dim <= entries:
        r += 1
    return r


def assign_codewords(lengths):
    """The specification's assignment: each used entry (length > 0) takes the numerically lowest codeword of its length
    that no earlier codeword prefixes or is prefixed by.  {entry: (code, length)}; ValueError when over-full.  The
    free codewords are kept as a set of prefixes, split on demand (the lowest free one of a length is a prefix's first
    extension)."""
    free = {(0, 0)}  # (code, length) of free subtrees
    out = {}
    for e, L in enumerate(lengths):
        if L <= 0:
            continue
        cands = [(c << (L - l), c, l) for (c, l) in free if l <= L]
        if not cands:
            raise ValueError("over-full codebook")
        low, c, l = min(cands)
        free.remove((c, l))
        for d in range(l, L):  # split: keep the upper halves free
            free.add(((low >> (L - d - 1)) | 1, d + 1))
        out[e] = (low, L)
    return out


@dataclasses.dataclass
class Book:
    dim: int
    lengths: list  # per entry, 0: unused
    lookup: int = 0
    minimum: float = 0.0
    delta: float = 1.0
    value_bits: int = 4
    sequence_p: int = 0
    multiplicands: list = None
    ordered: bool = False  # write the lengths in the ordered form (they must not decrease)
    sparse: bool = None    # None: sparse when an entry is unused

    @property
    def entries(self):
        return len(self.lengths)

    def codes(self):
        if getattr(self, "_codes", None) is None:
            self._codes = assign_codewords(self.lengths)
        return self._codes

    def vectors(self) -> np.ndarray:
        """[entries, dim] float64 VQ vectors."""
        if getattr(self, "_vq", None) is None:
            self._vq = self._expand()
        return self._vq

    def _expand(self) -> np.ndarray:
        n = self.entries
        mult = self.multiplicands
        out = np.zeros((n, self.dim))
        lv = lookup1_values(n, self.dim) if self.lookup == 1 else n * self.dim
        mn, delta = float32_unpack(float32_pack(self.minimum)), float32_unpack(float32_pack(self.delta))
        for e in range(n):
            last, div = 0.0, 1
            for j in range(self.dim):
                off = (e // div) % lv if self.lookup == 1 else e * self.dim + j
                v = mult[off] * delta + mn + last
                if self.sequence_p:
                    last = v
                out[e, j] = v
                div *= lv
        return out


def lattice_book(dim: int, values: int, delta: float, length_of=None, **kw) -> Book:
    """A lookup-type-1 book of values^dim entries: multiplicand m maps to (m - (values - 1) / 2) * delta."""
    n = values ** dim
    lengths = [length_of(e) if length_of else 0 for e in range(n)]
    if length_of is None:
        lengths = complete_lengths(n)
    return Book(dim, lengths, lookup=1, minimum=-(values - 1) / 2 * delta, delta=delta,
                value_bits=max(1, int(values - 1).bit_length()), multiplicands=list(range(values)), **kw)


def complete_lengths(n: int):
    """Lengths of a complete prefix code over n entries: as balanced as possible."""
    if n == 1:
        return [1]
    L = (n - 1).bit_length()
    short = (1 << L) - n  # entries that take L - 1 bits
    return [L - 1] * short + [L] * (n - short)


def scalar_book(n: int, **kw) -> Book:
    return Book(1, complete_lengths(n), **kw)


# ------------------------------------------------------------------------------------------------ setup description


@dataclasses.dataclass
class Floor1:
    partition_class: list
    class_dim: list
    class_sub: list
    class_master: list
    sub_books: list  # per class, 2^sub entries: book index or -1
    multiplier: int
    rangebits: int
    xs: list  # the X values after the first two

    @property
    def x(self):
        return [0, 1 << self.rangebits] + list(self.xs)


@dataclasses.dataclass
class Residue:
    type: int
    begin: int
    end: int
    partition_size: int
    classifications: int
    classbook: int
    books: list  # [classification][pass]: book index or -1


@dataclasses.dataclass
class Mapping:
    submaps: int = 1
    coupling: list = dataclasses.field(default_factory=list)  # (magnitude, angle)
    mux: list = None
    submap_floor: list = dataclasses.field(default_factory=lambda: [0])
    submap_residue: list = dataclasses.field(default_factory=lambda: [0])


@dataclasses.dataclass
class Setup:
    channels: int
    rate: int
    bs: tuple  # (blocksize_0, blocksize_1)
    books: list
    floors: list
    residues: list
    mappings: list
    modes: list  # (blockflag, mapping)
    floor_type: int = 1


def ilog(v: int) -> int:
    return int(v).bit_length() if v > 0 else 0


def id_header(s: Setup) -> bytes:
    b0, b1 = ilog(s.bs[0]) - 1, ilog(s.bs[1]) - 1
    return (b"\x01vorbis" + struct.pack("<IBIiii", 0, s.channels, s.rate, 0, 128000, 0) + bytes([b0 | (b1 << 4)])
            + b"\x01")


def comment_header() -> bytes:
    vendor = b"beat_this_b200 test encoder"
    return b"\x03vorbis" + struct.pack("<I", len(vendor)) + vendor + struct.pack("<I", 0) + b"\x01"


def setup_header(s: Setup) -> bytes:
    w = BitWriter()
    w.write(len(s.books) - 1, 8)
    for bk in s.books:
        w.write(0x564342, 24)
        w.write(bk.dim, 16)
        w.write(bk.entries, 24)
        if bk.ordered:
            w.write(1, 1)
            L = bk.lengths
            w.write(L[0] - 1, 5)
            e = 0
            cur = L[0]
            while e < len(L):
                num = 0
                while e + num < len(L) and L[e + num] == cur:
                    num += 1
                w.write(num, ilog(len(L) - e))
                e += num
                cur += 1
        else:
            w.write(0, 1)
            sparse = any(v == 0 for v in bk.lengths) if bk.sparse is None else bk.sparse
            w.write(int(sparse), 1)
            for L in bk.lengths:
                if sparse:
                    w.write(int(L > 0), 1)
                    if L > 0:
                        w.write(L - 1, 5)
                else:
                    w.write(L - 1, 5)
        w.write(bk.lookup, 4)
        if bk.lookup:
            w.write(float32_pack(bk.minimum), 32)
            w.write(float32_pack(bk.delta), 32)
            w.write(bk.value_bits - 1, 4)
            w.write(bk.sequence_p, 1)
            for m in bk.multiplicands:
                w.write(m, bk.value_bits)
    w.write(0, 6)
    w.write(0, 16)
    w.write(len(s.floors) - 1, 6)
    for f in s.floors:
        w.write(s.floor_type, 16)
        if s.floor_type == 0:
            w.write(0, 8), w.write(0, 16), w.write(0, 16), w.write(0, 6), w.write(0, 8), w.write(0, 4), w.write(0, 8)
            continue
        w.write(len(f.partition_class), 5)
        for c in f.partition_class:
            w.write(c, 4)
        for c in range(max(f.partition_class, default=-1) + 1):
            w.write(f.class_dim[c] - 1, 3)
            w.write(f.class_sub[c], 2)
            if f.class_sub[c]:
                w.write(f.class_master[c], 8)
            for j in range(1 << f.class_sub[c]):
                w.write(f.sub_books[c][j] + 1, 8)
        w.write(f.multiplier - 1, 2)
        w.write(f.rangebits, 4)
        for x in f.xs:
            w.write(x, f.rangebits)
    w.write(len(s.residues) - 1, 6)
    for r in s.residues:
        w.write(r.type, 16)
        w.write(r.begin, 24)
        w.write(r.end, 24)
        w.write(r.partition_size - 1, 24)
        w.write(r.classifications - 1, 6)
        w.write(r.classbook, 8)
        for c in range(r.classifications):
            casc = sum(1 << p for p in range(8) if r.books[c][p] >= 0)
            w.write(casc & 7, 3)
            w.write(int(casc > 7), 1)
            if casc > 7:
                w.write(casc >> 3, 5)
        for c in range(r.classifications):
            for p in range(8):
                if r.books[c][p] >= 0:
                    w.write(r.books[c][p], 8)
    w.write(len(s.mappings) - 1, 6)
    for m in s.mappings:
        w.write(0, 16)
        w.write(int(m.submaps > 1), 1)
        if m.submaps > 1:
            w.write(m.submaps - 1, 4)
        w.write(int(bool(m.coupling)), 1)
        if m.coupling:
            w.write(len(m.coupling) - 1, 8)
            for a, b in m.coupling:
                w.write(a, ilog(s.channels - 1))
                w.write(b, ilog(s.channels - 1))
        w.write(0, 2)
        if m.submaps > 1:
            for c in range(s.channels):
                w.write(m.mux[c], 4)
        for i in range(m.submaps):
            w.write(0, 8)
            w.write(m.submap_floor[i], 8)
            w.write(m.submap_residue[i], 8)
    w.write(len(s.modes) - 1, 6)
    for bf, mp in s.modes:
        w.write(bf, 1)
        w.write(0, 16)
        w.write(0, 16)
        w.write(mp, 8)
    w.write(1, 1)
    return b"\x05vorbis" + w.bytes()


# ------------------------------------------------------------------------------------------------ the decoder (oracle)

RANGES = {1: 256, 2: 128, 3: 86, 4: 64}
DB = 10.0 ** (7.0 * (np.arange(256) - 255) / 256.0)  # floor1 inverse dB table


def slope(n: int) -> np.ndarray:
    """The rising half of the Vorbis window of a block of n: sin(pi/2 sin^2((i + 1/2) / (n/2) pi/2))."""
    i = np.arange(n // 2)
    return np.sin(np.pi / 2 * np.sin((i + 0.5) / (n // 2) * np.pi / 2) ** 2)


def window(n: int, long_block: bool, prev_long: bool, next_long: bool, b0: int) -> np.ndarray:
    w = np.zeros(n)
    if long_block and not prev_long:
        ls, le = n // 4 - b0 // 4, n // 4 + b0 // 4
    else:
        ls, le = 0, n // 2
    if long_block and not next_long:
        rs, re = 3 * n // 4 - b0 // 4, 3 * n // 4 + b0 // 4
    else:
        rs, re = n // 2, n
    w[ls:le] = slope(2 * (le - ls))
    w[le:rs] = 1
    w[rs:re] = slope(2 * (re - rs))[::-1]
    return w


def imdct(X: np.ndarray) -> np.ndarray:
    """y[n] = sum_k X[k] cos(2 pi / N (n + 1/2 + N/4)(k + 1/2)), N = 2 len(X), through one 2N-point inverse FFT."""
    M = len(X)
    N = 2 * M
    m = 2 * np.arange(N) + 1 + N // 2
    z = np.fft.ifft(X, 2 * N) * (2 * N)
    return np.real(np.exp(1j * np.pi * m / (2 * N)) * z[m % (2 * N)])


def render_point(x0, y0, x1, y1, x):
    dy, adx = y1 - y0, x1 - x0
    off = abs(dy) * (x - x0) // adx
    return y0 - off if dy < 0 else y0 + off


def render_line(x0, y0, x1, y1, v):
    dy, adx = y1 - y0, x1 - x0
    base = int(dy / adx)
    ady = abs(dy) - abs(base) * adx
    sy = base - 1 if dy < 0 else base + 1
    y, err = y0, 0
    if x0 < len(v):
        v[x0] = y
    for x in range(x0 + 1, x1):
        err += ady
        if err >= adx:
            err -= adx
            y += sy
        else:
            y += base
        if x < len(v):
            v[x] = y


class Decoder:
    """The oracle: decode(data) -> Decoded(pcm [n, channels] float64, rate)."""

    def __init__(self, setup_packets):
        ident, _, setup = setup_packets
        assert ident[:7] == b"\x01vorbis"
        self.channels = ident[11]
        self.rate = struct.unpack("<I", ident[12:16])[0]
        self.bs = (1 << (ident[28] & 15), 1 << (ident[28] >> 4))
        self.l1 = []  # per packet: a bound on the magnitude of every value its fp32 arithmetic forms
        self._parse_setup(setup)

    def _parse_setup(self, data):
        r = BitReader(data[7:])
        self.books = []
        for _ in range(r.read(8) + 1):
            assert r.read(24) == 0x564342
            dim, entries = r.read(16), r.read(24)
            lengths = [0] * entries
            if not r.read(1):
                sparse = r.read(1)
                for e in range(entries):
                    if not sparse or r.read(1):
                        lengths[e] = r.read(5) + 1
            else:
                e, L = 0, r.read(5) + 1
                while e < entries:
                    num = r.read(ilog(entries - e))
                    lengths[e:e + num] = [L] * num
                    e += num
                    L += 1
            lookup = r.read(4)
            bk = Book(dim, lengths, lookup)
            if lookup:
                bk.minimum, bk.delta = float32_unpack(r.read(32)), float32_unpack(r.read(32))
                bk.value_bits, bk.sequence_p = r.read(4) + 1, r.read(1)
                nv = lookup1_values(entries, dim) if lookup == 1 else entries * dim
                bk.multiplicands = [r.read(bk.value_bits) for _ in range(nv)]
            bk.codes_ = {code: e for e, code in bk.codes().items()}
            bk.vq = self._vectors(bk) if lookup else None
            self.books.append(bk)
        for _ in range(r.read(6) + 1):
            assert r.read(16) == 0
        self.floors = []
        for _ in range(r.read(6) + 1):
            assert r.read(16) == 1
            pc = [r.read(4) for _ in range(r.read(5))]
            dims, subs, masters, sbooks = [], [], [], []
            for _ in range(max(pc, default=-1) + 1):
                dims.append(r.read(3) + 1)
                subs.append(r.read(2))
                masters.append(r.read(8) if subs[-1] else 0)
                sbooks.append([r.read(8) - 1 for _ in range(1 << subs[-1])])
            mult, rb = r.read(2) + 1, r.read(4)
            xs = [r.read(rb) for c in pc for _ in range(dims[c])]
            self.floors.append(Floor1(pc, dims, subs, masters, sbooks, mult, rb, xs))
        self.residues = []
        for _ in range(r.read(6) + 1):
            t, b, e, ps, nc, cb = r.read(16), r.read(24), r.read(24), r.read(24) + 1, r.read(6) + 1, r.read(8)
            casc = []
            for _ in range(nc):
                c = r.read(3)
                if r.read(1):
                    c |= r.read(5) << 3
                casc.append(c)
            books = [[r.read(8) if casc[c] >> p & 1 else -1 for p in range(8)] for c in range(nc)]
            self.residues.append(Residue(t, b, e, ps, nc, cb, books))
        self.mappings = []
        for _ in range(r.read(6) + 1):
            assert r.read(16) == 0
            m = Mapping()
            m.submaps = r.read(4) + 1 if r.read(1) else 1
            if r.read(1):
                cb = ilog(self.channels - 1)
                m.coupling = [(r.read(cb), r.read(cb)) for _ in range(r.read(8) + 1)]
            assert r.read(2) == 0
            m.mux = [r.read(4) for _ in range(self.channels)] if m.submaps > 1 else [0] * self.channels
            m.submap_floor, m.submap_residue = [], []
            for _ in range(m.submaps):
                r.read(8)
                m.submap_floor.append(r.read(8))
                m.submap_residue.append(r.read(8))
            self.mappings.append(m)
        self.modes = []
        for _ in range(r.read(6) + 1):
            bf = r.read(1)
            r.read(16), r.read(16)
            self.modes.append((bf, r.read(8)))
        assert r.read(1) == 1

    @staticmethod
    def _vectors(bk):
        # the decoder's own expansion (the specification's loop), rounded to float32 as the device tables are not
        out = np.zeros((bk.entries, bk.dim))
        lv = lookup1_values(bk.entries, bk.dim) if bk.lookup == 1 else bk.entries * bk.dim
        for e in range(bk.entries):
            last, div = 0.0, 1
            for j in range(bk.dim):
                off = (e // div) % lv if bk.lookup == 1 else e * bk.dim + j
                v = bk.multiplicands[off] * bk.delta + bk.minimum + last
                if bk.sequence_p:
                    last = v
                out[e, j] = v
                div *= lv
        return out

    def entry(self, r: BitReader, b: int) -> int:
        bk = self.books[b]
        code, L = 0, 0
        maxlen = max(bk.lengths)
        while True:
            code = (code << 1) | r.bit()
            L += 1
            if (code, L) in bk.codes_:
                return bk.codes_[(code, L)]
            if L >= maxlen:
                raise ValueError("codeword not in the book")

    def packet(self, data: bytes):
        """(n, prev_long, next_long, blockflag, [channel vectors of n floats: windowed IMDCT output])."""
        r = BitReader(data)
        assert r.read(1) == 0
        mode = r.read(ilog(len(self.modes) - 1))
        if mode >= len(self.modes):
            raise ValueError("mode number out of range")
        bf, mp = self.modes[mode]
        n = self.bs[bf]
        prev = nxt = 0
        if bf:
            prev, nxt = r.read(1), r.read(1)
        m = self.mappings[mp]
        ch = self.channels
        floors = [None] * ch
        spec = np.zeros((ch, n // 2))
        pre = np.zeros((ch, n // 2))  # the residue vectors before uncoupling
        try:
            for c in range(ch):
                floors[c] = self.floor_decode(r, self.floors[m.submap_floor[m.mux[c]]])
        except EndOfPacket:
            floors = [None] * ch
        else:
            nonzero = [f is not None for f in floors]
            for a, b in m.coupling:
                if nonzero[a] or nonzero[b]:
                    nonzero[a] = nonzero[b] = True
            try:
                for s in range(m.submaps):
                    chans = [c for c in range(ch) if m.mux[c] == s]
                    self.residue_decode(r, self.residues[m.submap_residue[s]], spec, chans,
                                        [not nonzero[c] for c in chans], n // 2)
            except EndOfPacket:
                pass
            pre[:] = spec
            for a, b in reversed(m.coupling):
                M, A = spec[a].copy(), spec[b].copy()
                pos = M > 0
                apos = A > 0
                spec[a] = np.where(pos, np.where(apos, M, M + A), np.where(apos, M, M - A))
                spec[b] = np.where(pos, np.where(apos, M - A, M), np.where(apos, M + A, M))
        out = []
        w = window(n, bf, prev, nxt, self.bs[0])
        l1 = 0.0
        for c in range(ch):
            if floors[c] is None:
                out.append(np.zeros(n))
                continue
            curve = self.floor_curve(self.floors[m.submap_floor[m.mux[c]]], floors[c], n // 2)
            l1 += np.sum(np.abs(spec[c]) * curve) + np.sum(np.abs(pre[c])) * curve.max()
            out.append(imdct(spec[c] * curve) * w)
        self.l1.append(l1)
        return n, out

    def floor_decode(self, r, f: Floor1):
        if not r.read(1):
            return None
        rng = RANGES[f.multiplier]
        y = [r.read(ilog(rng - 1)), r.read(ilog(rng - 1))]
        for cls in f.partition_class:
            cdim, cbits = f.class_dim[cls], f.class_sub[cls]
            cval = self.entry(r, f.class_master[cls]) if cbits else 0
            for _ in range(cdim):
                book = f.sub_books[cls][cval & ((1 << cbits) - 1)]
                cval >>= cbits
                y.append(self.entry(r, book) if book >= 0 else 0)
        return y

    @staticmethod
    def floor_curve(f: Floor1, y, n2):
        rng = RANGES[f.multiplier]
        x = f.x
        fy, used = list(y[:2]), [True, True] + [False] * (len(x) - 2)
        for i in range(2, len(x)):
            lo = max((j for j in range(i) if x[j] < x[i]), key=lambda j: x[j])
            hi = min((j for j in range(i) if x[j] > x[i]), key=lambda j: x[j])
            pred = render_point(x[lo], fy[lo], x[hi], fy[hi], x[i])
            val, high, low = y[i], rng - pred, pred
            room = min(high, low) * 2
            if val:
                used[lo] = used[hi] = used[i] = True
                if val >= room:
                    fy.append(val - low + pred if high > low else pred - val + high - 1)
                else:
                    fy.append(pred - (val + 1) // 2 if val & 1 else pred + val // 2)
            else:
                fy.append(pred)
        v = np.zeros(n2, dtype=np.int64)
        order = sorted(range(len(x)), key=lambda i: x[i])
        lx, ly = 0, fy[0] * f.multiplier
        hx, hy = 0, ly
        for i in order[1:]:
            if used[i]:
                hx, hy = x[i], fy[i] * f.multiplier
                render_line(lx, ly, hx, hy, v)
                lx, ly = hx, hy
        if hx < n2:
            render_line(hx, hy, n2, hy, v)
        return DB[np.clip(v, 0, 255)]

    def residue_decode(self, r, res: Residue, spec, chans, skip, n2):
        nch = len(chans)
        if res.type == 2:
            if all(skip):
                return
            vecs = [np.zeros(n2 * nch)]
            skip = [False]
        else:
            vecs = [np.zeros(n2) for _ in chans]
        size = len(vecs[0])
        lb, le = min(res.begin, size), min(res.end, size)
        parts = (le - lb) // res.partition_size
        cpw = self.books[res.classbook].dim
        cls = [[0] * (parts + cpw) for _ in vecs]
        try:
            if le - lb > 0 and parts:
                for p in range(8):
                    pc = 0
                    while pc < parts:
                        if p == 0:
                            for j in range(len(vecs)):
                                if skip[j]:
                                    continue
                                temp = self.entry(r, res.classbook)
                                for i in range(cpw - 1, -1, -1):
                                    cls[j][i + pc] = temp % res.classifications
                                    temp //= res.classifications
                        i = 0
                        while i < cpw and pc < parts:
                            for j in range(len(vecs)):
                                if skip[j]:
                                    continue
                                book = res.books[cls[j][pc]][p]
                                if book >= 0:
                                    self._partition(r, res, book, vecs[j], lb + pc * res.partition_size)
                            i += 1
                            pc += 1
        finally:
            if res.type == 2:
                for k, c in enumerate(chans):
                    spec[c] += vecs[0][k::nch]
            else:
                for k, c in enumerate(chans):
                    spec[c] += vecs[k]

    def _partition(self, r, res, book, v, off):
        bk = self.books[book]
        d, n = bk.dim, res.partition_size
        if res.type == 0:
            step = n // d
            for j in range(step):
                e = self.entry(r, book)
                for k in range(d):
                    v[off + j + k * step] += bk.vq[e, k]
        else:
            j = 0
            while j < n:
                e = self.entry(r, book)
                for k in range(d):
                    v[off + j] += bk.vq[e, k]
                    j += 1


@dataclasses.dataclass
class Decoded:
    pcm: np.ndarray  # [n, channels] float64
    rate: int
    skip: int
    n_packets: int
    l1: float        # the largest per-packet magnitude bound


def packets_of(data: bytes):
    """[(packet bytes, page index it completes on)] and per-page granules, from complete pages."""
    pages = read_pages(data)
    out, cur = [], b""
    for k, (_, _, _, _, pieces) in enumerate(pages):
        for piece, done in pieces:
            cur += piece
            if done:
                out.append((cur, k))
                cur = b""
    return out, [p[1] for p in pages]


def decode(data: bytes) -> Decoded:
    pk, granules = packets_of(data)
    dec = Decoder([p for p, _ in pk[:3]])
    blocks, pages = [], []
    for p, pg in pk[3:]:
        if not p or p[0] & 1:
            continue
        try:
            n, out = dec.packet(p)
        except EndOfPacket:
            continue  # a packet that ends before its mode and window flags is dropped
        blocks.append((n, np.stack(out)))
        pages.append(pg)
    ch = dec.channels
    ends = [0]
    for k in range(1, len(blocks)):
        ends.append(ends[-1] + blocks[k - 1][0] // 4 + blocks[k][0] // 4)
    total = ends[-1] if blocks else 0
    pcm = np.zeros((total, ch))
    for k in range(1, len(blocks)):
        na, a = blocks[k - 1]
        nb, b = blocks[k]
        for t in range(ends[k - 1], ends[k]):
            d = t - ends[k - 1]
            ia, ib = na // 2 + d, nb // 4 - na // 4 + d
            pcm[t] = (a[:, ia] if ia < na else 0) + (b[:, ib] if ib >= 0 else 0)
    base, g_end, first = 0, -1, True
    for k in range(len(blocks)):
        if k + 1 < len(blocks) and pages[k + 1] == pages[k]:
            continue
        g = granules[pages[k]]
        if g == -1:
            continue
        if first:
            base = g - ends[k]
        first = False
        g_end = g
    skip = max(0, -base)
    stop = total if g_end < 0 else min(total, g_end - base)
    return Decoded(pcm[skip:max(stop, skip)], dec.rate, skip, len(blocks), max(dec.l1, default=0.0))


# ------------------------------------------------------------------------------------------------ the encoder


def ends_of(flags, bs):
    ns = [bs[f] for f in flags]
    ends = [0]
    for k in range(1, len(ns)):
        ends.append(ends[-1] + ns[k - 1] // 4 + ns[k] // 4)
    return ns, ends


def analysis(signal: np.ndarray, flags, bs):
    """MDCT spectra [packet][channel] of signal [n, ch] under the Vorbis windows of the block sequence `flags`: decoded
    sample t of the stream is signal[t] (packet 0 is centred on sample 0)."""
    ns, ends = ends_of(flags, bs)
    out = []
    for k, n in enumerate(ns):
        start = ends[k] - n // 2  # block k's index n/2 is decoded sample ends[k]
        prev = flags[k - 1] if k > 0 else flags[k]
        nxt = flags[k + 1] if k + 1 < len(flags) else flags[k]
        w = window(n, flags[k], prev, nxt, bs[0])
        seg = np.zeros((n, signal.shape[1]))
        lo, hi = max(start, 0), min(start + n, len(signal))
        if hi > lo:
            seg[lo - start:hi - start] = signal[lo:hi]
        out.append([mdct(seg[:, c] * w) for c in range(signal.shape[1])])
    return out, ns, ends


def mdct(x: np.ndarray) -> np.ndarray:
    """X[k] = (4 / N) sum_n x[n] cos(2 pi / N (n + 1/2 + N/4)(k + 1/2)), the analysis transform whose imdct under the
    power-complementary window overlap-adds back to the signal; through one 4N-point FFT of x placed at
    m_n = 2n + 1 + N/2, since cos(pi m (2k + 1) / 2N) = Re e^{-2 pi i m (2k + 1) / 4N}."""
    N = len(x)
    m = 2 * np.arange(N) + 1 + N // 2
    buf = np.zeros(4 * N)
    buf[m] = x
    return (4.0 / N) * np.real(np.fft.fft(buf)[2 * np.arange(N // 2) + 1])


@dataclasses.dataclass
class Plan:
    """How the encoder codes a stream."""
    setup: Setup
    flags: list                  # block flag of every packet
    trim_front: int = 0          # decoded samples the first page's granule trims
    trim_end: int = 0            # samples the last page's granule trims
    packets_per_page: int = None
    page_bytes: int = 4000
    cut: dict = None             # {packet index: bytes kept}: packets cut short


def fit_floor(f: Floor1, mag: np.ndarray, books=None):
    """Decoded Y values that make floor `f` follow the log magnitude envelope of one spectrum (n/2 lines): the target
    at each post from the largest magnitude near it, coded against the decoder's prediction (floor1 step 2 inverted).
    Posts whose subclass has no book keep the prediction."""
    rng = RANGES[f.multiplier]
    x = f.x
    n2 = len(mag)

    def target(xi):
        lo, hi = max(0, xi - 4), min(n2, xi + 5)
        m = mag[lo:hi].max() if hi > lo else 0.0
        db = int(np.clip(np.round(255 + 256 / 7 * np.log10(max(m, 1e-7))), 0, 255))
        return min(rng - 1, db // f.multiplier)

    y = [target(x[0]), target(min(x[1], n2 - 1))]
    fy = list(y)
    # posts in coding order with the book (or none) that codes them
    post_class = []
    for cls in f.partition_class:
        for j in range(f.class_dim[cls]):
            post_class.append(cls)
    subs = []
    for i in range(2, len(x)):
        lo = max((j for j in range(i) if x[j] < x[i]), key=lambda j: x[j])
        hi = min((j for j in range(i) if x[j] > x[i]), key=lambda j: x[j])
        pred = render_point(x[lo], fy[lo], x[hi], fy[hi], x[i])
        t = target(min(x[i], n2 - 1))
        high, low = rng - pred, pred
        room = min(high, low) * 2
        cls = post_class[i - 2]
        has_book = any(b >= 0 for b in f.sub_books[cls])
        d = t - pred
        if d == 0 or not has_book:
            val = 0
        elif 0 < 2 * d < room:
            val = 2 * d
        elif d < 0 and 2 * -d - 1 < room:
            val = 2 * -d - 1
        elif high > low:
            val = t if t >= room else 0
        else:
            val = pred - t + high - 1
            if val < room:
                val = 0
        if val and books is not None and not any(
                b >= 0 and val < books[b].entries and books[b].lengths[val] > 0 for b in f.sub_books[cls]):
            val = 0  # no book of the post's class codes it
        if val:
            fy.append(val - low + pred if val >= room and high > low else
                      (pred - val + high - 1 if val >= room else (pred - (val + 1) // 2 if val & 1 else pred + val // 2)))
        else:
            fy.append(pred)
        y.append(val)
    return y


def encode_floor(w: BitWriter, f: Floor1, y, books):
    """The floor1 packet data of decoded values y (the subclass of a post: the first with a book when y != 0, else
    one with none when there is one)."""
    rng = RANGES[f.multiplier]
    w.write(1, 1)
    w.write(y[0], ilog(rng - 1))
    w.write(y[1], ilog(rng - 1))
    off = 2
    for cls in f.partition_class:
        cdim, cbits = f.class_dim[cls], f.class_sub[cls]
        sb = f.sub_books[cls]
        choice = []
        for j in range(cdim):
            v = y[off + j]
            with_book = [s for s in range(1 << cbits) if sb[s] >= 0 and v < books[sb[s]].entries
                         and books[sb[s]].lengths[v] > 0]
            without = [s for s in range(1 << cbits) if sb[s] < 0]
            choice.append(without[0] if v == 0 and without else with_book[0])
        if cbits:
            cval = sum(s << (cbits * j) for j, s in enumerate(choice))
            code, L = books[f.class_master[cls]].codes()[cval]
            w.code(code, L)
        for j in range(cdim):
            b = sb[choice[j]]
            if b >= 0:
                code, L = books[b].codes()[y[off + j]]
                w.code(code, L)
        off += cdim


def quantise(vec: np.ndarray, book: Book, kind: int, step_of=None):
    """Entries of `book` that code vec (partition values) for residue type 0 (interleaved by step) or 1/2 (in order),
    chosen greedily per vector; (entries, the coded values)."""
    vq = book.vectors()
    used = np.array([L > 0 for L in book.lengths])
    d = book.dim
    n = len(vec)
    coded = np.zeros(n)
    entries = []
    if kind == 0:
        step = n // d
        groups = [np.arange(j, n, step)[:d] for j in range(step)]
    else:
        groups = [np.arange(j, j + d) for j in range(0, n, d)]
    for g in groups:
        err = np.sum((vq - vec[g][None, :]) ** 2, axis=1)
        err[~used] = np.inf
        e = int(np.argmin(err))
        entries.append(e)
        coded[g] = vq[e]
    return entries, coded


def encode_residue(w: BitWriter, res: Residue, books, vectors, skip, classify):
    """The residue data of `vectors` (the decoder's vectors: one interleaved vector for type 2), in the decoder's
    order: classification words in pass 0, then each partition's cascade.  classify(values) picks the class of a
    partition.  Returns the vectors as the decoder will rebuild them."""
    size = len(vectors[0])
    lb, le = min(res.begin, size), min(res.end, size)
    ps = res.partition_size
    parts = (le - lb) // ps if le > lb else 0
    out = [np.zeros(size) for _ in vectors]
    if not parts:
        return out
    cpw = books[res.classbook].dim
    cls = [[classify(v[lb + p * ps: lb + (p + 1) * ps]) for p in range(parts)] + [0] * cpw for v in vectors]
    for p in range(8):
        pc = 0
        while pc < parts:
            if p == 0:
                for j, v in enumerate(vectors):
                    if skip[j]:
                        continue
                    word = 0
                    for i in range(cpw):
                        word = word * res.classifications + cls[j][pc + i]
                    code, L = books[res.classbook].codes()[word]
                    w.code(code, L)
            i = 0
            while i < cpw and pc < parts:
                for j, v in enumerate(vectors):
                    if skip[j]:
                        continue
                    book = res.books[cls[j][pc]][p]
                    if book < 0:
                        continue
                    off = lb + pc * ps
                    target = v[off:off + ps] - out[j][off:off + ps]
                    ents, coded = quantise(target, books[book], 0 if res.type == 0 else 1)
                    for e in ents:
                        code, L = books[book].codes()[e]
                        w.code(code, L)
                    out[j][off:off + ps] += coded
                i += 1
                pc += 1
    return out


def encode(signal: np.ndarray, plan: Plan) -> bytes:
    """An Ogg Vorbis stream of signal [n] or [n, ch] under `plan`: trim_front zeros go before the signal and the first
    audio page's granule trims them; the last page's granule drops trim_end samples of the last block."""
    s = plan.setup
    x = signal.reshape(len(signal), -1).astype(np.float64)
    assert x.shape[1] == s.channels
    x = np.concatenate([np.zeros((plan.trim_front, s.channels)), x])
    flags = list(plan.flags)
    spectra, ns, ends = analysis(x, flags, s.bs)
    packets = []
    mode_of = {}
    for i, (bf, _) in enumerate(s.modes):
        mode_of.setdefault(bf, i)
    for k, bf in enumerate(flags):
        mode = mode_of[bf]
        m = s.mappings[s.modes[mode][1]]
        w = BitWriter()
        w.write(0, 1)
        w.write(mode, ilog(len(s.modes) - 1))
        if bf:
            w.write(flags[k - 1] if k > 0 else bf, 1)
            w.write(flags[k + 1] if k + 1 < len(flags) else bf, 1)
        n2 = ns[k] // 2
        X = np.stack(spectra[k])
        floors = []
        for c in range(s.channels):
            f = s.floors[m.submap_floor[m.mux[c] if m.mux else 0]]
            y = fit_floor(f, np.abs(X[c]), s.books)
            floors.append((f, y))
            encode_floor(w, f, y, s.books)
        curves = np.stack([Decoder.floor_curve(f, y, n2) for f, y in floors])
        R = X / curves
        for a, b in m.coupling:  # square-polar coupling in the residue domain
            l, r = R[a].copy(), R[b].copy()
            R[a] = np.where(l > r, np.where(l > 0, l, r), np.where(r > 0, r, np.where(l == r, r, l)))
            R[b] = np.where(l > r, np.where(l > 0, l - r, r - l), np.where(r > 0, l - r, np.where(l == r, r - l, r - l)))
        mux = m.mux or [0] * s.channels
        for sm in range(m.submaps):
            chans = [c for c in range(s.channels) if mux[c] == sm]
            res = s.residues[m.submap_residue[sm]]
            if res.type == 2:
                v = np.zeros(n2 * len(chans))
                for j, c in enumerate(chans):
                    v[j::len(chans)] = R[c]
                vecs = [v]
            else:
                vecs = [R[c] for c in chans]
            encode_residue(w, res, s.books, vecs, [False] * len(vecs), _classifier(res, s.books))
        packets.append(w.bytes())
    for k, keep in (plan.cut or {}).items():
        packets[k] = packets[k][:keep]
    total = ends[-1]
    gran = []
    for k in range(len(packets)):
        gran.append(ends[k] - plan.trim_front)
    if plan.trim_end:
        gran[-1] = total - plan.trim_front - plan.trim_end
    heads = [id_header(s), comment_header(), setup_header(s)]
    return ogg_stream(heads + packets, [0, 0, 0] + gran, page_bytes=plan.page_bytes,
                      packets_per_page=plan.packets_per_page)


def _classifier(res: Residue, books):
    """Class 0 when a partition is all near zero and class 0 has no books, else the last class."""
    def pick(vals):
        if all(b < 0 for b in res.books[0]) and np.max(np.abs(vals), initial=0) < 0.25:
            return 0
        return res.classifications - 1
    return pick


# ------------------------------------------------------------------------------------------------ ready-made setups


def standard_setup(channels=2, bs=(256, 2048), residue_type=2, lookup=1, sequence_p=0, ordered=False, sparse=False,
                   submaps=1, coupled=True, partition=16, mult=2, cascade=2, floor_posts=(), rate=44100):
    """A setup in the manner of libvorbis's: floor1 with a master book and a "no book" subclass, one residue with a
    coarse and a fine VQ book (cascade passes), square-polar coupling of channel pairs."""
    books = []
    # 0: floor master book over 2-bit subclass words of a 2-post class (subclass 0: no book, 1: book 1)
    books.append(Book(1, complete_lengths(16), ordered=ordered))
    # 1: floor Y values
    rng = RANGES[mult]
    books.append(Book(1, complete_lengths(rng)))
    # 2: residue classbook: 2 classes, 4 per word -> 16 entries
    books.append(Book(4, complete_lengths(16)))
    # 3: coarse VQ, 4: fine VQ
    if lookup == 1:
        books.append(lattice_book(2, 9, 2.0, sequence_p=sequence_p))
        books.append(lattice_book(2, 5, 0.5))
    else:
        vals = 9
        coarse = Book(2, complete_lengths(vals * vals), lookup=2, minimum=-8.0, delta=2.0, value_bits=4,
                      sequence_p=sequence_p, multiplicands=[v for e in range(vals * vals) for v in (e % vals, e // vals)])
        books.append(coarse)
        books.append(lattice_book(2, 5, 0.5))
    if sparse:  # the floor's Y book written sparse, with unused entries after the used ones
        books[1] = Book(1, complete_lengths(rng) + [0] * 5, sparse=True)
    n2 = bs[1] // 2
    rb = ilog(n2 - 1)
    xs = list(floor_posts) or sorted(set(int(v) for v in np.geomspace(2, n2 - 1, 14)) - {0, n2})
    if len(xs) % 2:
        xs = xs[:-1]
    fl = Floor1(partition_class=[0] * (len(xs) // 2), class_dim=[2], class_sub=[1], class_master=[0],
                sub_books=[[-1, 1]], multiplier=mult, rangebits=rb, xs=xs)
    # the floor's X values are in units of the long block's lines; short blocks use a floor of their own
    n2s = bs[0] // 2
    xs_s = sorted(set(int(v) for v in np.geomspace(2, n2s - 1, 6)) - {0, n2s})
    if len(xs_s) % 2:
        xs_s = xs_s[:-1]
    fl_s = Floor1(partition_class=[0] * (len(xs_s) // 2), class_dim=[2], class_sub=[1], class_master=[0],
                  sub_books=[[-1, 1]], multiplier=mult, rangebits=ilog(n2s - 1), xs=xs_s)
    passes = [3, 4] if cascade == 2 else [3]
    res = Residue(residue_type, 0, n2 * (channels if residue_type == 2 else 1), partition, 2, 2,
                  [[-1] * 8, [passes[p] if p < len(passes) else -1 for p in range(8)]])
    res_s = dataclasses.replace(res, end=n2s * (channels if residue_type == 2 else 1))
    coupling = [(c, c + 1) for c in range(0, channels - 1, 2)] if coupled else []
    mux = [c % submaps for c in range(channels)] if submaps > 1 else None
    m_long = Mapping(submaps, coupling, mux, [1] * submaps, [1] * submaps)
    m_short = Mapping(submaps, coupling, mux, [0] * submaps, [0] * submaps)
    return Setup(channels, rate, bs, books, [fl_s, fl], [res_s, res], [m_short, m_long], [(0, 0), (1, 1)])
