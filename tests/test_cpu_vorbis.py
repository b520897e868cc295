"""CPU tests of native Ogg Vorbis input: the reference against the Vorbis I specification's own examples, the transforms
and the encoder round trip, bt_debug_vorbis_decode_host against the float64 decoder of vorbis_reference.py on a
synthetic corpus, the probe's refusals, staging errors, corrupt streams and the kernels' SASS."""
import struct

import numpy as np
import pytest

import vorbis_reference as V
import vorbis_support as S
from beat_this_b200 import _lib
from support import sass


@pytest.fixture(scope="module")
def corpus(tmp_path_factory, lib_built):
    d = tmp_path_factory.mktemp("vorbis")
    out = []
    for name, data in S.corpus():
        p = d / f"{name}.ogg"
        p.write_bytes(data)
        out.append((str(p), data, V.decode(data)))
    return out


def test_codewords_of_the_specification_example():
    got = V.assign_codewords([2, 4, 4, 4, 4, 2, 3, 3])
    want = ["00", "0100", "0101", "0110", "0111", "10", "110", "111"]
    assert [format(c, f"0{L}b") for c, L in (got[e] for e in range(8))] == want
    with pytest.raises(ValueError):
        V.assign_codewords([1, 1, 1])  # over-full


def test_float32_unpack_and_lookup1_values():
    assert V.float32_unpack((788 << 21) | 1) == 1.0
    assert V.float32_unpack(0x80000000 | ((788 + 1) << 21) | 3) == -6.0
    assert V.float32_unpack((788 - 20) << 21 | (1 << 20)) == 1.0
    for entries, dim, want in ((81, 4, 3), (80, 4, 2), (25, 2, 5), (26, 2, 5), (1, 3, 1), (1000, 3, 10)):
        assert V.lookup1_values(entries, dim) == want


def test_single_used_entry_codebook(tmp_path, lib_built):
    """A book with one used entry: its codeword is the all-zero word of its length, and it decodes."""
    assert V.assign_codewords([0, 3, 0]) == {1: (0, 3)}
    setup = V.standard_setup(channels=1, coupled=False, residue_type=1)
    setup.books[1] = V.Book(1, [0] * 40 + [4] + [0] * 87)  # floor Y values: only entry 40 is codable
    data = V.encode(S.signal(6000, 1, 20), V.Plan(setup, S.flags(4, 20)))
    p = tmp_path / "single.ogg"
    p.write_bytes(data)
    want = V.decode(data).pcm[:, 0]
    got, st, _ = S.host_decode([str(p)])
    assert st == [0] and np.abs(got[0] - want).max() <= S.max_err(V.decode(data).l1)


@pytest.mark.parametrize("fl", [[1] * 6, [0] * 6, [1, 0, 1, 0, 0, 1, 1], [0, 1, 1, 0, 1, 0, 0]])
def test_mdct_imdct_and_overlap_add_rebuild_the_signal(fl):
    """The analysis MDCT under the Vorbis windows, then the decoder's IMDCT, windows and overlap-add: the signal again
    to float64 rounding (above 250 dB) across every window transition."""
    bs = (256, 2048)
    ns, ends = V.ends_of(fl, bs)
    x = np.random.default_rng(1).standard_normal((ends[-1] + 2048, 1))
    spectra, ns, ends = V.analysis(x, fl, bs)
    blocks = [V.imdct(spectra[k][0]) * V.window(n, fl[k], fl[k - 1] if k else fl[k], fl[k + 1] if k + 1 < len(fl)
                                                else fl[k], bs[0]) for k, n in enumerate(ns)]
    out = np.zeros(ends[-1])
    for k in range(1, len(ns)):
        na, nb = ns[k - 1], ns[k]
        d = np.arange(ends[k] - ends[k - 1])
        ia, ib = na // 2 + d, nb // 4 - na // 4 + d
        out[ends[k - 1]:ends[k]] = np.where(ia < na, blocks[k - 1][np.minimum(ia, na - 1)], 0) + np.where(
            ib >= 0, blocks[k][np.maximum(ib, 0)], 0)
    err = out - x[: ends[-1], 0]
    assert 10 * np.log10(np.sum(x[: ends[-1], 0] ** 2) / np.sum(err**2)) > 250


def test_imdct_is_the_specification_sum():
    X = np.random.default_rng(2).standard_normal(64)
    n, k = np.arange(128)[:, None], np.arange(64)[None, :]
    assert np.abs(np.cos(2 * np.pi / 128 * (n + 0.5 + 32) * (k + 0.5)) @ X - V.imdct(X)).max() < 1e-12


def test_encoded_signals_decode_above_the_quantiser_bound(corpus):
    """After the coarse and the fine pass a residue value within the coarse book's range is off by at most half the fine
    step (1/4) times the floor, and the floor follows the spectrum's local peak to within a factor of two, so the
    decoded signal keeps an SNR of at least 20 log10(1 / (1/4 x 2)) = 6 dB.  Streams where that premise does not hold
    are left out: cut packets, a single pass, and blocks of 8192 whose floor posts are too sparse for the fit."""
    for path, data, dec in corpus:
        if "cut" in path or "trim" in path or "one_pass" in path or "8192" in path:
            continue
        name = path.rsplit("/", 1)[-1][:-4]
        src = dict(S.corpus_signals())[name]
        n = min(len(dec.pcm), len(src))
        err = dec.pcm[:n] - src[:n]
        assert 10 * np.log10(np.sum(src[:n] ** 2) / np.sum(err**2)) > 6, name


def test_host_hook_against_the_float64_decoder(corpus):
    got, st, infos = S.host_decode([p for p, _, _ in corpus])
    assert st == [0] * len(corpus)
    for (path, data, dec), g, info in zip(corpus, got, infos):
        want = dec.pcm if dec.pcm.shape[1] > 1 else dec.pcm[:, 0]
        assert g.shape == want.shape, path
        assert info.skip == dec.skip
        assert np.abs(g - want).max() <= S.max_err(dec.l1), path
    mono, st, _ = S.host_decode([p for p, _, _ in corpus], _lib.BT_VORBIS_MONO_F32)
    for (path, data, dec), g in zip(corpus, mono):
        assert np.abs(g - dec.pcm.mean(axis=1)).max() <= S.max_err(dec.l1) + 2.0**-24, path


def test_trims_and_cut_files(corpus, tmp_path):
    by = {p.rsplit("/", 1)[-1][:-4]: (p, d, dec) for p, d, dec in corpus}
    p, data, dec = by["front_end_trim"]
    assert dec.skip == 700
    # a file cut inside its last page: the page is dropped, the output ends at the last whole page's granule
    cut = tmp_path / "cut.ogg"
    cut.write_bytes(data[:-100])
    code, info = S.probe(cut)
    want = V.decode(data[:-100])
    assert code == 0 and info.n_samples == len(want.pcm) < len(dec.pcm)
    got, st, _ = S.host_decode([str(cut)])
    assert st == [0] and np.abs(got[0] - want.pcm).max() <= S.max_err(want.l1)


def _pages(data):
    out, pos = [], 0
    while pos < len(data):
        nseg = data[pos + 26]
        size = 27 + nseg + sum(data[pos + 27:pos + 27 + nseg])
        out.append(bytearray(data[pos:pos + size]))
        pos += size
    return out


def _recrc(pg):
    pg[22:26] = b"\0\0\0\0"
    pg[22:26] = struct.pack("<I", V.ogg_crc(bytes(pg)))
    return pg


def test_refusals(tmp_path, corpus, lib_built):
    data = corpus[1][1]
    pages = _pages(data)
    setup = V.standard_setup()

    def refused(name, blob):
        p = tmp_path / name
        p.write_bytes(blob)
        assert S.probe(p)[0] == -6, name

    floor0 = V.Setup(**{**setup.__dict__, "floor_type": 0})
    refused("floor0.ogg", V.ogg_stream([V.id_header(setup), V.comment_header(), V.setup_header(floor0)], [0, 0, 0]))
    refused("opus.ogg", V.ogg_stream([b"OpusHead\x01\x02" + b"\0" * 9, b"OpusTags"], [0, 0]))
    refused("oggflac.ogg", V.ogg_stream([b"\x7fFLAC\x01\x00" + b"\0" * 40], [0]))
    other = V.ogg_stream([V.id_header(setup), V.comment_header(), V.setup_header(setup)], [0, 0, 0], serial=99)
    refused("chained.ogg", data + other)
    pg = _pages(other)[0]
    refused("multiplexed.ogg", bytes(pages[0]) + bytes(pg) + b"".join(bytes(p) for p in pages[1:]))
    nine = V.Setup(**{**setup.__dict__, "channels": 9})
    refused("nine.ogg", V.ogg_stream([V.id_header(nine), V.comment_header(), V.setup_header(setup)], [0, 0, 0]))
    bad = [bytearray(p) for p in pages]
    bad[1][40] ^= 0x10  # a header page that fails its CRC
    refused("header_crc.ogg", b"".join(bytes(p) for p in bad))
    refused("riff.ogg", b"RIFF" + data[4:])


def test_audio_page_crc_and_sequence_are_io_errors(tmp_path, corpus):
    data = corpus[1][1]
    pages = _pages(data)
    bad = [bytearray(p) for p in pages]
    bad[3][60] ^= 1  # an audio page's body: the probe takes it, staging refuses the file alone
    p1 = tmp_path / "crc.ogg"
    p1.write_bytes(b"".join(bytes(p) for p in bad))
    gap = [bytearray(p) for p in pages]
    for k in range(3, len(gap)):
        gap[k][18:22] = struct.pack("<I", k + 1)
        _recrc(gap[k])
    p2 = tmp_path / "gap.ogg"
    p2.write_bytes(b"".join(bytes(p) for p in gap))
    good = corpus[0][0]
    for p in (p1, p2):
        assert S.probe(p)[0] == 0
    infos = [S.probe(p)[1] for p in (good, p1, p2)]
    _, npk, _, _, status = S.stage([str(good), str(p1), str(p2)], infos)
    assert status == [0, -5, -5] and npk[1:] == [0, 0] and npk[0] > 0


def test_corrupted_streams_end_as_statuses(corpus):
    """Fixed byte flips in the staged packets and packet tables end as statuses or decodes, never as reads outside the
    staged data (the host hook runs the kernels' code under the same bounds)."""
    paths = [p for p, _, _ in corpus[:3]]
    rng = np.random.default_rng(7)
    for trial in range(6):
        def corrupt(buf, infos, npk, trial=trial):
            fo, status_at, bo, total = _lib.vorbis_layout(infos)
            if trial < 3:  # the packet bytes
                for _ in range(20):
                    buf[bo[0] + int(rng.integers(0, infos[0].packet_bytes))] ^= 1 << int(rng.integers(0, 8))
            elif trial == 3:  # a mode number past the modes
                buf[fo[0] * _lib.VORBIS_PACKET_BYTES + 28 + 5 * _lib.VORBIS_PACKET_BYTES] = 63
            elif trial == 4:  # a packet entry outside its stream
                e = np.frombuffer(buf, dtype=np.int64, count=1, offset=(fo[0] + 2) * _lib.VORBIS_PACKET_BYTES)
                e[0] = 1 << 40
            else:  # an entry out of step with the one before
                e = np.frombuffer(buf, dtype=np.int64, count=1, offset=(fo[0] + 4) * _lib.VORBIS_PACKET_BYTES + 8)
                e[0] += 1
        got, st, _ = S.host_decode(paths, corrupt=corrupt)
        assert st[1:] == [0, 0]
        if trial >= 3:
            assert st[0] == -5
        if st[0] != 0:
            assert not np.any(got[0])


def test_decode_kernels_have_no_local_memory(lib_built):
    fn = None
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
        elif fn and "vorbis_" in fn and ("LDL" in line or "STL" in line):
            pytest.fail(f"{fn} uses local memory: {line.strip()}")


def test_probe_audio_answers_vorbis(corpus):
    kinds = _lib.probe_audio([p for p, _, _ in corpus])
    assert [k for k, _ in kinds] == ["vorbis"] * len(corpus)
    assert kinds[0][1].n_samples == len(corpus[0][2].pcm)
