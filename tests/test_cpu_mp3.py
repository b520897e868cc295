"""CPU tests of native MP3 input: the code tables against a real encoder's stream, the probe and its refusals, the
staged frame tables, the decode kernels' machine code, and the decoder itself through its host test hook (the same
per-lane code the kernels run) against the float64 decoder of mp3_reference.py."""
import re
from fractions import Fraction

import numpy as np
import pytest

import mp3_reference as M
from beat_this_b200 import _lib
import mp3_support as S
from mp3_support import FIXTURE, N_FIXTURE, assert_close, host_decode, probe, stage, write
from support import sass


@pytest.fixture(scope="module")
def fixture_bytes():
    return open(FIXTURE, "rb").read()


@pytest.fixture(scope="module")
def fixture_pcm(fixture_bytes):
    return M.decode(fixture_bytes).pcm


# ---- tables -------------------------------------------------------------------------------------------------------
def test_code_tables_are_complete_prefix_codes():
    for t, (size, hl, hc) in M._H.items():
        assert len(hl) == len(hc) == size * size
        assert sum(Fraction(1, 2**l) for l in hl) == 1, t
        codes = sorted(format(c, f"0{l}b") for l, c in zip(hl, hc))
        assert all(not b.startswith(a) for a, b in zip(codes, codes[1:])), t
    for hl, hc in (M.COUNT1_A, M.COUNT1_B):
        assert sum(Fraction(1, 2**l) for l in hl) == 1


def test_tables_against_a_real_encoder(fixture_bytes):
    """Every granule of the fixture (all Huffman tables but 7 and 10; long, start, short and stop blocks, preflag and
    scalefac_scale): the Huffman data ends exactly at part2_3_length, or it fills the spectrum (no
    further count1 quadruple fits) and every bit after it up to part2_3_length is a 1 -- the encoder's stuffing, which
    decodes to nothing.  A wrong table entry desynchronises the walk and breaks this."""
    frames = M.frames_of(fixture_bytes)
    assert len(frames) == N_FIXTURE
    main, sides, starts = M.main_data_layout(fixture_bytes, frames)
    used = set()
    kinds = set()
    for f, si in enumerate(sides):
        bit = 8 * starts[f]
        for gr in range(2):
            for ch in range(2):
                g = si.gr[gr][ch]
                br = M.BitReader(main, bit)
                M.read_scalefactors(br, g, si.scfsi[ch], gr, {"l": [0] * 22})
                _, n = M.huffman_lines(br, g, bit + g.part2_3_length, 44100)
                end = bit + g.part2_3_length
                if br.pos != end:
                    assert n > 572 and all(M.BitReader(main, p).read(1) for p in range(br.pos, end))
                used.update(t for t in g.table_select[: 2 if g.window_switching else 3])
                used.add(32 + g.count1_table)
                kinds.update({("block", g.block_type), ("preflag", g.preflag), ("scale", g.scalefac_scale)})
                bit = end
    families = {t if t < 16 or t >= 32 else 16 if t < 24 else 24 for t in used}
    # every code table but 7 and 10, which the recording's encoder never chose (the prefix-code test covers them)
    assert families >= {0, 1, 2, 3, 5, 6, 8, 9, 11, 12, 13, 15, 16, 24, 32, 33}
    assert kinds >= {("block", b) for b in range(4)} | {("preflag", 1), ("scale", 1)}


# ---- the host hook against the float64 decoder ------------------------------------------------------------------
def test_host_hook_on_the_fixture(fixture_pcm):
    (out,), st, (info,) = host_decode([FIXTURE])
    assert st == [0] and info.n_samples == 1152 * N_FIXTURE and info.skip == 0
    assert_close(out, fixture_pcm)
    (mono,), st, _ = host_decode([FIXTURE], _lib.BT_MP3_MONO_F32)
    assert st == [0]
    want = ((out[:, 0] + out[:, 1]) / 2).astype(np.float32)
    assert np.array_equal(mono.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("mode_ext", [1, 2, 3], ids=["intensity", "mid_side", "mid_side_intensity"])
def test_host_hook_on_stereo_coding(tmp_path, fixture_bytes, mode_ext):
    """The fixture's frames with mid/side and / or intensity stereo switched on in their headers: valid streams whose
    second channel is then a side or an intensity-position channel."""
    frames = M.split_frames(fixture_bytes)[:60]
    data = b"".join(M.with_header(f, mode_ext=mode_ext) for f in frames)
    path = write(tmp_path, "s.mp3", data)
    (out,), st, _ = host_decode([path])
    assert st == [0]
    assert_close(out, M.decode(data).pcm)


def test_several_streams_in_one_call(tmp_path, fixture_bytes, fixture_pcm):
    frames = M.split_frames(fixture_bytes)
    a = write(tmp_path, "a.mp3", b"".join(frames[:40]))
    b = write(tmp_path, "b.mp3", b"".join(M.with_header(f, mode_ext=2) for f in frames[100:130]))
    outs, st, _ = host_decode([a, FIXTURE, b])
    assert st == [0, 0, 0]
    assert_close(outs[0], M.decode(b"".join(frames[:40])).pcm)
    assert_close(outs[1], fixture_pcm)


# ---- probe, containers and frame tables ---------------------------------------------------------------------------
def test_probe_and_frame_table_of_the_fixture(fixture_bytes):
    code, info = probe(FIXTURE)
    assert code == 0
    assert (info.sample_rate, info.channels, info.n_frames, info.gapless) == (44100, 2, N_FIXTURE, 0)
    assert info.frames_offset == 0 and info.frames_bytes == len(fixture_bytes)
    buf, nf, mb, status = stage([FIXTURE], [info])
    assert status == [0] and nf == [N_FIXTURE]
    fo, _, bo, _ = _lib.mp3_layout([info])
    table = (_lib.bt_mp3_frame * N_FIXTURE).from_buffer(buf, _lib.MP3_FRAME_BYTES * fo[0])
    main, sides, starts = M.main_data_layout(fixture_bytes, M.frames_of(fixture_bytes))
    assert mb == [len(main)] and buf[bo[0] : bo[0] + mb[0]].tobytes() == main
    for k, (off, h) in enumerate(M.frames_of(fixture_bytes)):
        assert table[k].main_start == starts[k] and table[k].first_sample == 1152 * k
        assert table[k].header == int.from_bytes(fixture_bytes[off : off + 4], "big")
        assert bytes(table[k].side_info) == fixture_bytes[off + 4 : off + 36]


def test_tags_junk_and_truncation(tmp_path, fixture_bytes, fixture_pcm):
    frames = M.split_frames(fixture_bytes)[:30]
    body = b"".join(frames)
    want = M.decode(body).pcm
    # false syncs: 128 kbit/s headers (417 bytes long) and a cut 320 kbit/s frame, none followed by a header at the
    # length it gives
    false_sync = b"\x00\xff\xfb\x90\x64" * 60 + frames[0][:400]
    cases = {
        "id3": M.id3v2(2000) + body,
        "id3_footer": M.id3v2(777, footer=True) + body,
        "junk": false_sync + body,
        "id3_junk": M.id3v2(100) + false_sync + body,
        "id3v1": body + M.id3v1(),
        "ape": body + M.apev2(),
        "ape_id3v1": body + M.apev2() + M.id3v1(),
        "trailing_junk": body + bytes(range(256)) * 3,
        "truncated": body + frames[30 % len(frames)][:500],
    }
    for name, data in cases.items():
        path = write(tmp_path, name + ".mp3", data)
        code, info = probe(path)
        assert code == 0 and info.n_frames == 30 and info.n_samples == 30 * 1152, name
        (out,), st, _ = host_decode([path])
        assert st == [0], name
        assert_close(out, want)


def test_lost_sync_is_malformed(tmp_path, fixture_bytes):
    frames = M.split_frames(fixture_bytes)[:30]
    data = b"".join(frames[:10]) + b"\x00" * 100 + b"".join(frames[10:])
    path = write(tmp_path, "lost.mp3", data)
    code, info = probe(path)
    assert code == 0 and info.n_frames == 10
    _, _, _, status = stage([path], [info])
    assert status == [-5]  # BT_ERR_IO


def test_gapless_trim(tmp_path, fixture_bytes):
    frames = M.split_frames(fixture_bytes)[:40]
    body = b"".join(frames)
    (full,), _, _ = host_decode([write(tmp_path, "plain.mp3", body)])
    for delay, padding in ((576, 1000), (1105, 0), (0, 1700)):
        path = write(tmp_path, f"g{delay}_{padding}.mp3", M.xing_frame(frames[0], 40, delay, padding) + body)
        code, info = probe(path)
        start, stop = delay + 529, min(1152 * 40, 1152 * 40 - padding + 529)
        assert code == 0 and info.gapless == 1 and info.n_frames == 40
        assert (info.skip, info.n_samples) == (start, stop - start)
        (out,), st, _ = host_decode([path])
        assert st == [0] and np.array_equal(out, full[start:stop])
    for name, xf in (("no_tag", M.xing_frame(frames[0], 40)), ("count", M.xing_frame(frames[0], 41, 576, 100)),
                     ("lavc", M.xing_frame(frames[0], 40, 0, 0, b"Lavc61.3"))):
        code, info = probe(write(tmp_path, name + ".mp3", xf + body))
        assert code == 0 and info.n_frames == 40
        trimmed = name == "lavc"
        assert info.gapless == int(trimmed) and info.n_samples == (1152 * 40 - 529 if trimmed else 1152 * 40)


def test_refusals(tmp_path, fixture_bytes):
    frames = M.split_frames(fixture_bytes)[:20]
    bad = {
        "mpeg2": b"".join(M.with_header(f, version=2) for f in frames),
        "mpeg25": b"".join(M.with_header(f, version=0) for f in frames),
        "layer2": b"".join(M.with_header(f, layer=2) for f in frames),
        "layer1": b"".join(M.with_header(f, layer=3) for f in frames),
        "free_format": b"".join(M.with_header(f, bitrate_index=0) for f in frames),
        "bitrate15": b"".join(M.with_header(f, bitrate_index=15) for f in frames),
        "reserved_rate": b"".join(M.with_header(f, rate_index=3) for f in frames),
        "empty": b"",
        "noise": np.random.default_rng(0).integers(0, 256, 50000, dtype=np.uint8).tobytes(),
    }
    for name, data in bad.items():
        assert probe(write(tmp_path, name + ".mp3", data))[0] == -6, name
    # the rate changes between frames: 44.1 kHz frames, then a 48 kHz frame (length 960 bytes at 320 kbit/s)
    f48 = M.with_header(frames[5], rate_index=1)[:960]
    assert probe(write(tmp_path, "rate_change.mp3", b"".join(frames[:5]) + f48 + b"".join(frames[6:])))[0] == -6
    assert probe(tmp_path / "missing.mp3")[0] == -5


def test_probe_audio_keeps_its_answers(tmp_path, fixture_bytes):
    import flac_reference as F
    import flac_support as FS

    v = FS.signal(3000, 2, 16, 1)
    flac = write(tmp_path, "a.flac", F.encode(v, 44100, 16, 1024).data)
    wav = write(tmp_path, "a.wav", F.wav_twin(v, 44100, 16))
    junk = write(tmp_path, "a.bin", bytes(range(256)) * 40)
    mp3 = write(tmp_path, "a.mp3", fixture_bytes)
    kinds = [k for k, _ in _lib.probe_audio([wav, flac, junk, mp3])]
    assert kinds == ["wav", "flac", None, "mp3"]
    # neither WAV nor FLAC is claimed by the MP3 probe
    assert probe(wav)[0] == -6 and probe(flac)[0] == -6 and probe(junk)[0] == -6


def test_corrupted_streams_end_as_statuses(tmp_path, fixture_bytes):
    """A fixed set of byte flips and truncations in side info and main data: each stream decodes or ends as BT_ERR_IO,
    never reading outside its buffers (the host hook bounds every read as the kernels do)."""
    frames = M.split_frames(fixture_bytes)[:12]
    body = bytearray(b"".join(frames))
    rng = np.random.default_rng(7)
    paths = []
    for k in range(24):
        data = bytearray(body)
        f = int(rng.integers(0, 12))
        at = 1044 * f + (4 + int(rng.integers(0, 32)) if k % 2 == 0 else 36 + int(rng.integers(0, 1000)))
        data[at] ^= 1 << int(rng.integers(0, 8))
        paths.append(write(tmp_path, f"c{k}.mp3", bytes(data)))
    outs, st, _ = host_decode(paths)
    for out, s in zip(outs, st):
        assert s in (0, -5)
        assert np.all(np.isfinite(out))
        if s != 0:
            assert not np.any(out)

    # frame tables that point outside their stream, and main data cut short: statuses, zero output
    def cut(buf, infos, nf, mb):
        fo = _lib.mp3_layout(infos)[0]
        t = (_lib.bt_mp3_frame * nf[0]).from_buffer(buf, _lib.MP3_FRAME_BYTES * fo[0])
        t[3].main_start = mb[0] + 10
        t[5].main_start = -10**6  # before the 511 bytes the reservoir can reach: outside the stream, not a cut
        t1 = (_lib.bt_mp3_frame * nf[1]).from_buffer(buf, _lib.MP3_FRAME_BYTES * fo[1])
        t1[2].side_info[0] = 0xFF  # main_data_begin is not read from the table: the start is; part2_3 of granule 0:
        t1[2].side_info[2] = 0xFF  # 4095 bits, past the stream's end in the last frames
        mb[2] = 100
    outs, st, _ = host_decode([write(tmp_path, "x0.mp3", bytes(body)), write(tmp_path, "x1.mp3", bytes(body)),
                               write(tmp_path, "x2.mp3", bytes(body))], corrupt=cut)
    assert st[0] == -5 and st[2] == -5 and not np.any(outs[0]) and not np.any(outs[2])
    assert st[1] in (0, -5)


def test_decode_kernels_have_no_local_memory(lib_built):
    names = ("mp3_granules_kernel", "mp3_hybrid_kernel", "mp3_synth_kernel")
    found, fn = set(), None
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
            hit = [n for n in names if n in fn]
            fn = hit[0] if hit else None
            if fn:
                found.add(fn)
        elif fn and re.search(r"\b(STL|LDL)(\.\w+)*\b", line):
            pytest.fail(f"{fn} uses local memory: {line.strip()}")
    assert found == set(names)


# ---- the analysis side: encoder round trips -------------------------------------------------------------------------
DELAY = 481 + 576  # the polyphase pair's delay (511 - 31 + 1) plus one granule of the hybrid (MDCT) pair
PATTERNS = {"long": [S.G()], "short": [S.G(block_type=2)], "mixed": [S.G(block_type=2, mixed=1)], "switch": S.SWITCH}


def _snr(y, x):
    n = len(x) - DELAY - 1152
    e = y[DELAY : DELAY + n] - x[:n]
    return 10 * np.log10(np.sum(x[:n] ** 2) / np.sum(e**2))


@pytest.mark.parametrize("pattern", list(PATTERNS))
def test_filterbanks_invert_each_other(pattern):
    """The encoder's analysis filter bank, MDCT and forward butterflies against the decoder's transforms (no
    quantisation): the signal returns at DELAY.  The polyphase pair of the standard is not a perfect reconstruction
    bank; its own error is below -80 dB, and every block pattern (window shapes, short-block order, mixed blocks,
    alias butterflies, frequency inversion) adds nothing to it."""
    x = S.signal(1152 * 8, 1, 20)
    Sb = np.concatenate([np.zeros((18, 32)), M.analysis(x)])
    specs = PATTERNS[pattern]
    n_gr = len(x) // 576
    blocks = np.zeros((n_gr + 1, 32, 36))
    for gi in range(n_gr):
        sp = specs[gi % len(specs)]
        g = M.Granule(window_switching=int(sp.block_type != 0), block_type=sp.block_type, mixed=sp.mixed)
        xr = M.forward_hybrid(Sb[18 * gi : 18 * gi + 18], Sb[18 * gi + 18 : 18 * gi + 36], g, 44100)
        blocks[gi + 1] = M.imdct(M.alias(M.reorder(xr, g, 44100), g), g)
    sub = blocks[1:, :, :18] + blocks[:-1, :, 18:]
    sub[:, 1::2, 1::2] *= -1
    y = M.synthesize(sub.transpose(0, 2, 1).reshape(-1, 32))
    assert _snr(y, x) >= 80


def _unit_energy(short: bool) -> float:
    """Output energy of one unit line of one granule through the decoder's transforms (the same for every line up to
    the polyphase bank's ripple; the largest of a spread of lines is taken)."""
    g = M.Granule(window_switching=int(short), block_type=2 if short else 0)
    best = 0.0
    for k in (0, 7, 100, 301, 575):
        xr = np.zeros(576)
        xr[k] = 1.0
        blocks = np.zeros((3, 32, 36))
        blocks[1] = M.imdct(M.alias(M.reorder(xr, g, 44100), g), g)
        sub = blocks[1:, :, :18] + blocks[:-1, :, 18:]
        sub[:, 1::2, 1::2] *= -1
        best = max(best, float(np.sum(M.synthesize(sub.transpose(0, 2, 1).reshape(-1, 32)) ** 2)))
    return best


@pytest.mark.parametrize("pattern, ms", [(p, False) for p in PATTERNS] + [("switch", True), ("long", True)])
def test_encoded_signal_returns_at_a_fixed_delay(pattern, ms):
    """Encode a known signal, decode it with the float64 decoder: it returns at DELAY within a stated SNR bound.
    Bound: rounding a line to is changes it by at most gain * ((|is| + 1/2)^(4/3) - |is|^(4/3)) = d; the
    transforms map independent line errors to output energy at most E_unit (per long or short line, measured on
    unit lines) times sum d^2; the polyphase bank's own error adds at most 1e-8 of the signal energy (the test
    above).  M/S is a rotation and changes none of it."""
    x = S.signal(1152 * 10, 2 if ms else 1, 21)
    data, _ = M.encode(x, 44100, PATTERNS[pattern], ms=ms, max_is=60)
    dec = M.decode(data)
    xs = x if x.ndim == 2 else x[:, None]
    e_long, e_short = _unit_energy(False), _unit_energy(True)
    noise = 0.0
    for fl, fg, fs in zip(dec.lines, dec.gains, dec.short):
        for gl, gg, gs in zip(fl, fg, fs):
            for q, gain, sh in zip(gl, gg, gs):
                a = np.abs(q).astype(np.float64)
                d = gain * ((a + 0.5) ** (4 / 3) - a ** (4 / 3))
                noise += e_long * np.sum(d[~sh] ** 2) + e_short * np.sum(d[sh] ** 2)
    signal_energy = float(np.sum(xs[: len(xs) - DELAY - 1152] ** 2))
    bound = 10 * np.log10(signal_energy / (noise + 1e-8 * signal_energy))
    assert bound > 12  # the quantiser chosen (after the rate loop) leaves a meaningful bound
    for c in range(xs.shape[1]):
        assert _snr(dec.pcm[:, c], xs[:, c]) >= bound


# ---- synthetic streams through the host hook --------------------------------------------------------------------
@pytest.fixture(scope="module")
def synthetic():
    return S.variants()


def test_synthetic_streams_have_their_features(synthetic):
    v = dict(synthetic)
    side = {}
    for name, data in synthetic:
        fr = M.frames_of(data)
        main, sides, starts = M.main_data_layout(data, fr)
        side[name] = (fr, sides)
    fr, sides = side["reservoir_511"]
    assert max(si.main_data_begin for si in sides) == 511
    fr, _ = side["reservoir_vbr"]
    assert len({h.bitrate for _, h in fr}) > 3
    assert all(h.crc for _, h in side["mono_switch_crc"][0]) and all(h.channels == 1 for _, h in side["mono_long"][0])
    assert {fr[0][1].sample_rate for fr, _ in side.values()} == {32000, 44100, 48000}
    gs = [g for _, sides in side.values() for si in sides for row in si.gr for g in row]
    assert any(g.mixed for g in gs) and any(max(g.subblock_gain) for g in gs) and any(g.preflag for g in gs)
    assert any(sum(sum(s) for s in si.scfsi) for si in side["scfsi"][1])
    assert any(fr[0][1].mode_ext == 2 for fr, _ in side.values())
    used = {t for g in gs for t in g.table_select[: 2 if g.window_switching else 3] if g.big_values}
    assert {2, 3, 5, 6, 7, 8, 9, 10, 11, 12, 13, 15} <= used and any(t >= 16 for t in used)
    assert len(v) == len(synthetic)


def test_host_hook_on_synthetic_streams(tmp_path, synthetic):
    paths = [write(tmp_path, f"{name}.mp3", data) for name, data in synthetic]
    outs, st, infos = host_decode(paths)
    assert st == [0] * len(paths)
    for (name, data), out in zip(synthetic, outs):
        want = M.decode(data).pcm
        assert_close(out, want if want.shape[1] > 1 else want[:, 0])


def test_a_stream_cut_inside_the_reservoir(tmp_path, synthetic):
    """The reservoir stream without its first two frames: the granules whose main data lay in them decode as zeros,
    the rest as the float64 decoder gives them."""
    frames = M.split_frames(dict(synthetic)["reservoir_511"])
    data = b"".join(frames[2:])
    main, sides, starts = M.main_data_layout(data, M.frames_of(data))
    assert starts[0] < 0
    (out,), st, _ = host_decode([write(tmp_path, "cut.mp3", data)])
    assert st == [0]
    assert_close(out, M.decode(data).pcm)


def test_streams_that_are_not_decoded_are_zero_filled(tmp_path, fixture_bytes):
    """A file whose staging failed (lost sync: no frames) and one marked bad on entry get zeros over their whole
    output, not what the buffer held."""
    frames = M.split_frames(fixture_bytes)
    good = write(tmp_path, "good.mp3", b"".join(frames[:20]))
    lost = write(tmp_path, "lost.mp3", b"".join(frames[:10]) + bytes(100) + b"".join(frames[10:20]))
    outs, st, infos = host_decode([good, lost, good])
    assert st == [0, -5, 0] and infos[1].n_samples == 10 * 1152
    assert np.array_equal(outs[1], np.zeros_like(outs[1])) and np.all(np.isfinite(outs[0]))

    outs2, st2, _ = host_decode([good, good], preset_status=[0, -5])
    assert st2 == [0, -5] and not np.any(outs2[1]) and np.array_equal(outs2[0], outs[0])
