"""The device DBN post-processor (bt_dbn_track_device, bt_debug_dbn_viterbi; csrc/kernels_dbn.cu) against the host C++
tracker it restates (bt_dbn_track, bt_dbn_viterbi; csrc/dbn_host.cpp), which tests/test_cpu_host.py ties to a dense
brute-force Viterbi and to madmom's documented known answers.  The device decoder does the host's arithmetic operation
for operation, so everything below is compared for equality, not within a tolerance."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

REF = dict(min_interval=60.0 * 50 / 215.0, max_interval=60.0 * 50 / 55.0)  # the reference's 14..55 frames at 50 fps


@pytest.fixture(scope="module")
def eng(lib_built):
    from beat_this_b200.engine import Engine

    return Engine.mel_only("cuda:0")  # a weight-less context, as Postprocessor uses


def _bar_models():
    from beat_this_b200.dbn import _BarModel

    return {
        "3/4 ref": _BarModel(3, REF["min_interval"], REF["max_interval"], None, 100, 16),
        "4/4 ref": _BarModel(4, REF["min_interval"], REF["max_interval"], None, 100, 16),
        "4/4 num_tempi=20": _BarModel(4, REF["min_interval"], REF["max_interval"], 20, 100, 16),
        "3/4 fps10": _BarModel(3, 60.0 * 10 / 215.0, 60.0 * 10 / 55.0, None, 100, 16),
        "4/4 fps10": _BarModel(4, 60.0 * 10 / 215.0, 60.0 * 10 / 55.0, None, 100, 16),
    }


def _host_viterbi(lib, m, dens):
    dens = np.ascontiguousarray(dens, dtype=np.float64)
    iv = np.ascontiguousarray(m.intervals, dtype=np.int32)
    lt = np.ascontiguousarray(m.log_tempo, dtype=np.float64)
    pt = np.ascontiguousarray(m.pointers, dtype=np.int32)
    path = np.empty(len(dens), dtype=np.int64)
    logp = ctypes.c_double()
    code = lib.bt_dbn_viterbi(dens.ctypes.data, len(dens), m.beats, len(iv), iv.ctypes.data, lt.ctypes.data, pt.ctypes.data,
                              path.ctypes.data, ctypes.byref(logp))
    assert code == 0
    return path, logp.value


def _densities(m, kind, T, rng):
    if kind == "constant":  # every path through the same tempo ties exactly: exercises both tie-breaks
        return m.log_densities(np.full((T, 2), 0.1))
    act = rng.uniform(0.002, 0.3, (T, 2))
    act[rng.random(T) < 0.05] = (0.8, 0.05)
    act[rng.random(T) < 0.02] = (0.05, 0.8)
    return m.log_densities(act)


@pytest.mark.parametrize("T", [1, 2, 40, 1501, 15000])
def test_device_viterbi_equals_host_bitwise(eng, T):
    rng = np.random.default_rng(T)
    for name, m in _bar_models().items():
        for kind in ("random", "constant"):
            dens = _densities(m, kind, T, rng)
            ref_path, ref_logp = _host_viterbi(eng.lib, m, dens)
            path, logp = eng.debug_dbn_viterbi(torch.from_numpy(dens).cuda(), m.beats, m.intervals, m.log_tempo, m.pointers)
            assert np.array_equal(path, ref_path), (name, kind, T, int(np.argmax(path != ref_path)))
            assert logp == ref_logp, (name, kind, T, logp, ref_logp)  # bitwise: the same adds in the same order


def test_device_viterbi_rejects_other_pointer_forms(eng):
    from beat_this_b200._lib import BTError

    m = _bar_models()["4/4 fps10"]
    pt = m.pointers.copy()
    pt[m.first_states[1, 3] + 2] = 1  # a (down)beat observation after a "no beat" position
    dens = torch.zeros((5, 3), dtype=torch.float64, device="cuda:0")
    with pytest.raises(BTError, match="leading run"):
        eng.debug_dbn_viterbi(dens, m.beats, m.intervals, m.log_tempo, pt)


def _pulse_pieces(rng):
    """The pieces of test_native_dbn_cxx_tracker_equals_numpy_twin: noisy pulse trains, silence, one frame, frame 0 only."""
    pieces = []
    for period, meter, T in ((23.7, 4, 900), (31.2, 3, 700), (17.0, 4, 400)):
        pieces.append(_pulse_train(rng, period, meter, T))
    only0 = np.full((50, 2), 0.001)
    only0[0, 0] = 0.9
    return pieces + [np.full((120, 2), 0.001), np.full((1, 2), 0.4), only0]


def _pulse_train(rng, period, meter, T):
    act = rng.uniform(0.001, 0.08, (T, 2))
    f, k = rng.uniform(0, period), 0
    while f < T:
        act[int(f)] = (0.05, 0.7) if k % meter == 0 else (0.75, 0.03)
        f += period * (1 + 0.02 * rng.standard_normal())
        k += 1
    return act


def _meter_pieces():
    """The 120-BPM 4/4 and 90-BPM 3/4 impulse trains of test_native_dbn_tracks_synthetic_meters."""
    a = np.full((1000, 2), 0.01)
    for k, f in enumerate(range(110, 900, 25)):
        a[f, 1 if k % 4 == 0 else 0] = 0.9
    b = np.full((1000, 2), 0.01)
    for k in range(29):
        b[int(round(7 + k * 100 / 3)), 1 if k % 3 == 0 else 0] = 0.8
    return [a, b]


def _ragged_pieces(rng, n=64):
    lens = np.r_[1, 15000, 2, rng.integers(1, 15001, n - 3)]
    out = []
    for i, T in enumerate(lens):
        if i % 9 == 4:
            out.append(np.full((T, 2), 0.002))  # silence: below the threshold everywhere
        else:
            out.append(_pulse_train(rng, rng.uniform(14, 56), (3, 4)[i % 2], int(T)))
    return out


def _device_track(eng, trk, pieces):
    fo = np.zeros(len(pieces) + 1, dtype=np.int64)
    fo[1:] = np.cumsum([len(p) for p in pieces])
    act = torch.from_numpy(np.concatenate(pieces).astype(np.float64)).cuda().contiguous()
    return eng.dbn_cat(None, None, fo.tolist(), trk.track_params, activations=act)


def _assert_same(got, ref, what):
    assert len(got) == len(ref)
    for i, ((gb, gd), r) in enumerate(zip(got, ref)):
        rb, rd = r[:, 0], r[r[:, 1] == 1][:, 0]
        assert gb.dtype == np.float64 and np.array_equal(gb, rb) and np.array_equal(gd, rd), (what, i, len(gb), len(rb))


@pytest.mark.parametrize("kw", [{}, {"num_tempi": 20}, {"correct": False}], ids=["default", "num_tempi20", "nocorrect"])
def test_device_tracker_equals_host_on_activations(eng, kw):
    from beat_this_b200.dbn import DBNDownBeatTracker

    rng = np.random.default_rng(4)
    trk = DBNDownBeatTracker(**kw)
    pieces = _pulse_pieces(rng) + _meter_pieces() + _ragged_pieces(rng)
    ref = trk.batch(pieces)
    got = _device_track(eng, trk, pieces)
    _assert_same(got, ref, kw)
    assert len(got[0][0]) > 15 and len(got[3][0]) == 0 and len(got[5][0]) == 0
    n_beats = sum(len(g[0]) for g in got)
    print(f"{kw}: {len(pieces)} pieces, {n_beats} beats, identical to bt_dbn_track")
    again = _device_track(eng, trk, pieces)
    for (a, b), (c, d) in zip(got, again):
        assert np.array_equal(a, c) and np.array_equal(b, d)


def _logits(rng, T, period):
    x = rng.normal(-4.0, 1.5, T)
    d = rng.normal(-6.0, 1.5, T)
    f, k = rng.uniform(0, period), 0
    while f < T:
        x[int(f)] += rng.uniform(6, 10)
        if k % 4 == 0:
            d[int(f)] += rng.uniform(6, 10)
        f += period
        k += 1
    return x.astype(np.float32), d.astype(np.float32)


def test_postprocessor_device_equals_native_on_logits(eng):
    from beat_this_b200.postprocessor import Postprocessor

    rng = np.random.default_rng(11)
    dev = Postprocessor("dbn", engine=eng, dbn_impl="device")
    nat = Postprocessor("dbn", engine=eng, dbn_impl="native")
    b, d = _logits(rng, 1500, 24.5)
    bt, dt = (torch.from_numpy(v).cuda() for v in (b, d))
    g, r = dev(bt, dt), nat(bt, dt)
    assert len(g[0]) > 20 and np.array_equal(g[0], r[0]) and np.array_equal(g[1], r[1])
    B, T = 5, 1200
    pairs = [_logits(rng, T, p) for p in (15.0, 21.3, 30.0, 44.0, 52.5)]
    bb = torch.from_numpy(np.stack([p[0] for p in pairs])).cuda()
    db = torch.from_numpy(np.stack([p[1] for p in pairs])).cuda()
    mask = torch.ones((B, T), dtype=torch.bool, device="cuda")
    for i, n in enumerate((1200, 1000, 37, 1, 700)):
        mask[i, n:] = False
    for pm in (None, mask):
        g, r = dev(bb, db, pm), nat(bb, db, pm)
        for k in range(2):
            assert len(g[k]) == B and all(np.array_equal(u, v) for u, v in zip(g[k], r[k])), pm is None
    # batch_host on host logits uploads them and runs the same kernels
    fo = [0, 1500, 1500 + 900]
    hb = np.concatenate([b, pairs[0][0][:900]])
    hd = np.concatenate([d, pairs[0][1][:900]])
    for (gb, gd), (rb, rd) in zip(dev.batch_host(hb, hd, fo), nat.batch_host(hb, hd, fo)):
        assert np.array_equal(gb, rb) and np.array_equal(gd, rd)


def test_errors_before_any_launch(eng):
    from beat_this_b200._lib import BTError
    from beat_this_b200.dbn import DBNDownBeatTracker

    act = torch.full((100, 2), 0.1, dtype=torch.float64, device="cuda:0")
    before = eng.launches
    ref = DBNDownBeatTracker().track_params
    too_many = dict(ref, min_bpm=5.0, num_tempi=0)  # every interval of 14..600 frames: 587 tempi
    with pytest.raises(BTError, match="255"):
        eng.dbn_cat(None, None, [0, 100], too_many, activations=act)
    too_big = dict(ref, min_bpm=5.0)  # 60 log-spaced tempi of up to 600 frames per beat
    with pytest.raises(BTError, match="shared memory"):
        eng.dbn_cat(None, None, [0, 100], too_big, activations=act)
    assert eng.launches == before


def _clips():
    from beat_this_b200 import synthetic

    secs = [30.0] * 66 + [0.5, 2.0, 7.3, 45.0, 1.2]
    return [synthetic.synth_clip(200 + i, s) for i, s in enumerate(secs)]


@pytest.mark.parametrize("float16", [False, True])
def test_audio2beats_device_dbn_equals_native(small0_ckpt, float16):
    """Clips over more than one group (64 clips of 30 s fill one), short ones included."""
    from beat_this_b200.inference import Audio2Beats, load_model

    model = load_model(small0_ckpt, "cuda:0", float16)
    dev = Audio2Beats.from_model(model, dbn=True, dbn_impl="device")
    nat = Audio2Beats.from_model(model, dbn=True, dbn_impl="native")
    clips = _clips()
    g = dev.batch(clips, 22050)
    assert dev.pipeline.stats["groups"] >= 2
    r = nat.batch(clips, 22050)
    for i, ((gb, gd), (rb, rd)) in enumerate(zip(g, r)):
        assert np.array_equal(gb, rb) and np.array_equal(gd, rd), (float16, i, len(gb), len(rb))
    assert sum(len(x[0]) for x in g) > 1000
    again = dev.batch(clips, 22050)  # bitwise repeatable
    assert all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(g, again))
    sub = [64, 3, 70, 66, 67]  # other groupings: a different batch, and one clip per call
    for i, (sb, sd) in zip(sub, dev.batch([clips[i] for i in sub], 22050)):
        assert np.array_equal(sb, g[i][0]) and np.array_equal(sd, g[i][1])
    for i in (66, 68):
        sb, sd = dev(clips[i], 22050)
        assert np.array_equal(sb, g[i][0]) and np.array_equal(sd, g[i][1])


def test_file2beats_and_cli_device_dbn(small0_ckpt, tmp_path):
    from scipy.io import wavfile

    from beat_this_b200 import cli, synthetic
    from beat_this_b200.inference import File2Beats

    src = tmp_path / "in"
    (src / "sub").mkdir(parents=True)
    paths = []
    for i, secs in enumerate((30.0, 6.5, 1.0, 12.0)):
        x = synthetic.synth_clip(300 + i, secs)
        p = src / ("sub" if i % 2 else ".") / f"c{i}.wav"
        wavfile.write(p, 22050, np.round(x * 32767).astype(np.int16))
        paths.append(p)
    dev = File2Beats(small0_ckpt, "cuda:0", dbn=True, dbn_impl="device").batch(paths)
    nat = File2Beats(small0_ckpt, "cuda:0", dbn=True, dbn_impl="native").batch(paths)
    for (gb, gd), (rb, rd) in zip(dev, nat):
        assert np.array_equal(gb, rb) and np.array_equal(gd, rd)
    outs = {}
    for impl in ("device", "native"):
        out = tmp_path / impl
        assert cli.main([str(src), "-o", str(out), "--model", small0_ckpt, "--dbn", "--dbn-impl", impl]) == 0
        outs[impl] = {p.relative_to(out): p.read_bytes() for p in sorted(out.rglob("*.beats"))}
    assert len(outs["device"]) == 4 and outs["device"] == outs["native"]
