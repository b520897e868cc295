"""Generate tests/golden/kings_of_swing_383.mp3: the first 383 frames (about 10 s) of the recording the reference's own
inference test decodes (tests/It Don't Mean A Thing - Kings of Swing.mp3 in the reference's source tree).

    BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_mp3.py

The recording is MPEG-1 Layer III, 320 kbit/s CBR at 44.1 kHz, joint stereo, without CRC or a Xing / LAME frame, and
main_data_begin is 0 in every frame, so any run of whole frames is a valid stream.  The frames are cut by walking the
headers from the first byte (the file has no ID3v2 tag): every frame is 144000 * bitrate / rate + padding bytes.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
N_FRAMES = 383


def main():
    ref = os.environ.get("BEAT_THIS_REFERENCE")
    if not ref:
        sys.exit("usage: BEAT_THIS_REFERENCE=<beat_this source tree> python oracle/make_golden_mp3.py")
    data = open(os.path.join(ref, "tests", "It Don't Mean A Thing - Kings of Swing.mp3"), "rb").read()
    pos = 0
    for _ in range(N_FRAMES):
        h = int.from_bytes(data[pos : pos + 4], "big")
        assert h >> 21 == 0x7FF and (h >> 19) & 3 == 3 and (h >> 17) & 3 == 1, "not an MPEG-1 Layer III header"
        kbps = [0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320][(h >> 12) & 15]
        rate = [44100, 48000, 32000][(h >> 10) & 3]
        pos += 144000 * kbps // rate + ((h >> 9) & 1)
    out = os.path.join(ROOT, "tests", "golden", "kings_of_swing_383.mp3")
    with open(out, "wb") as f:
        f.write(data[:pos])
    print(f"wrote {out}: {N_FRAMES} frames, {pos} bytes")


if __name__ == "__main__":
    main()
