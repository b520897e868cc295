"""MPEG-1 Layer III written from ISO/IEC 11172-3, for the MP3 tests: a float64 decoder (the oracle of the device
decoder), and the analysis side as an encoder and bitstream writer (polyphase analysis, MDCT of every block type,
forward alias butterflies, M/S, quantisation with chosen side info, Huffman coding, frame packing with the bit
reservoir, CBR or VBR, CRC), plus tag, junk and Xing-frame writers, so that every feature the native decoder takes can
be produced on demand and the decoder's transforms can be held to the analysis side.

The Huffman code tables are the standard's Table 3-B.7 as (hlen, hcod) rows of x, y; the synthesis window is Table
3-B.3, whose coefficients are multiples of 2^-16 (stored here as those integers, D[0 .. 256]; the rest follow from the
window's symmetry)."""
from __future__ import annotations

import dataclasses
import math

import numpy as np

# ------------------------------------------------------------------------------------------------ tables
BITRATES = [0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320]  # kbit/s, index 0: free format
RATES = [44100, 48000, 32000]

SFB_LONG = {  # scalefactor band widths, long blocks
    44100: [4, 4, 4, 4, 4, 4, 6, 6, 8, 8, 10, 12, 16, 20, 24, 28, 34, 42, 50, 54, 76, 158],
    48000: [4, 4, 4, 4, 4, 4, 6, 6, 6, 8, 10, 12, 16, 18, 22, 28, 34, 40, 46, 54, 54, 192],
    32000: [4, 4, 4, 4, 4, 4, 6, 6, 8, 10, 12, 16, 20, 24, 30, 38, 46, 56, 68, 84, 102, 26],
}
SFB_SHORT = {  # per window, short blocks
    44100: [4, 4, 4, 4, 6, 8, 10, 12, 14, 18, 22, 30, 56],
    48000: [4, 4, 4, 4, 6, 6, 10, 12, 14, 16, 20, 26, 66],
    32000: [4, 4, 4, 4, 6, 8, 12, 16, 20, 26, 34, 42, 12],
}
PRETAB = [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 3, 2, 0]
SLEN = [(0, 0), (0, 1), (0, 2), (0, 3), (3, 0), (1, 1), (1, 2), (1, 3), (2, 1), (2, 2), (2, 3), (3, 1), (3, 2), (3, 3),
        (4, 2), (4, 3)]
ALIAS_C = [-0.6, -0.535, -0.33, -0.185, -0.095, -0.041, -0.0142, -0.0037]

# D[i] * 65536 for i = 0 .. 256 (Table 3-B.3)
SYNTH_WINDOW_HALF = [
    0, -1, -1, -1, -1, -1, -1, -2, -2, -2, -2, -3, -3, -4, -4, -5, -5, -6, -7, -7, -8, -9, -10, -11, -13, -14, -16, -17,
    -19, -21, -24, -26, -29, -31, -35, -38, -41, -45, -49, -53, -58, -63, -68, -73, -79, -85, -91, -97, -104, -111,
    -117, -125, -132, -139, -147, -154, -161, -169, -176, -183, -190, -196, -202, -208, 213, 218, 222, 225, 227, 228,
    228, 227, 224, 221, 215, 208, 200, 189, 177, 163, 146, 127, 106, 83, 57, 29, -2, -36, -72, -111, -153, -197, -244,
    -294, -347, -401, -459, -519, -581, -645, -711, -779, -848, -919, -991, -1064, -1137, -1210, -1283, -1356, -1428,
    -1498, -1567, -1634, -1698, -1759, -1817, -1870, -1919, -1962, -2001, -2032, -2057, -2075, -2085, -2087, -2080,
    -2063, 2037, 2000, 1952, 1893, 1822, 1739, 1644, 1535, 1414, 1280, 1131, 970, 794, 605, 402, 185, -45, -288, -545,
    -814, -1095, -1388, -1692, -2006, -2330, -2663, -3004, -3351, -3705, -4063, -4425, -4788, -5153, -5517, -5879,
    -6237, -6589, -6935, -7271, -7597, -7910, -8209, -8491, -8755, -8998, -9219, -9416, -9585, -9727, -9838, -9916,
    -9959, -9966, -9935, -9863, -9750, -9592, -9389, -9139, -8840, -8492, -8092, -7640, -7134, 6574, 5959, 5288, 4561,
    3776, 2935, 2037, 1082, 70, -998, -2122, -3300, -4533, -5818, -7154, -8540, -9975, -11455, -12980, -14548, -16155,
    -17799, -19478, -21189, -22929, -24694, -26482, -28289, -30112, -31947, -33791, -35640, -37489, -39336, -41176,
    -43006, -44821, -46617, -48390, -50137, -51853, -53534, -55178, -56778, -58333, -59838, -61289, -62684, -64019,
    -65290, -66494, -67629, -68692, -69679, -70590, -71420, -72169, -72835, -73415, -73908, -74313, -74630, -74856,
    -74992, 75038]


def synth_window() -> np.ndarray:
    """The 512 coefficients D[i] (Table 3-B.3): D[512 - i] = D[i] for i a multiple of 64, -D[i] otherwise."""
    d = np.zeros(512)
    for i, v in enumerate(SYNTH_WINDOW_HALF):
        d[i] = v
        if i:
            d[512 - i] = v if i % 64 == 0 else -v
    return d / 65536.0


# Huffman code tables (Table 3-B.7): (size, hlen rows, hcod rows); tables 16..23 and 24..31 share codes, with linbits
_H = {
    1: (2, [1, 3, 2, 3], [1, 1, 1, 0]),
    2: (3, [1, 3, 6, 3, 3, 5, 5, 5, 6], [1, 2, 1, 3, 1, 1, 3, 2, 0]),
    3: (3, [2, 2, 6, 3, 2, 5, 5, 5, 6], [3, 2, 1, 1, 1, 1, 3, 2, 0]),
    5: (4, [1, 3, 6, 7, 3, 3, 6, 7, 6, 6, 7, 8, 7, 6, 7, 8], [1, 2, 6, 5, 3, 1, 4, 4, 7, 5, 7, 1, 6, 1, 1, 0]),
    6: (4, [3, 3, 5, 7, 3, 2, 4, 5, 4, 4, 5, 6, 6, 5, 6, 7], [7, 3, 5, 1, 6, 2, 3, 2, 5, 4, 4, 1, 3, 3, 2, 0]),
    7: (6, [1, 3, 6, 8, 8, 9, 3, 4, 6, 7, 7, 8, 6, 5, 7, 8, 8, 9, 7, 7, 8, 9, 9, 9, 7, 7, 8, 9, 9, 10, 8, 8, 9, 10,
            10, 10],
        [1, 2, 10, 19, 16, 10, 3, 3, 7, 10, 5, 3, 11, 4, 13, 17, 8, 4, 12, 11, 18, 15, 11, 2, 7, 6, 9, 14, 3, 1, 6, 4, 5,
         3, 2, 0]),
    8: (6, [2, 3, 6, 8, 8, 9, 3, 2, 4, 8, 8, 8, 6, 4, 6, 8, 8, 9, 8, 8, 8, 9, 9, 10, 8, 7, 8, 9, 10, 10, 9, 8, 9, 9,
            11, 11],
        [3, 4, 6, 18, 12, 5, 5, 1, 2, 16, 9, 3, 7, 3, 5, 14, 7, 3, 19, 17, 15, 13, 10, 4, 13, 5, 8, 11, 5, 1, 12, 4, 4,
         1, 1, 0]),
    9: (6, [3, 3, 5, 6, 8, 9, 3, 3, 4, 5, 6, 8, 4, 4, 5, 6, 7, 8, 6, 5, 6, 7, 7, 8, 7, 6, 7, 7, 8, 9, 8, 7, 8, 8, 9,
            9],
        [7, 5, 9, 14, 15, 7, 6, 4, 5, 5, 6, 7, 7, 6, 8, 8, 8, 5, 15, 6, 9, 10, 5, 1, 11, 7, 9, 6, 4, 1, 14, 4, 6, 2, 6,
         0]),
    10: (8, [1, 3, 6, 8, 9, 9, 9, 10, 3, 4, 6, 7, 8, 9, 8, 8, 6, 6, 7, 8, 9, 10, 9, 9, 7, 7, 8, 9, 10, 10, 9, 10, 8, 8,
             9, 10, 10, 10, 10, 10, 9, 9, 10, 10, 11, 11, 10, 11, 8, 8, 9, 10, 10, 10, 11, 11, 9, 8, 9, 10, 10, 11, 11,
             11],
         [1, 2, 10, 23, 35, 30, 12, 17, 3, 3, 8, 12, 18, 21, 12, 7, 11, 9, 15, 21, 32, 40, 19, 6, 14, 13, 22, 34, 46,
          23, 18, 7, 20, 19, 33, 47, 27, 22, 9, 3, 31, 22, 41, 26, 21, 20, 5, 3, 14, 13, 10, 11, 16, 6, 5, 1, 9, 8, 7,
          8, 4, 4, 2, 0]),
    11: (8, [2, 3, 5, 7, 8, 9, 8, 9, 3, 3, 4, 6, 8, 8, 7, 8, 5, 5, 6, 7, 8, 9, 8, 8, 7, 6, 7, 9, 8, 10, 8, 9, 8, 8, 8,
             9, 9, 10, 9, 10, 8, 8, 9, 10, 10, 11, 10, 11, 8, 7, 7, 8, 9, 10, 10, 10, 8, 7, 8, 9, 10, 10, 10, 10],
         [3, 4, 10, 24, 34, 33, 21, 15, 5, 3, 4, 10, 32, 17, 11, 10, 11, 7, 13, 18, 30, 31, 20, 5, 25, 11, 19, 59, 27,
          18, 12, 5, 35, 33, 31, 58, 30, 16, 7, 5, 28, 26, 32, 19, 17, 15, 8, 14, 14, 12, 9, 13, 14, 9, 4, 1, 11, 4, 6,
          6, 6, 3, 2, 0]),
    12: (8, [4, 3, 5, 7, 8, 9, 9, 9, 3, 3, 4, 5, 7, 7, 8, 8, 5, 4, 5, 6, 7, 8, 7, 8, 6, 5, 6, 6, 7, 8, 8, 8, 7, 6, 7,
             7, 8, 8, 8, 9, 8, 7, 8, 8, 8, 9, 8, 9, 8, 7, 7, 8, 8, 9, 9, 10, 9, 8, 8, 9, 9, 9, 9, 10],
         [9, 6, 16, 33, 41, 39, 38, 26, 7, 5, 6, 9, 23, 16, 26, 11, 17, 7, 11, 14, 21, 30, 10, 7, 17, 10, 15, 12, 18,
          28, 14, 5, 32, 13, 22, 19, 18, 16, 9, 5, 40, 17, 31, 29, 17, 13, 4, 2, 27, 12, 11, 15, 10, 7, 4, 1, 27, 12, 8,
          12, 6, 3, 1, 0]),
    13: (16, [
        1, 4, 6, 7, 8, 9, 9, 10, 9, 10, 11, 11, 12, 12, 13, 13, 3, 4, 6, 7, 8, 8, 9, 9, 9, 9, 10, 10, 11, 12, 12, 12,
        6, 6, 7, 8, 9, 9, 10, 10, 9, 10, 10, 11, 11, 12, 13, 13, 7, 7, 8, 9, 9, 10, 10, 10, 10, 11, 11, 11, 11, 12, 13,
        13, 8, 7, 9, 9, 10, 10, 11, 11, 10, 11, 11, 12, 12, 13, 13, 14, 9, 8, 9, 10, 10, 10, 11, 11, 11, 11, 12, 11, 13,
        13, 14, 14, 9, 9, 10, 10, 11, 11, 11, 11, 11, 12, 12, 12, 13, 13, 14, 14, 10, 9, 10, 11, 11, 11, 12, 12, 12, 12,
        13, 13, 13, 14, 16, 16, 9, 8, 9, 10, 10, 11, 11, 12, 12, 12, 12, 13, 13, 14, 15, 15, 10, 9, 10, 10, 11, 11, 11,
        13, 12, 13, 13, 14, 14, 14, 16, 15, 10, 10, 10, 11, 11, 12, 12, 13, 12, 13, 14, 13, 14, 15, 16, 17, 11, 10, 10,
        11, 12, 12, 12, 12, 13, 13, 13, 14, 15, 15, 15, 16, 11, 11, 11, 12, 12, 13, 12, 13, 14, 14, 15, 15, 15, 16, 16,
        16, 12, 11, 12, 13, 13, 13, 14, 14, 14, 14, 14, 15, 16, 15, 16, 16, 13, 12, 12, 13, 13, 13, 15, 14, 14, 17, 15,
        15, 15, 17, 16, 16, 12, 12, 13, 14, 14, 14, 15, 14, 15, 15, 16, 16, 19, 18, 19, 16], [
        1, 5, 14, 21, 34, 51, 46, 71, 42, 52, 68, 52, 67, 44, 43, 19, 3, 4, 12, 19, 31, 26, 44, 33, 31, 24, 32, 24, 31,
        35, 22, 14, 15, 13, 23, 36, 59, 49, 77, 65, 29, 40, 30, 40, 27, 33, 42, 16, 22, 20, 37, 61, 56, 79, 73, 64, 43,
        76, 56, 37, 26, 31, 25, 14, 35, 16, 60, 57, 97, 75, 114, 91, 54, 73, 55, 41, 48, 53, 23, 24, 58, 27, 50, 96, 76,
        70, 93, 84, 77, 58, 79, 29, 74, 49, 41, 17, 47, 45, 78, 74, 115, 94, 90, 79, 69, 83, 71, 50, 59, 38, 36, 15, 72,
        34, 56, 95, 92, 85, 91, 90, 86, 73, 77, 65, 51, 44, 43, 42, 43, 20, 30, 44, 55, 78, 72, 87, 78, 61, 46, 54, 37,
        30, 20, 16, 53, 25, 41, 37, 44, 59, 54, 81, 66, 76, 57, 54, 37, 18, 39, 11, 35, 33, 31, 57, 42, 82, 72, 80, 47,
        58, 55, 21, 22, 26, 38, 22, 53, 25, 23, 38, 70, 60, 51, 36, 55, 26, 34, 23, 27, 14, 9, 7, 34, 32, 28, 39, 49, 75,
        30, 52, 48, 40, 52, 28, 18, 17, 9, 5, 45, 21, 34, 64, 56, 50, 49, 45, 31, 19, 12, 15, 10, 7, 6, 3, 48, 23, 20,
        39, 36, 35, 53, 21, 16, 23, 13, 10, 6, 1, 4, 2, 16, 15, 17, 27, 25, 20, 29, 11, 17, 12, 16, 8, 1, 1, 0, 1]),
    15: (16, [
        3, 4, 5, 7, 7, 8, 9, 9, 9, 10, 10, 11, 11, 11, 12, 13, 4, 3, 5, 6, 7, 7, 8, 8, 8, 9, 9, 10, 10, 10, 11,
        11, 5, 5, 5, 6, 7, 7, 8, 8, 8, 9, 9, 10, 10, 11, 11, 11, 6, 6, 6, 7, 7, 8, 8, 9, 9, 9, 10, 10, 10, 11,
        11, 11, 7, 6, 7, 7, 8, 8, 9, 9, 9, 9, 10, 10, 10, 11, 11, 11, 8, 7, 7, 8, 8, 8, 9, 9, 9, 9, 10, 10, 11,
        11, 11, 12, 9, 7, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10, 11, 11, 12, 12, 9, 8, 8, 9, 9, 9, 9, 10, 10, 10, 10,
        10, 11, 11, 11, 12, 9, 8, 8, 9, 9, 9, 9, 10, 10, 10, 10, 11, 11, 12, 12, 12, 9, 8, 9, 9, 9, 9, 10, 10,
        10, 11, 11, 11, 11, 12, 12, 12, 10, 9, 9, 9, 10, 10, 10, 10, 10, 11, 11, 11, 11, 12, 13, 12, 10, 9, 9,
        9, 10, 10, 10, 10, 11, 11, 11, 11, 12, 12, 12, 13, 11, 10, 9, 10, 10, 10, 11, 11, 11, 11, 11, 11, 12,
        12, 13, 13, 11, 10, 10, 10, 10, 11, 11, 11, 11, 12, 12, 12, 12, 12, 13, 13, 12, 11, 11, 11, 11, 11, 11,
        11, 12, 12, 12, 12, 13, 13, 12, 13, 12, 11, 11, 11, 11, 11, 11, 12, 12, 12, 12, 12, 13, 13, 13, 13], [
        7, 12, 18, 53, 47, 76, 124, 108, 89, 123, 108, 119, 107, 81, 122, 63, 13, 5, 16, 27, 46, 36, 61, 51, 42, 70, 52,
        83, 65, 41, 59, 36, 19, 17, 15, 24, 41, 34, 59, 48, 40, 64, 50, 78, 62, 80, 56, 33, 29, 28, 25, 43, 39, 63, 55,
        93, 76, 59, 93, 72, 54, 75, 50, 29, 52, 22, 42, 40, 67, 57, 95, 79, 72, 57, 89, 69, 49, 66, 46, 27, 77, 37, 35,
        66, 58, 52, 91, 74, 62, 48, 79, 63, 90, 62, 40, 38, 125, 32, 60, 56, 50, 92, 78, 65, 55, 87, 71, 51, 73, 51, 70,
        30, 109, 53, 49, 94, 88, 75, 66, 122, 91, 73, 56, 42, 64, 44, 21, 25, 90, 43, 41, 77, 73, 63, 56, 92, 77, 66,
        47, 67, 48, 53, 36, 20, 71, 34, 67, 60, 58, 49, 88, 76, 67, 106, 71, 54, 38, 39, 23, 15, 109, 53, 51, 47, 90,
        82, 58, 57, 48, 72, 57, 41, 23, 27, 62, 9, 86, 42, 40, 37, 70, 64, 52, 43, 70, 55, 42, 25, 29, 18, 11, 11, 118,
        68, 30, 55, 50, 46, 74, 65, 49, 39, 24, 16, 22, 13, 14, 7, 91, 44, 39, 38, 34, 63, 52, 45, 31, 52, 28, 19, 14,
        8, 9, 3, 123, 60, 58, 53, 47, 43, 32, 22, 37, 24, 17, 12, 15, 10, 2, 1, 71, 37, 34, 30, 28, 20, 17, 26, 21, 16,
        10, 6, 8, 6, 2, 0]),
    16: (16, [
        1, 4, 6, 8, 9, 9, 10, 10, 11, 11, 11, 12, 12, 12, 13, 9, 3, 4, 6, 7, 8, 9, 9, 9, 10, 10, 10, 11, 12, 11,
        12, 8, 6, 6, 7, 8, 9, 9, 10, 10, 11, 10, 11, 11, 11, 12, 12, 9, 8, 7, 8, 9, 9, 10, 10, 10, 11, 11, 12,
        12, 12, 13, 13, 10, 9, 8, 9, 9, 10, 10, 11, 11, 11, 12, 12, 12, 13, 13, 13, 9, 9, 8, 9, 9, 10, 11, 11,
        12, 11, 12, 12, 13, 13, 13, 14, 10, 10, 9, 9, 10, 11, 11, 11, 11, 12, 12, 12, 12, 13, 13, 14, 10, 10, 9,
        10, 10, 11, 11, 11, 12, 12, 13, 13, 13, 13, 15, 15, 10, 10, 10, 10, 11, 11, 11, 12, 12, 13, 13, 13, 13,
        14, 14, 14, 10, 11, 10, 10, 11, 11, 12, 12, 13, 13, 13, 13, 14, 13, 14, 13, 11, 11, 11, 10, 11, 12, 12,
        12, 12, 13, 14, 14, 14, 15, 15, 14, 10, 12, 11, 11, 11, 12, 12, 13, 14, 14, 14, 14, 14, 14, 13, 14, 11,
        12, 12, 12, 12, 12, 13, 13, 13, 13, 15, 14, 14, 14, 14, 16, 11, 14, 12, 12, 12, 13, 13, 14, 14, 14, 16,
        15, 15, 15, 17, 15, 11, 13, 13, 11, 12, 14, 14, 13, 14, 14, 15, 16, 15, 17, 15, 14, 11, 9, 8, 8, 9, 9,
        10, 10, 10, 11, 11, 11, 11, 11, 11, 11, 8], [
        1, 5, 14, 44, 74, 63, 110, 93, 172, 149, 138, 242, 225, 195, 376, 17, 3, 4, 12, 20, 35, 62, 53, 47, 83, 75, 68,
        119, 201, 107, 207, 9, 15, 13, 23, 38, 67, 58, 103, 90, 161, 72, 127, 117, 110, 209, 206, 16, 45, 21, 39, 69, 64,
        114, 99, 87, 158, 140, 252, 212, 199, 387, 365, 26, 75, 36, 68, 65, 115, 101, 179, 164, 155, 264, 246, 226, 395,
        382, 362, 9, 66, 30, 59, 56, 102, 185, 173, 265, 142, 253, 232, 400, 388, 378, 445, 16, 111, 54, 52, 100, 184,
        178, 160, 133, 257, 244, 228, 217, 385, 366, 715, 10, 98, 48, 91, 88, 165, 157, 148, 261, 248, 407, 397, 372,
        380, 889, 884, 8, 85, 84, 81, 159, 156, 143, 260, 249, 427, 401, 392, 383, 727, 713, 708, 7, 154, 76, 73, 141,
        131, 256, 245, 426, 406, 394, 384, 735, 359, 710, 352, 11, 139, 129, 67, 125, 247, 233, 229, 219, 393, 743, 737,
        720, 885, 882, 439, 4, 243, 120, 118, 115, 227, 223, 396, 746, 742, 736, 721, 712, 706, 223, 436, 6, 202, 224,
        222, 218, 216, 389, 386, 381, 364, 888, 443, 707, 440, 437, 1728, 4, 747, 211, 210, 208, 370, 379, 734, 723, 714,
        1735, 883, 877, 876, 3459, 865, 2, 377, 369, 102, 187, 726, 722, 358, 711, 709, 866, 1734, 871, 3458, 870, 434,
        0, 12, 10, 7, 11, 10, 17, 11, 9, 13, 12, 10, 7, 5, 3, 1, 3]),
    24: (16, [
        4, 4, 6, 7, 8, 9, 9, 10, 10, 11, 11, 11, 11, 11, 12, 9, 4, 4, 5, 6, 7, 8, 8, 9, 9, 9, 10, 10, 10, 10,
        10, 8, 6, 5, 6, 7, 7, 8, 8, 9, 9, 9, 9, 10, 10, 10, 11, 7, 7, 6, 7, 7, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10,
        10, 7, 8, 7, 7, 8, 8, 8, 8, 9, 9, 9, 10, 10, 10, 10, 11, 7, 9, 7, 8, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10,
        10, 10, 7, 9, 8, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10, 10, 10, 11, 7, 10, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10,
        10, 10, 11, 11, 8, 10, 9, 9, 9, 9, 9, 9, 9, 9, 10, 10, 10, 10, 11, 11, 8, 10, 9, 9, 9, 9, 9, 9, 10, 10,
        10, 10, 10, 11, 11, 11, 8, 11, 9, 9, 9, 9, 10, 10, 10, 10, 10, 10, 11, 11, 11, 11, 8, 11, 10, 9, 9, 9,
        10, 10, 10, 10, 10, 10, 11, 11, 11, 11, 8, 11, 10, 10, 10, 10, 10, 10, 10, 10, 10, 11, 11, 11, 11, 11,
        8, 11, 10, 10, 10, 10, 10, 10, 10, 11, 11, 11, 11, 11, 11, 11, 8, 12, 10, 10, 10, 10, 10, 10, 11, 11,
        11, 11, 11, 11, 11, 11, 8, 8, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 8, 8, 8, 8, 4], [
        15, 13, 46, 80, 146, 262, 248, 434, 426, 669, 653, 649, 621, 517, 1032, 88, 14, 12, 21, 38, 71, 130, 122, 216,
        209, 198, 327, 345, 319, 297, 279, 42, 47, 22, 41, 74, 68, 128, 120, 221, 207, 194, 182, 340, 315, 295, 541, 18,
        81, 39, 75, 70, 134, 125, 116, 220, 204, 190, 178, 325, 311, 293, 271, 16, 147, 72, 69, 135, 127, 118, 112, 210,
        200, 188, 352, 323, 306, 285, 540, 14, 263, 66, 129, 126, 119, 114, 214, 202, 192, 180, 341, 317, 301, 281, 262,
        12, 249, 123, 121, 117, 113, 215, 206, 195, 185, 347, 330, 308, 291, 272, 520, 10, 435, 115, 111, 109, 211, 203,
        196, 187, 353, 332, 313, 298, 283, 531, 381, 17, 427, 212, 208, 205, 201, 193, 186, 177, 169, 320, 303, 286, 268,
        514, 377, 16, 335, 199, 197, 191, 189, 181, 174, 333, 321, 305, 289, 275, 521, 379, 371, 11, 668, 184, 183, 179,
        175, 344, 331, 314, 304, 290, 277, 530, 383, 373, 366, 10, 652, 346, 171, 168, 164, 318, 309, 299, 287, 276, 263,
        513, 375, 368, 362, 6, 648, 322, 316, 312, 307, 302, 292, 284, 269, 261, 512, 376, 370, 364, 359, 4, 620, 300,
        296, 294, 288, 282, 273, 266, 515, 380, 374, 369, 365, 361, 357, 2, 1033, 280, 278, 274, 267, 264, 259, 382, 378,
        372, 367, 363, 360, 358, 356, 0, 43, 20, 19, 17, 15, 13, 11, 9, 7, 6, 4, 7, 5, 3, 1, 3]),
}
COUNT1_A = ([1, 4, 4, 5, 4, 6, 5, 6, 4, 5, 5, 6, 5, 6, 6, 6], [1, 5, 4, 5, 6, 5, 4, 4, 7, 3, 6, 0, 7, 2, 3, 1])
COUNT1_B = ([4] * 16, [15 - v for v in range(16)])
LINBITS = {**{t: 0 for t in range(16)}, 16: 1, 17: 2, 18: 3, 19: 4, 20: 6, 21: 8, 22: 10, 23: 13,
           24: 4, 25: 5, 26: 6, 27: 7, 28: 8, 29: 9, 30: 11, 31: 13}


def code_table(t: int):
    """(size, hlen, hcod) of big-values table t (None for table 0, 4 and 14)."""
    if t in (0, 4, 14):
        return None
    return _H[16 if 16 <= t < 24 else 24 if t >= 24 else t]


# ------------------------------------------------------------------------------------------------ bits
class BitReader:
    def __init__(self, data: bytes, pos: int = 0):
        self.data = bytes(data) + b"\0" * 8
        self.n = 8 * len(data)
        self.pos = pos

    def read(self, k: int) -> int:
        if k == 0:
            return 0
        if self.pos < 0 or self.pos + k > self.n:
            raise EOFError
        p = self.pos
        v = int.from_bytes(self.data[p >> 3 : (p >> 3) + 4], "big")
        self.pos += k
        return (v >> (32 - (p & 7) - k)) & ((1 << k) - 1)


class BitWriter:
    def __init__(self):
        self.bits = []

    def write(self, v: int, k: int):
        for i in range(k - 1, -1, -1):
            self.bits.append((v >> i) & 1)

    def getvalue(self) -> bytes:
        b = self.bits + [0] * (-len(self.bits) % 8)
        return np.packbits(np.array(b, dtype=np.uint8)).tobytes() if b else b""


_DECODERS = {}


def _decoder(key, hlen, hcod, size):
    """{(length, code): (x, y)} of one table."""
    if key not in _DECODERS:
        _DECODERS[key] = {(l, c): (i // size, i % size) for i, (l, c) in enumerate(zip(hlen, hcod))}
    return _DECODERS[key]


def _decode_symbol(br: BitReader, dec):
    code, length = 0, 0
    while length < 20:
        code = (code << 1) | br.read(1)
        length += 1
        if (length, code) in dec:
            return dec[(length, code)]
    raise ValueError("no Huffman code")


# ------------------------------------------------------------------------------------------------ headers and side info
@dataclasses.dataclass
class Header:
    raw: int
    crc: bool
    bitrate: int
    sample_rate: int
    padding: int
    mode: int
    mode_ext: int

    @property
    def channels(self):
        return 1 if self.mode == 3 else 2

    @property
    def length(self):
        return 144000 * self.bitrate // self.sample_rate + self.padding

    @property
    def side_bytes(self):
        return 17 if self.mode == 3 else 32


def parse_header(b: bytes):
    """The MPEG-1 Layer III header at b[0:4], or None (not a sync, another version or layer, free format, reserved)."""
    if len(b) < 4:
        return None
    v = int.from_bytes(b[:4], "big")
    if (v >> 21) != 0x7FF or ((v >> 19) & 3) != 3 or ((v >> 17) & 3) != 1:
        return None
    bi, si, emph = (v >> 12) & 15, (v >> 10) & 3, v & 3
    if bi in (0, 15) or si == 3 or emph == 2:
        return None
    return Header(v, not (v >> 16) & 1, BITRATES[bi], RATES[si], (v >> 9) & 1, (v >> 6) & 3, (v >> 4) & 3)


@dataclasses.dataclass
class Granule:
    part2_3_length: int = 0
    big_values: int = 0
    global_gain: int = 0
    scalefac_compress: int = 0
    window_switching: int = 0
    block_type: int = 0
    mixed: int = 0
    table_select: tuple = (0, 0, 0)
    subblock_gain: tuple = (0, 0, 0)
    region0_count: int = 0
    region1_count: int = 0
    preflag: int = 0
    scalefac_scale: int = 0
    count1_table: int = 0


@dataclasses.dataclass
class SideInfo:
    main_data_begin: int
    private_bits: int
    scfsi: list            # [ch][4]
    gr: list               # [2][ch] Granule


def parse_side_info(b: bytes, nch: int) -> SideInfo:
    br = BitReader(b)
    mdb = br.read(9)
    priv = br.read(5 if nch == 1 else 3)
    scfsi = [[br.read(1) for _ in range(4)] for _ in range(nch)]
    grs = []
    for _ in range(2):
        row = []
        for _ in range(nch):
            g = Granule(br.read(12), br.read(9), br.read(8), br.read(4), br.read(1))
            if g.window_switching:
                g.block_type, g.mixed = br.read(2), br.read(1)
                g.table_select = (br.read(5), br.read(5), 0)
                g.subblock_gain = (br.read(3), br.read(3), br.read(3))
                g.region0_count = 7 if (g.block_type != 2 or g.mixed) else 8
                g.region1_count = 20 - g.region0_count
            else:
                g.table_select = (br.read(5), br.read(5), br.read(5))
                g.region0_count, g.region1_count = br.read(4), br.read(3)
            g.preflag, g.scalefac_scale, g.count1_table = br.read(1), br.read(1), br.read(1)
            row.append(g)
        grs.append(row)
    return SideInfo(mdb, priv, scfsi, grs)


def write_side_info(si: SideInfo, nch: int) -> bytes:
    bw = BitWriter()
    bw.write(si.main_data_begin, 9)
    bw.write(si.private_bits, 5 if nch == 1 else 3)
    for ch in range(nch):
        for v in si.scfsi[ch]:
            bw.write(v, 1)
    for gr in range(2):
        for ch in range(nch):
            g = si.gr[gr][ch]
            bw.write(g.part2_3_length, 12)
            bw.write(g.big_values, 9)
            bw.write(g.global_gain, 8)
            bw.write(g.scalefac_compress, 4)
            bw.write(g.window_switching, 1)
            if g.window_switching:
                bw.write(g.block_type, 2)
                bw.write(g.mixed, 1)
                bw.write(g.table_select[0], 5)
                bw.write(g.table_select[1], 5)
                for v in g.subblock_gain:
                    bw.write(v, 3)
            else:
                for v in g.table_select:
                    bw.write(v, 5)
                bw.write(g.region0_count, 4)
                bw.write(g.region1_count, 3)
            bw.write(g.preflag, 1)
            bw.write(g.scalefac_scale, 1)
            bw.write(g.count1_table, 1)
    out = bw.getvalue()
    assert len(out) == (17 if nch == 1 else 32)
    return out


def skip_id3v2(data: bytes) -> int:
    if len(data) >= 10 and data[:3] == b"ID3":
        return 10 + ((data[6] & 0x7F) << 21 | (data[7] & 0x7F) << 14 | (data[8] & 0x7F) << 7 | (data[9] & 0x7F)) + (
            10 if data[5] & 0x10 else 0)
    return 0


def frames_of(data: bytes):
    """[(offset, Header)] of the frames of an MPEG-1 Layer III stream, as bt_mp3_probe walks it: after an ID3v2 tag,
    the first header followed by two more consistent headers at the lengths the headers give (or by the end of the
    data); then header after header while the next one continues the stream (same rate and channels).  A truncated
    last frame is dropped.  (Trailing tags are not stripped: the tests' streams put none in front of a decode.)"""
    pos = skip_id3v2(data)
    n = len(data)

    def ok(p, first):
        h = parse_header(data[p : p + 4])
        return h if h and (first is None or (h.sample_rate, h.channels) == (first.sample_rate, first.channels)) else None

    def confirmed(p):
        h = ok(p, None)
        if not h or p + h.length > n:
            return False
        q, m = p, h
        for k in range(2):
            q += m.length
            if q == n:
                return True
            m = ok(q, h)
            if m is None or q + m.length > n:
                return k > 0 and q + 4 > n
        return True

    while pos + 4 <= n and not confirmed(pos):
        pos += 1
    if pos + 4 > n:
        return []
    out = []
    first = parse_header(data[pos : pos + 4])
    while pos + 4 <= n:
        h = ok(pos, first)
        if h is None or pos + h.length > n:
            break
        out.append((pos, h))
        pos += h.length
    return out


# ------------------------------------------------------------------------------------------------ containers
FIXTURE = "kings_of_swing_383.mp3"  # tests/golden: the first 383 frames of the reference's test recording


def split_frames(data: bytes):
    """The frames of a tag-less stream whose first byte is a header, as a list of bytes objects."""
    return [data[o : o + h.length] for o, h in frames_of(data)]


def with_header(frame: bytes, **fields) -> bytes:
    """frame with header fields replaced: mode_ext, mode, version (2 bits), layer (2 bits), bitrate_index,
    rate_index."""
    v = int.from_bytes(frame[:4], "big")
    pos = {"mode_ext": (4, 3), "mode": (6, 3), "rate_index": (10, 3), "bitrate_index": (12, 15), "layer": (17, 3),
           "version": (19, 3)}
    for k, val in fields.items():
        sh, m = pos[k]
        v = (v & ~(m << sh)) | (val << sh)
    return v.to_bytes(4, "big") + frame[4:]


def id3v2(size: int, footer: bool = False) -> bytes:
    body = (bytes(range(251)) * (size // 251 + 1))[:size]
    ss = bytes([(size >> 21) & 0x7F, (size >> 14) & 0x7F, (size >> 7) & 0x7F, size & 0x7F])
    head = b"ID3\x04\x00" + bytes([0x10 if footer else 0]) + ss
    return head + body + (b"3DI\x04\x00\x10" + ss if footer else b"")


def id3v1() -> bytes:
    return (b"TAG" + b"title".ljust(30, b"\0") + b"\xff\xfb" * 40)[:128].ljust(128, b"\0")


def apev2(items: bytes = b"\xff\xfb\x90\x64" * 8) -> bytes:
    def block(flags):
        return b"APETAGEX" + (2000).to_bytes(4, "little") + (len(items) + 32).to_bytes(4, "little") + \
            (1).to_bytes(4, "little") + flags.to_bytes(4, "little") + bytes(8)
    return block(0xA0000000) + items + block(0x80000000)


def xing_frame(template: bytes, n_frames: int, delay: int = None, padding: int = 0, encoder: bytes = b"LAME3.100") -> bytes:
    """An Info frame of template's header (a silent frame: zero side info) giving n_frames, and a LAME-style tag with
    the encoder delay and padding unless delay is None."""
    h = parse_header(template[:4])
    f = bytearray(h.length)
    f[:4] = template[:4]
    x = 4 + (2 if h.crc else 0) + h.side_bytes
    f[x : x + 4] = b"Info"
    f[x + 4 : x + 8] = (1 | 2 | 4 | 8).to_bytes(4, "big")
    f[x + 8 : x + 12] = n_frames.to_bytes(4, "big")
    q = x + 8 + 4 + 4 + 100 + 4
    if delay is not None:
        f[q : q + 9] = encoder[:9].ljust(9, b" ")
        f[q + 21 : q + 24] = bytes([delay >> 4, ((delay & 15) << 4) | (padding >> 8), padding & 0xFF])
    return bytes(f)


# ------------------------------------------------------------------------------------------------ decoder
def sfb_bounds(widths):
    return np.concatenate([[0], np.cumsum(widths)])


def read_scalefactors(br, g: Granule, scfsi, gr, prev):
    """Scalefactors of one granule and channel: {"l": [22]} or {"s": [13][3]} (mixed: both, long 0..7)."""
    s1, s2 = SLEN[g.scalefac_compress]
    sf = {"l": [0] * 22, "s": [[0] * 3 for _ in range(13)]}
    if g.window_switching and g.block_type == 2:
        if g.mixed:
            for b in range(8):
                sf["l"][b] = br.read(s1)
            start = 3
        else:
            start = 0
        for b in range(start, 12):
            for w in range(3):
                sf["s"][b][w] = br.read(s1 if b < 6 else s2)
    else:
        groups = [(0, 6), (6, 11), (11, 16), (16, 21)]
        for k, (a, e) in enumerate(groups):
            for b in range(a, e):
                if gr == 1 and scfsi[k]:
                    sf["l"][b] = prev["l"][b]
                else:
                    sf["l"][b] = br.read(s1 if k < 2 else s2)
    return sf


def huffman_lines(br, g: Granule, end: int, rate: int):
    """The 576 quantised lines of one granule and channel, reading up to bit `end`; the number of lines decoded."""
    x = np.zeros(576, dtype=np.int64)
    bv = g.big_values * 2
    if bv > 576:
        raise ValueError("big_values > 288")
    if g.window_switching:
        r1, r2 = 36, 576
    else:
        b = sfb_bounds(SFB_LONG[rate])
        r1 = b[min(g.region0_count + 1, 22)]
        r2 = b[min(g.region0_count + g.region1_count + 2, 22)]
    i = 0
    while i < bv:
        t = g.table_select[0 if i < r1 else 1 if i < r2 else 2]
        ct = code_table(t)
        if ct is None:
            if t != 0:
                raise ValueError(f"table {t}")
            x[i] = x[i + 1] = 0
            i += 2
            continue
        size, hlen, hcod = ct
        dec = _decoder(size * 100 + (16 if 16 <= t < 24 else 24 if t >= 24 else t), hlen, hcod, size)
        a, c = _decode_symbol(br, dec)
        lb = LINBITS[t]
        vals = []
        for v in (a, c):
            if lb and v == 15:
                v += br.read(lb)
            if v and br.read(1):
                v = -v
            vals.append(v)
        x[i], x[i + 1] = vals
        i += 2
    if br.pos > end:
        raise ValueError("big_values past part2_3_length")
    hl, hc = COUNT1_B if g.count1_table else COUNT1_A
    dec = _decoder(("c1", g.count1_table), hl, hc, 16)
    while i + 4 <= 576 and br.pos < end:
        save = br.pos
        q = _decode_symbol(br, dec)
        q = q[0] * 16 + q[1]
        vals = []
        for k in (3, 2, 1, 0):
            v = (q >> k) & 1
            if v and br.read(1):
                v = -v
            vals.append(v)
        if br.pos > end:  # a quadruple that overshoots part2_3_length is dropped
            br.pos = save
            break
        x[i : i + 4] = vals
        i += 4
    return x, i


def requantize(x, g: Granule, sf, rate):
    """Dequantised lines (float64), and for short bands the window of every line."""
    xr = np.sign(x) * np.abs(x).astype(np.float64) ** (4.0 / 3.0)
    mult = 0.5 * (1 + g.scalefac_scale)
    gain = np.zeros(576)
    bl, bs = sfb_bounds(SFB_LONG[rate]), sfb_bounds(SFB_SHORT[rate])
    base = g.global_gain - 210
    if g.window_switching and g.block_type == 2:
        long_end = 36 if g.mixed else 0
        for b in range(8 if g.mixed else 0):
            gain[bl[b] : bl[b + 1]] = 0.25 * base - mult * (sf["l"][b] + g.preflag * PRETAB[b])
        for b in range(3 if g.mixed else 0, 13):
            w_ = bs[b + 1] - bs[b]
            for w in range(3):
                a = 3 * bs[b] + w * w_
                gain[a : a + w_] = 0.25 * (base - 8 * g.subblock_gain[w]) - mult * sf["s"][b][w]
        assert long_end in (0, 36)
    else:
        for b in range(22):
            gain[bl[b] : bl[b + 1]] = 0.25 * base - mult * (sf["l"][b] + g.preflag * PRETAB[b])
    return xr * np.exp2(gain)


def _short_start(g):
    return 3 if g.mixed else 0


def stereo(xr, grs, sfs, hdr, nz, rate):
    """M/S and intensity stereo in place on xr[2][576]."""
    ms = hdr.mode == 1 and hdr.mode_ext & 2
    is_ = hdr.mode == 1 and hdr.mode_ext & 1
    if not (ms or is_):
        return
    g = grs[1]
    is_line = np.zeros(576, dtype=bool)
    ratio = np.zeros(576)
    if is_:
        bl, bs = sfb_bounds(SFB_LONG[rate]), sfb_bounds(SFB_SHORT[rate])
        r = xr[1]
        nzr = np.nonzero(r)[0]
        if g.window_switching and g.block_type == 2:
            any_short_nz = False
            for w in range(3):
                last = -1  # last short band of window w with a nonzero line
                for b in range(_short_start(g), 13):
                    wd = bs[b + 1] - bs[b]
                    a = 3 * bs[b] + w * wd
                    if np.any(r[a : a + wd] != 0):
                        last = b
                if last >= 0:
                    any_short_nz = True
                for b in range(max(last + 1, _short_start(g)), 13):
                    wd = bs[b + 1] - bs[b]
                    a = 3 * bs[b] + w * wd
                    pos = sfs[1]["s"][b if b < 12 else 11][w]
                    if pos != 7:
                        is_line[a : a + wd] = True
                        ratio[a : a + wd] = math.tan(pos * math.pi / 12)
            if g.mixed and not any_short_nz:
                last = int(nzr[-1]) if len(nzr) else -1
                for b in range(8):
                    if bl[b] > last:
                        pos = sfs[1]["l"][b]
                        if pos != 7:
                            is_line[bl[b] : bl[b + 1]] = True
                            ratio[bl[b] : bl[b + 1]] = math.tan(pos * math.pi / 12)
        else:
            last = int(nzr[-1]) if len(nzr) else -1
            for b in range(22):
                if bl[b] > last:
                    pos = sfs[1]["l"][b if b < 21 else 20]
                    if pos != 7:
                        is_line[bl[b] : bl[b + 1]] = True
                        ratio[bl[b] : bl[b + 1]] = math.tan(pos * math.pi / 12)
    l, r = xr[0].copy(), xr[1].copy()
    if ms:
        msl = ~is_line
        xr[0][msl] = (l[msl] + r[msl]) / math.sqrt(2)
        xr[1][msl] = (l[msl] - r[msl]) / math.sqrt(2)
    k = ratio[is_line] / (1 + ratio[is_line])
    xr[0][is_line] = l[is_line] * k
    xr[1][is_line] = l[is_line] * (1 - k)


def reorder(xr, g, rate):
    """Short bands from [window][line] to line-interleaved order (index 3 * line + window within the band)."""
    if not (g.window_switching and g.block_type == 2):
        return xr
    out = xr.copy()
    bs = sfb_bounds(SFB_SHORT[rate])
    for b in range(_short_start(g), 13):
        wd = bs[b + 1] - bs[b]
        for w in range(3):
            for j in range(wd):
                out[3 * bs[b] + 3 * j + w] = xr[3 * bs[b] + w * wd + j]
    return out


def alias(xr, g):
    if g.window_switching and g.block_type == 2 and not g.mixed:
        return xr
    xr = xr.copy()
    cs = [1 / math.sqrt(1 + c * c) for c in ALIAS_C]
    ca = [c / math.sqrt(1 + c * c) for c in ALIAS_C]
    last = 2 if (g.window_switching and g.block_type == 2) else 32
    for sb in range(1, last):
        for i in range(8):
            bu, bd = xr[18 * sb - 1 - i], xr[18 * sb + i]
            xr[18 * sb - 1 - i] = bu * cs[i] - bd * ca[i]
            xr[18 * sb + i] = bd * cs[i] + bu * ca[i]
    return xr


def window(block_type: int) -> np.ndarray:
    i = np.arange(36)
    w = np.sin(np.pi / 36 * (i + 0.5))
    if block_type == 1:
        w[18:24] = 1
        w[24:30] = np.sin(np.pi / 12 * (i[24:30] - 18 + 0.5))
        w[30:] = 0
    elif block_type == 3:
        w[:6] = 0
        w[6:12] = np.sin(np.pi / 12 * (i[6:12] - 6 + 0.5))
        w[12:18] = 1
    return w


_COS36 = np.cos(np.pi / 72 * np.outer(2 * np.arange(36) + 1 + 18, 2 * np.arange(18) + 1))
_COS12 = np.cos(np.pi / 24 * np.outer(2 * np.arange(12) + 1 + 6, 2 * np.arange(6) + 1))
_WIN12 = np.sin(np.pi / 12 * (np.arange(12) + 0.5))


def imdct(xr, g) -> np.ndarray:
    """The windowed 36-value block of every subband, [32][36]."""
    z = np.zeros((32, 36))
    short = g.window_switching and g.block_type == 2
    for sb in range(32):
        X = xr[18 * sb : 18 * sb + 18]
        if short and not (g.mixed and sb < 2):
            for w in range(3):
                y = _COS12 @ X[w::3] * _WIN12
                z[sb, 6 + 6 * w : 18 + 6 * w] += y
        else:
            bt = 0 if short else (g.block_type if g.window_switching else 0)
            z[sb] = (_COS36 @ X) * window(bt)
    return z


_N = np.cos(np.outer(16 + np.arange(64), 2 * np.arange(32) + 1) * np.pi / 64)


def synthesize(S: np.ndarray) -> np.ndarray:
    """Polyphase synthesis of subband samples S [slots, 32]: PCM [slots * 32]."""
    D = synth_window()
    V = S @ _N.T  # [slots, 64]
    T = len(S)
    Vp = np.concatenate([np.zeros((16, 64)), V])
    out = np.zeros((T, 32))
    for i in range(8):
        out += Vp[16 - 2 * i : 16 - 2 * i + T, :32] * D[64 * i : 64 * i + 32]
        out += Vp[15 - 2 * i : 15 - 2 * i + T, 32:] * D[64 * i + 32 : 64 * i + 64]
    return out.reshape(-1)


@dataclasses.dataclass
class Decoded:
    pcm: np.ndarray            # [samples, channels] float64, every decoded sample (no gapless trim)
    rate: int
    granule_ends: list         # (bits consumed, part2_3_length) per granule and channel
    lines: list                # quantised lines [frame][gr][ch]
    gains: list = None         # the requantisation gain of every line [frame][gr][ch]
    short: list = None         # whether every line is in a short (12-point) block [frame][gr][ch]


def main_data_layout(data: bytes, frames):
    """The compacted main data of the frames (each frame's bytes after header, CRC and side info, in order), every
    frame's side info and its main-data start in the compacted bytes (may be negative)."""
    main = bytearray()
    sides, starts = [], []
    for off, h in frames:
        s = off + 4 + (2 if h.crc else 0)
        si = parse_side_info(data[s : s + h.side_bytes], h.channels)
        starts.append(len(main) - si.main_data_begin)
        sides.append(si)
        main += data[s + h.side_bytes : off + h.length]
    return bytes(main), sides, starts


def decode(data: bytes, frames=None) -> Decoded:
    """Every frame of the stream in float64 (raises ValueError on a malformed granule)."""
    frames = frames_of(data) if frames is None else frames
    if not frames:
        raise ValueError("no frames")
    rate, nch = frames[0][1].sample_rate, frames[0][1].channels
    main, sides, starts = main_data_layout(data, frames)
    nbits = 8 * len(main)
    blocks = np.zeros((len(frames) * 2 + 1, nch, 32, 36))
    ends, all_lines, all_gains, all_short = [], [], [], []
    for f, ((off, h), si, start) in enumerate(zip(frames, sides, starts)):
        bit = 8 * start
        flines, fgains, fshort = [], [], []
        prev_sf = [None] * nch
        for gr in range(2):
            xr = np.zeros((nch, 576))
            sfs, nzs, glines, ggains, gshort = [], [], [], [], []
            for ch in range(nch):
                g = si.gr[gr][ch]
                if bit < 0:  # main data before the stream's first byte: a zero spectrum
                    sf = {"l": [0] * 22, "s": [[0] * 3 for _ in range(13)]}
                    x, nz = np.zeros(576, dtype=np.int64), 0
                else:
                    if bit + g.part2_3_length > nbits:
                        raise ValueError("main data past the end")
                    br = BitReader(main, bit)
                    sf = read_scalefactors(br, g, si.scfsi[ch], gr, prev_sf[ch] or {"l": [0] * 22})
                    if br.pos - bit > g.part2_3_length:
                        raise ValueError("scalefactors past part2_3_length")
                    x, nz = huffman_lines(br, g, bit + g.part2_3_length, rate)
                    ends.append((br.pos - bit, g.part2_3_length))
                if g.window_switching and g.block_type == 0:
                    raise ValueError("window switching with block type 0")
                prev_sf[ch] = sf
                sfs.append(sf)
                nzs.append(nz)
                glines.append(x)
                xr[ch] = requantize(x, g, sf, rate)
                ggains.append(requantize(np.ones(576, dtype=np.int64), g, sf, rate))
                sh = np.zeros(576, dtype=bool)
                if g.window_switching and g.block_type == 2:
                    sh[36 if g.mixed else 0 :] = True
                gshort.append(sh)
                bit += g.part2_3_length
            flines.append(glines)
            fgains.append(ggains)
            fshort.append(gshort)
            if nch == 2:
                stereo(xr, si.gr[gr], sfs, h, nzs, rate)
            for ch in range(nch):
                g = si.gr[gr][ch]
                blocks[1 + 2 * f + gr, ch] = imdct(alias(reorder(xr[ch], g, rate), g), g)
        all_lines.append(flines)
        all_gains.append(fgains)
        all_short.append(fshort)
    # overlap-add with the previous granule's tail, frequency inversion, synthesis
    S = blocks[1:, :, :, :18] + blocks[:-1, :, :, 18:]  # [granules, ch, 32, 18]
    S[:, :, 1::2, 1::2] *= -1
    pcm = np.stack([synthesize(S[:, ch].transpose(0, 2, 1).reshape(-1, 32)) for ch in range(nch)], axis=1)
    return Decoded(pcm, rate, ends, all_lines, all_gains, all_short)


# ------------------------------------------------------------------------------------------------ encoder and writer
# The analysis side of the standard: the polyphase analysis filter bank (window C[i] = D[i] / 32, Annex C), the MDCT
# of every block type, the forward alias butterflies, optional M/S, fine quantisation and Huffman coding, packed into
# frames with or without the bit reservoir.  Every side-info field is the caller's to choose, so each decoder feature
# can be produced on demand; the quantised lines are the encoder's own (the decoder of this module is not consulted).
_MK = np.cos(np.outer(2 * np.arange(32) + 1, np.arange(64) - 16) * np.pi / 64)


def analysis(x: np.ndarray) -> np.ndarray:
    """Subband samples [slots, 32] of mono samples x (len a multiple of 32; zeros before the start)."""
    C = synth_window() / 32
    xp = np.concatenate([np.zeros(512), x])
    T = len(x) // 32
    idx = 512 + 32 * np.arange(T)[:, None] + 31 - np.arange(512)[None, :]
    Y = (xp[idx] * C).reshape(T, 8, 64).sum(1)
    return Y @ _MK.T


def _mdct_long(z, bt):
    return (_COS36.T @ (z * window(bt))) / 9.0


def _mdct_short(z):
    out = np.zeros(18)
    for w in range(3):
        out[w::3] = (_COS12.T @ (z[6 + 6 * w : 18 + 6 * w] * _WIN12)) / 3.0
    return out


def forward_hybrid(S_prev, S_cur, g: Granule, rate):
    """The 576 lines (decoder order before reordering, i.e. short bands [window][line]) of one granule from its 18
    subband slots [18, 32] and the previous granule's, with frequency inversion and forward alias butterflies."""
    z = np.concatenate([S_prev, S_cur], axis=0).T.copy()  # [32, 36]
    z[1::2, 1::2] *= -1  # frequency inversion (the decoder's is on the overlap-added output, odd slots of odd bands)
    short = g.window_switching and g.block_type == 2
    xr = np.zeros(576)
    for sb in range(32):
        if short and not (g.mixed and sb < 2):
            xr[18 * sb : 18 * sb + 18] = _mdct_short(z[sb])
        else:
            xr[18 * sb : 18 * sb + 18] = _mdct_long(z[sb], 0 if short else (g.block_type if g.window_switching else 0))
    if not (short and not g.mixed):
        cs = [1 / math.sqrt(1 + c * c) for c in ALIAS_C]
        ca = [c / math.sqrt(1 + c * c) for c in ALIAS_C]
        for sb in range(1, 2 if short else 32):
            for i in range(8):
                bu, bd = xr[18 * sb - 1 - i], xr[18 * sb + i]
                xr[18 * sb - 1 - i] = bu * cs[i] + bd * ca[i]
                xr[18 * sb + i] = bd * cs[i] - bu * ca[i]
    if short:  # from [line][window] interleaved to [window][line] within each short band
        out = xr.copy()
        bs = sfb_bounds(SFB_SHORT[rate])
        for b in range(_short_start(g), 13):
            wd = bs[b + 1] - bs[b]
            for w in range(3):
                for j in range(wd):
                    out[3 * bs[b] + w * wd + j] = xr[3 * bs[b] + 3 * j + w]
        xr = out
    return xr


def gains(g: Granule, sf, rate) -> np.ndarray:
    """2^(quarter steps / 4) of every line (requantize's gain)."""
    return requantize(np.ones(576, dtype=np.int64), g, sf, rate)


def quantize(xr, g: Granule, sf, rate, max_is: int):
    """Lines is = nint((|xr| / gain)^(3/4)) with the smallest global_gain that keeps |is| <= max_is (sets g)."""
    for gg in range(256):
        g.global_gain = gg
        q = np.abs(xr) / gains(g, sf, rate)
        if np.max(q, initial=0) ** 0.75 <= max_is:
            return (np.sign(xr) * np.floor(q**0.75 + 0.5)).astype(np.int64)
    raise ValueError("no global gain fits")


_ENC = {}


def _enc_table(t):
    size, hl, hc = code_table(t)
    return size, hl, hc


def _pair_bits(t, a, b):
    if t == 0:
        return 0 if a == b == 0 else None
    ct = code_table(t)
    if ct is None:
        return None
    size, hl, _ = ct
    lb = LINBITS[t]
    x, y = abs(a), abs(b)
    cap = 15 + (1 << lb) - 1 if lb else size - 1
    if x > cap or y > cap:
        return None
    xi, yi = (min(x, 15), min(y, 15)) if lb else (x, y)
    return hl[xi * size + yi] + (lb if lb and x >= 15 else 0) + (lb if lb and y >= 15 else 0) + (x > 0) + (y > 0)


def best_table(pairs, allowed=None):
    """The table (of `allowed`, default all) that codes the pairs in the fewest bits."""
    best = (None, 0)
    for t in allowed if allowed is not None else [0, 1, 2, 3, 5, 6, 7, 8, 9, 10, 11, 12, 13, 15, *range(16, 32)]:
        n = 0
        for a, b in pairs:
            c = _pair_bits(t, a, b)
            if c is None:
                n = None
                break
            n += c
        if n is not None and (best[0] is None or n < best[1]):
            best = (t, n)
    if best[0] is None:
        raise ValueError("no table codes these values")
    return best[0]


def _write_pair(bw, t, a, b):
    if t == 0:
        return
    size, hl, hc = code_table(t)
    lb = LINBITS[t]
    x, y = abs(a), abs(b)
    xi, yi = (min(x, 15), min(y, 15)) if lb else (x, y)
    bw.write(hc[xi * size + yi], hl[xi * size + yi])
    for v, vi in ((a, xi), (b, yi)):
        if lb and vi == 15:
            bw.write(abs(v) - 15, lb)
        if v:
            bw.write(1 if v < 0 else 0, 1)


def write_granule(bw, g: Granule, sf, scfsi, gr, lines, rate, tables=None, count1=None, region_counts=(5, 5)):
    """Scalefactors and Huffman data of one granule and channel into bw; sets the side-info fields that follow from
    the data (part2_3_length, big_values, tables, region counts, count1 table).  tables: the big-values tables to
    use (chosen by bit count when None); count1: 0 (A), 1 (B) or None (the shorter)."""
    start = len(bw.bits)
    s1, s2 = SLEN[g.scalefac_compress]
    if g.window_switching and g.block_type == 2:
        if g.mixed:
            for b in range(8):
                bw.write(sf["l"][b], s1)
        for b in range(3 if g.mixed else 0, 12):
            for w in range(3):
                bw.write(sf["s"][b][w], s1 if b < 6 else s2)
    else:
        for k, (a, e) in enumerate([(0, 6), (6, 11), (11, 16), (16, 21)]):
            if not (gr == 1 and scfsi[k]):
                for b in range(a, e):
                    bw.write(sf["l"][b], s1 if k < 2 else s2)
    x = [int(v) for v in lines]
    nz = [i for i in range(576) if x[i]]
    last = nz[-1] if nz else -1
    big = [i for i in range(576) if abs(x[i]) > 1]
    bv = ((big[-1] + 2) // 2) if big else 0
    # the count1 quadruples from 2 bv must end by 576: else the big-values region takes the tail
    while last >= 2 * bv and 2 * bv + 4 * ((last - 2 * bv) // 4 + 1) > 576:
        bv += 1
    if bv > 288:
        raise ValueError("big_values > 288")
    g.big_values = bv
    if g.window_switching:
        r1, r2 = 36, 576
    else:
        g.region0_count, g.region1_count = region_counts
        b = sfb_bounds(SFB_LONG[rate])
        r1 = b[min(g.region0_count + 1, 22)]
        r2 = b[min(g.region0_count + g.region1_count + 2, 22)]
    regions = [(0, min(r1, 2 * bv)), (min(r1, 2 * bv), min(r2, 2 * bv)), (min(r2, 2 * bv), 2 * bv)]
    chosen = []
    for k, (a, e) in enumerate(regions[: 2 if g.window_switching else 3]):
        pairs = [(x[i], x[i + 1]) for i in range(a, e, 2)]
        chosen.append(tables[k] if tables is not None else best_table(pairs))
    g.table_select = tuple(chosen) + ((0,) if g.window_switching else ())
    for k, (a, e) in enumerate(regions[: len(chosen)]):
        for i in range(a, e, 2):
            _write_pair(bw, chosen[k], x[i], x[i + 1])
    quads = [x[i : i + 4] for i in range(2 * bv, last + 1, 4)] if last >= 2 * bv else []
    costs = []
    for tab in (COUNT1_A, COUNT1_B):
        costs.append(sum(tab[0][8 * abs(q[0]) + 4 * abs(q[1]) + 2 * abs(q[2]) + abs(q[3])] + sum(v != 0 for v in q)
                         for q in quads))
    g.count1_table = count1 if count1 is not None else int(costs[1] < costs[0])
    hl, hc = (COUNT1_B if g.count1_table else COUNT1_A)
    for q in quads:
        v = 8 * abs(q[0]) + 4 * abs(q[1]) + 2 * abs(q[2]) + abs(q[3])
        bw.write(hc[v], hl[v])
        for u in q:
            if u:
                bw.write(1 if u < 0 else 0, 1)
    g.part2_3_length = len(bw.bits) - start


def scalefac_compress_for(sf, g: Granule):
    """The smallest scalefac_compress whose slen1 / slen2 hold the scalefactors."""
    if g.window_switching and g.block_type == 2:
        lo = [sf["l"][b] for b in range(8)] * g.mixed + [sf["s"][b][w] for b in range(3 if g.mixed else 0, 6)
                                                          for w in range(3)]
        hi = [sf["s"][b][w] for b in range(6, 12) for w in range(3)]
    else:
        lo, hi = sf["l"][:11], sf["l"][11:21]
    for k, (s1, s2) in enumerate(SLEN):
        if max(lo, default=0) < (1 << s1) and max(hi, default=0) < (1 << s2):
            return k
    raise ValueError("scalefactors too large")


def crc16(data: bytes) -> int:
    """CRC-16 of the header's last two bytes and the side info (polynomial 0x8005, initial 0xFFFF)."""
    c = 0xFFFF
    for byte in data:
        for i in range(7, -1, -1):
            bit = (byte >> i) & 1
            top = (c >> 15) & 1
            c = (c << 1) & 0xFFFF
            if top ^ bit:
                c ^= 0x8005
    return c


def header_word(bitrate_index, rate, padding, mode, mode_ext, crc):
    return (0x7FF << 21) | (3 << 19) | (1 << 17) | ((0 if crc else 1) << 16) | (bitrate_index << 12) | \
        (RATES.index(rate) << 10) | (padding << 9) | (mode << 6) | (mode_ext << 4)


@dataclasses.dataclass
class GranuleSpec:
    """What the encoder is told to write for one granule (both channels)."""
    block_type: int = 0          # 0 long, 1 start, 2 short, 3 stop
    mixed: int = 0
    subblock_gain: tuple = (0, 0, 0)
    preflag: int = 0
    scalefac_scale: int = 0
    scalefactors: str = "zero"   # "zero" or "random"
    tables: tuple = None         # forced big-values tables
    count1: int = None


def encode(signal: np.ndarray, rate: int, grans, *, bitrate=320, ms=False, crc=False, scfsi=None, max_is=30,
           reservoir=True, stuff_to=None, seed=0):
    """Frames of `signal` ([samples] mono or [samples, 2] stereo in [-1, 1]; 1152 samples per frame, zero padded) with
    granule g coded as grans[g % len(grans)] (GranuleSpec).  bitrate: kbit/s, or a list per frame (VBR).  ms: M/S
    stereo in every frame.  scfsi: the four scfsi bits of every channel (granule 1 then reuses granule 0's
    scalefactors of those bands; long blocks only).  reservoir: main data may begin up to 511 bytes back (as early as
    the earlier frames' free bytes allow, or at most stuff_to bytes back), else main_data_begin is 0.  Returns
    (stream bytes, list of per-frame main_data_begin)."""
    x = signal if signal.ndim == 2 else signal[:, None]
    nch = x.shape[1]
    n_frames = -(-len(x) // 1152)
    x = np.concatenate([x, np.zeros((n_frames * 1152 - len(x), nch))])
    rng = np.random.default_rng(seed)
    S = [analysis(x[:, c]) for c in range(nch)]  # [slots, 32]
    G = 2 * n_frames
    S = [np.concatenate([np.zeros((18, 32)), s]) for s in S]  # granule -1 is silence
    frames = []
    main = BitWriter()
    main_bytes = bytearray()
    slot_pos = 0
    begins = []
    for f in range(n_frames):
        br = bitrate[f % len(bitrate)] if isinstance(bitrate, (list, tuple)) else bitrate
        bi = BITRATES.index(br)
        mode = 3 if nch == 1 else 1
        def frame_bits(mi, f=f):
            si = SideInfo(0, 0, [list(scfsi or (0, 0, 0, 0)) for _ in range(nch)], [[None] * nch for _ in range(2)])
            bw = BitWriter()
            prev_sf = [None] * nch
            for gr in range(2):
                spec = grans[(2 * f + gr) % len(grans)]
                gi = 2 * f + gr
                xrs = []
                for c in range(nch):
                    g = Granule(window_switching=int(spec.block_type != 0), block_type=spec.block_type,
                                mixed=spec.mixed if spec.block_type == 2 else 0, subblock_gain=spec.subblock_gain
                                if spec.block_type == 2 else (0, 0, 0), preflag=spec.preflag,
                                scalefac_scale=spec.scalefac_scale)
                    xrs.append((g, forward_hybrid(S[c][18 * gi : 18 * gi + 18], S[c][18 * gi + 18 : 18 * gi + 36], g,
                                                  rate)))
                if ms and nch == 2:
                    (g0, l), (g1, r) = xrs
                    xrs = [(g0, (l + r) / math.sqrt(2)), (g1, (l - r) / math.sqrt(2))]
                for c, (g, xr) in enumerate(xrs):
                    if spec.scalefactors == "random":
                        sf = {"l": [int(v) for v in rng.integers(0, 8, 22)],
                              "s": [[int(v) for v in rng.integers(0, 4, 3)] for _ in range(13)]}
                        sf["l"][21] = 0
                        sf["s"][12] = [0, 0, 0]
                    else:
                        sf = {"l": [0] * 22, "s": [[0] * 3 for _ in range(13)]}
                    if gr == 1 and scfsi and not g.window_switching and prev_sf[c] is not None:
                        for k, (a, e) in enumerate([(0, 6), (6, 11), (11, 16), (16, 21)]):
                            if scfsi[k]:
                                sf["l"][a:e] = prev_sf[c]["l"][a:e]
                    g.scalefac_compress = scalefac_compress_for(sf, g)
                    lines = quantize(xr, g, sf, rate, mi)
                    write_granule(bw, g, sf, si.scfsi[c], gr, lines, rate, spec.tables, spec.count1)
                    si.gr[gr][c] = g
                    prev_sf[c] = sf
            return bw.getvalue(), si

        slots = 144000 * br // rate - 4 - (2 if crc else 0) - (17 if nch == 1 else 32)
        # place this frame's main data: as early as the reservoir allows
        free = slot_pos - len(main_bytes)
        cap = 511 if reservoir else 0
        if stuff_to is not None:
            cap = min(cap, stuff_to)
        if free > cap:
            main_bytes += bytes(free - cap)
        begin = slot_pos - len(main_bytes)
        mi = max_is  # the rate loop: a coarser quantiser until the frame's main data fits
        data, si = frame_bits(mi)
        while len(main_bytes) + len(data) > slot_pos + slots:
            if mi <= 1:
                raise ValueError(f"frame {f}: {len(data)} bytes of main data do not fit at {br} kbit/s")
            mi = max(1, mi * 2 // 3)
            data, si = frame_bits(mi)
        main_bytes += data
        si.main_data_begin = begin
        begins.append(begin)
        hw = header_word(bi, rate, 0, mode, 2 if (ms and nch == 2) else 0, crc)
        side = write_side_info(si, nch)
        frames.append([hw.to_bytes(4, "big"), side, slot_pos, slots])
        slot_pos += slots
    main_bytes += bytes(max(0, slot_pos - len(main_bytes)))
    out = bytearray()
    for hb, side, pos, slots in frames:
        out += hb
        if crc:
            out += crc16(hb[2:4] + side).to_bytes(2, "big")
        out += side + main_bytes[pos : pos + slots]
    return bytes(out), begins
