// MPEG-1 Layer III decoding (ISO/IEC 11172-3), shared by the device kernels (kernels_mp3.cu), the host staging and the
// host test hook (api_mp3.cu).  Every step is a __host__ __device__ function of one "lane" (a thread on the device, a
// loop index on the host), so the host hook runs the kernels' own arithmetic.
//
// Layout of a staged stream (bt_mp3_frame, include/beatthis.h): the main data of every frame (its bytes after header,
// CRC and side info) back to back, and per frame its raw side info and main-data start in that compacted stream
// (cumulative bytes minus main_data_begin, negative when the reservoir reaches before the stream).  The granule and
// channel (gr, ch) of frame f then start at bit 8 * main_start + the part2_3_length of the frame's earlier granules and
// channels, so the device never sees the bit reservoir.
#pragma once

#include <cmath>
#include <cstdint>

#include "../../include/beatthis.h"

#if defined(__CUDACC__)
#define BT_MP3_HD __host__ __device__ __forceinline__
#else
#define BT_MP3_HD inline
#endif

namespace bt {
namespace mp3 {

// Tables indexed at run time live in constant memory on the device (an indexed local array would go to local memory)
// and in a static array on the host; BT_MP3_AT(name) is the one the caller's side reads.
#define BT_MP3_TABLE(T, name, N, ...)                  \
  static __constant__ const T name##_dev[N] = __VA_ARGS__; \
  static const T name##_host[N] = __VA_ARGS__;
#if defined(__CUDA_ARCH__)
#define BT_MP3_AT(name) name##_dev
#else
#define BT_MP3_AT(name) name##_host
#endif

constexpr int kLines = 576;
constexpr int kSlots = 18;   // time slots of a granule
constexpr int kBlock = 36;   // windowed IMDCT values per subband

// ---- headers ---------------------------------------------------------------------------------------------------------
struct Header {
  int bitrate, sample_rate, padding, crc, mode, mode_ext, channels, length, side_bytes;
};

BT_MP3_TABLE(int16_t, kBitrates, 15, {0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320})

// The MPEG-1 Layer III header h (big-endian word), or false: no sync, another version or layer, free format or a
// reserved value.
BT_MP3_HD bool parse_header(uint32_t h, Header* o) {
  if ((h >> 21) != 0x7FF || ((h >> 19) & 3) != 3 || ((h >> 17) & 3) != 1) return false;
  const int bi = (h >> 12) & 15, si = (h >> 10) & 3;
  if (bi == 0 || bi == 15 || si == 3 || (h & 3) == 2) return false;
  o->bitrate = BT_MP3_AT(kBitrates)[bi];
  o->sample_rate = si == 0 ? 44100 : si == 1 ? 48000 : 32000;
  o->padding = (h >> 9) & 1;
  o->crc = !((h >> 16) & 1);
  o->mode = (h >> 6) & 3;
  o->mode_ext = (h >> 4) & 3;
  o->channels = o->mode == 3 ? 1 : 2;
  o->length = 144000 * o->bitrate / o->sample_rate + o->padding;
  o->side_bytes = o->channels == 1 ? 17 : 32;
  return true;
}

BT_MP3_HD int rate_index(int sample_rate) { return sample_rate == 44100 ? 0 : sample_rate == 48000 ? 1 : 2; }

// scalefactor band starts, long (23) and short (14, per window) at 44.1, 48 and 32 kHz
BT_MP3_TABLE(int16_t, kSfbLong, 3 * 23,
             {0, 4, 8, 12, 16, 20, 24, 30, 36, 44, 52, 62, 74, 90, 110, 134, 162, 196, 238, 288, 342, 418, 576,
              0, 4, 8, 12, 16, 20, 24, 30, 36, 42, 50, 60, 72, 88, 106, 128, 156, 190, 230, 276, 330, 384, 576,
              0, 4, 8, 12, 16, 20, 24, 30, 36, 44, 54, 66, 82, 102, 126, 156, 194, 240, 296, 364, 448, 550, 576})
BT_MP3_TABLE(int16_t, kSfbShort, 3 * 14,
             {0, 4, 8, 12, 16, 22, 30, 40, 52, 66, 84, 106, 136, 192, 0, 4, 8, 12, 16, 22, 28, 38, 50, 64, 80, 100, 126,
              192, 0, 4, 8, 12, 16, 22, 30, 42, 58, 78, 104, 138, 180, 192})
BT_MP3_HD int sfb_long(int ri, int b) { return BT_MP3_AT(kSfbLong)[ri * 23 + b]; }
BT_MP3_HD int sfb_short(int ri, int b) { return BT_MP3_AT(kSfbShort)[ri * 14 + b]; }

// ---- side info -------------------------------------------------------------------------------------------------------
struct Granule {
  int part2_3, big_values, global_gain, sfc, block_type, mixed, short_blocks, table[3], subblock[3], region1, region2,
      preflag, sf_scale, count1;
};

struct Bits {  // big-endian bit reader over p[0 .. n) (reads past the end give zeros; the caller bounds its reads)
  const uint8_t* p;
  int64_t n, pos;
  BT_MP3_HD uint32_t peek(int k) const {  // k <= 24
    uint32_t v = 0;
    const int64_t b = pos >> 3;
    for (int i = 0; i < 4; ++i) v = (v << 8) | ((b + i >= 0 && b + i < n) ? p[b + i] : 0u);
    return (v << (pos & 7)) >> (32 - k);
  }
  BT_MP3_HD uint32_t read(int k) {
    if (k == 0) return 0;
    const uint32_t v = peek(k);
    pos += k;
    return v;
  }
};

// Side info of granule gr, channel ch of a frame (side: its 17 or 32 bytes), its scfsi bits and main_data_begin.
BT_MP3_HD void parse_side(const uint8_t* side, int nch, int gr, int ch, int ri, Granule* g, int* scfsi,
                          int* main_data_begin) {
  Bits b{side, nch == 1 ? 17 : 32, 0};
  *main_data_begin = static_cast<int>(b.read(9));
  b.pos += nch == 1 ? 5 : 3;
  b.pos += 4 * ch;
  *scfsi = static_cast<int>(b.read(4));
  b.pos = 9 + (nch == 1 ? 5 : 3) + 4 * nch + 59 * (gr * nch + ch);
  g->part2_3 = b.read(12);
  g->big_values = b.read(9);
  g->global_gain = b.read(8);
  g->sfc = b.read(4);
  const int ws = b.read(1);
  g->block_type = g->mixed = 0;
  g->subblock[0] = g->subblock[1] = g->subblock[2] = 0;
  if (ws) {
    g->block_type = b.read(2);
    g->mixed = b.read(1);
    g->table[0] = b.read(5);
    g->table[1] = b.read(5);
    g->table[2] = 0;
    for (int w = 0; w < 3; ++w) g->subblock[w] = b.read(3);
    g->region1 = 36;
    g->region2 = kLines;
    if (g->block_type == 0) g->block_type = -1;  // window switching with block type 0: malformed
  } else {
    for (int r = 0; r < 3; ++r) g->table[r] = b.read(5);
    const int r0 = b.read(4), r1 = b.read(3);
    g->region1 = sfb_long(ri, r0 + 1 < 22 ? r0 + 1 : 22);
    g->region2 = sfb_long(ri, r0 + r1 + 2 < 22 ? r0 + r1 + 2 : 22);
  }
  g->short_blocks = g->block_type == 2;
  g->preflag = b.read(1);
  g->sf_scale = b.read(1);
  g->count1 = b.read(1);
}

// ---- Huffman lookup tables -----------------------------------------------------------------------------------------
// One flat uint32 array holds every table as nested lookups: an entry of a level of `k` bits is a leaf
// (bit 31, bits 16..20: code bits used at this level, bits 0..15: symbol) or a link (bits 24..28: bits of the next
// level, bits 0..23: its first entry).  Slot t (0..31 big-values tables by table_select, 32 and 33 the count1 tables A
// and B) starts at entry lut[kLutEntries + t] with kFirstBits bits; tables 0, 4 and 14 have none (never read).
constexpr int kFirstBits = 7;
constexpr int kLutEntries = 4608;   // enough for every table (api_mp3.cu checks)

BT_MP3_HD bool huff_decode(const uint32_t* lut, uint32_t start, Bits& b, int* sym) {
  int k = kFirstBits;
  uint32_t base = start;
  for (int guard = 0; guard < 4; ++guard) {
    const uint32_t e = lut[base + b.peek(k)];
    if (e & 0x80000000u) {
      b.pos += (e >> 16) & 31;
      *sym = static_cast<int>(e & 0xFFFF);
      return true;
    }
    if (e == 0) return false;
    b.pos += k;
    k = (e >> 24) & 31;
    base = e & 0xFFFFFF;
  }
  return false;
}

BT_MP3_TABLE(int8_t, kLinbits, 32, {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 2, 3, 4, 6, 8, 10, 13, 4, 5, 6, 7,
                                     8, 9, 11, 13})
BT_MP3_HD int linbits(int t) { return BT_MP3_AT(kLinbits)[t]; }

// ---- the decoded granule record (global scratch; one per frame, granule and channel) ---------------------------------
struct GranuleRec {
  int16_t lines[kLines];
  uint8_t sf[40];       // long blocks: sf[b], b < 22; short bands: sf[3 * b + w]
  uint8_t sf_long[8];   // mixed blocks: the long bands 0..7
  int16_t global_gain;
  int8_t block_type, mixed, short_blocks, preflag, sf_scale, zero;
  int8_t subblock[3];
  int8_t pad_;
};

BT_MP3_TABLE(int8_t, kSlen1, 16, {0, 0, 0, 0, 3, 1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4})
BT_MP3_TABLE(int8_t, kSlen2, 16, {0, 1, 2, 3, 0, 1, 2, 3, 1, 2, 3, 1, 2, 3, 2, 3})

// Decodes granule gr of channel ch of one frame: scalefactors (prev: the granule 0 record, for scfsi) and Huffman
// lines into rec.  start_bit: its first bit in the stream's main data (negative: a zero spectrum); false when malformed.
BT_MP3_HD bool decode_granule(const uint8_t* main, int64_t main_bytes, int64_t start_bit, const Granule& g, int scfsi,
                              int gr, int ri, const GranuleRec* prev, const uint32_t* lut, GranuleRec* rec) {
  rec->global_gain = static_cast<int16_t>(g.global_gain);
  rec->block_type = static_cast<int8_t>(g.block_type);
  rec->mixed = static_cast<int8_t>(g.mixed);
  rec->short_blocks = static_cast<int8_t>(g.short_blocks);
  rec->preflag = static_cast<int8_t>(g.preflag);
  rec->sf_scale = static_cast<int8_t>(g.sf_scale);
  for (int w = 0; w < 3; ++w) rec->subblock[w] = static_cast<int8_t>(g.subblock[w]);
  for (int i = 0; i < 40; ++i) rec->sf[i] = 0;
  for (int i = 0; i < 8; ++i) rec->sf_long[i] = 0;
  for (int i = 0; i < kLines; ++i) rec->lines[i] = 0;
  rec->zero = 0;
  if (g.block_type < 0 || g.big_values > 288) return false;
  if (start_bit < 0) {  // the reservoir reaches before the stream: a zero spectrum
    rec->zero = 1;
    return true;
  }
  const int64_t end = start_bit + g.part2_3;
  if (end > 8 * main_bytes) return false;
  Bits b{main, main_bytes, start_bit};
  const int s1 = BT_MP3_AT(kSlen1)[g.sfc], s2 = BT_MP3_AT(kSlen2)[g.sfc];
  if (g.short_blocks) {
    int first = 0;
    if (g.mixed) {
      for (int sb = 0; sb < 8; ++sb) rec->sf_long[sb] = static_cast<uint8_t>(b.read(s1));
      first = 3;
    }
    for (int sb = first; sb < 12; ++sb)
      for (int w = 0; w < 3; ++w) rec->sf[3 * sb + w] = static_cast<uint8_t>(b.read(sb < 6 ? s1 : s2));
  } else {
    for (int k = 0; k < 4; ++k)
      for (int sb = k == 0 ? 0 : 1 + 5 * k; sb < 6 + 5 * k; ++sb)
        rec->sf[sb] = (gr == 1 && ((scfsi >> (3 - k)) & 1)) ? prev->sf[sb]
                                                              : static_cast<uint8_t>(b.read(k < 2 ? s1 : s2));
  }
  if (b.pos > end) return false;
  const int bv = 2 * g.big_values;
  for (int i = 0; i < bv; i += 2) {
    const int t = i < g.region1 ? g.table[0] : i < g.region2 ? g.table[1] : g.table[2];
    if (t == 0) continue;
    if (t == 4 || t == 14) return false;
    const uint32_t start = lut[kLutEntries + t];
    int sym;
    if (!huff_decode(lut, start, b, &sym)) return false;
    int v[2] = {sym >> 4, sym & 15};
    const int lb = linbits(t);
    for (int k = 0; k < 2; ++k) {
      if (lb && v[k] == 15) v[k] += static_cast<int>(b.read(lb));
      if (v[k] && b.read(1)) v[k] = -v[k];
      rec->lines[i + k] = static_cast<int16_t>(v[k]);
    }
    if (b.pos > end) return false;
  }
  int i = bv;
  const uint32_t c1 = lut[kLutEntries + 32 + g.count1];
  while (i + 4 <= kLines && b.pos < end) {
    int q;
    if (!huff_decode(lut, c1, b, &q)) return false;
    int v[4];
    for (int k = 0; k < 4; ++k) {
      v[k] = (q >> (3 - k)) & 1;
      if (v[k] && b.read(1)) v[k] = -v[k];
    }
    if (b.pos > end) break;  // a quadruple that overshoots part2_3_length is dropped
    for (int k = 0; k < 4; ++k) rec->lines[i + k] = static_cast<int16_t>(v[k]);
    i += 4;
  }
  return true;
}

// ---- hybrid filter bank (one granule, both channels) -----------------------------------------------------------------
BT_MP3_TABLE(int8_t, kPretab, 22, {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 3, 2, 0})
BT_MP3_HD int pretab(int b) { return BT_MP3_AT(kPretab)[b]; }

// The band of line i: long band (returns it, *win = -1) or short band (*win = window, *pos = position in the band)
BT_MP3_HD int band_of(const GranuleRec& r, int ri, int i, int* win, int* pos) {
  if (!r.short_blocks || (r.mixed && i < 36)) {
    int b = 0;
    while (b < 21 && sfb_long(ri, b + 1) <= i) ++b;
    *win = -1;
    *pos = i - sfb_long(ri, b);
    return b;
  }
  int b = r.mixed ? 3 : 0;
  while (b < 12 && 3 * sfb_short(ri, b + 1) <= i) ++b;
  const int width = sfb_short(ri, b + 1) - sfb_short(ri, b);
  const int off = i - 3 * sfb_short(ri, b);
  *win = off / width;
  *pos = off % width;
  return b;
}

// The gain of a band as an integer e of quarter steps, gain = 2^(e / 4): global_gain - 210 (- 8 subblock_gain[w] in a
// short band) minus the scalefactor (+ preflag's pretab in a long band) times 2 or 4 quarter steps (scalefac_scale 0
// or 1).
BT_MP3_HD int gain_quarters(const GranuleRec& r, int band, int win) {
  const int mult = r.sf_scale ? 4 : 2;  // quarter steps per scalefactor unit
  if (win < 0) {
    const int sf = (r.short_blocks && r.mixed) ? r.sf_long[band] : r.sf[band];
    return r.global_gain - 210 - mult * (sf + r.preflag * pretab(band));
  }
  return r.global_gain - 210 - 8 * r.subblock[win] - mult * r.sf[3 * band + win];
}

BT_MP3_HD float requant(int q, int quarters) {
  if (q == 0) return 0.f;
  const double a = q < 0 ? -q : q;
  const double m = a * cbrt(a) * exp2(0.25 * quarters);
  return static_cast<float>(q < 0 ? -m : m);
}

// Intensity position of line i of the right channel (7: not coded) given its band
BT_MP3_HD int is_pos(const GranuleRec& r, int band, int win) {
  if (win < 0) {
    if (r.short_blocks && r.mixed) return r.sf_long[band];
    return r.sf[band < 21 ? band : 20];
  }
  return r.sf[3 * (band < 12 ? band : 11) + win];
}

// Short-block reorder: the input line feeding reordered line i ([band][3 * pos + window] from [band][window][pos])
BT_MP3_HD int reorder_src(const GranuleRec& r, int ri, int i) {
  if (!r.short_blocks || (r.mixed && i < 36)) return i;
  int b = r.mixed ? 3 : 0;
  while (b < 12 && 3 * sfb_short(ri, b + 1) <= i) ++b;
  const int width = sfb_short(ri, b + 1) - sfb_short(ri, b);
  const int off = i - 3 * sfb_short(ri, b);
  return 3 * sfb_short(ri, b) + (off % 3) * width + off / 3;
}

BT_MP3_TABLE(float, kAliasCs, 8, {0.857492925712544f, 0.881741997317705f, 0.949628649102733f, 0.983314592491790f,
                                 0.995517816067586f, 0.999160558178148f, 0.999899195244447f, 0.999993155070280f})
BT_MP3_TABLE(float, kAliasCa, 8, {-0.514495755427526f, -0.471731968564936f, -0.313377454203902f, -0.181913199610981f,
                                 -0.094574192526420f, -0.040965582885304f, -0.014198568572471f, -0.003699974673760f})
BT_MP3_HD float alias_cs(int k) { return BT_MP3_AT(kAliasCs)[k]; }
BT_MP3_HD float alias_ca(int k) { return BT_MP3_AT(kAliasCa)[k]; }

// Line i (0..575) after alias reduction, from the reordered spectrum x
BT_MP3_HD float antialias(const float* x, const GranuleRec& r, int i) {
  const int sb = i / 18, k = i % 18;
  const int limit = r.short_blocks ? (r.mixed ? 2 : 0) : 32;  // subbands whose lower boundary is reduced: 1 .. limit-1
  if (k < 8 && sb >= 1 && sb < limit) {  // lower side of boundary sb: bd = x[18 sb + k]
    const float bu = x[18 * sb - 1 - k], bd = x[i];
    return bd * alias_cs(k) + bu * alias_ca(k);
  }
  if (k >= 10 && sb + 1 < limit) {  // upper side of boundary sb + 1: bu = x[18 (sb + 1) - 1 - j]
    const int j = 17 - k;
    const float bu = x[i], bd = x[18 * (sb + 1) + j];
    return bu * alias_cs(j) - bd * alias_ca(j);
  }
  return x[i];
}

// The transform tables of the IMDCT: cos36[n * 18 + k] = cos(pi / 72 (2n + 1 + 18)(2k + 1)), cos12[m * 6 + k] =
// cos(pi / 24 (2m + 1 + 6)(2k + 1)), win[bt * 36 + n]: the long windows of block types 0, 1 and 3 (slot 2: the short
// window sin(pi / 12 (m + 1/2)) at n = m < 12).  The kernels keep them in shared memory.
constexpr int kTransformTable = 36 * 18 + 12 * 6 + 4 * 36;
// The float tables the kernels stage once per call: the transform tables, then D[0 .. 511] of the synthesis window,
// then N[64][32] of the matrixing (synth_window, synth_cos below)
constexpr int kWindowAt = kTransformTable, kCosAt = kTransformTable + 512, kFloatTables = kTransformTable + 512 + 64 * 32;

// cos(pi x) and sin(pi x) in float64 (the device's cospi / sinpi need no argument reduction, so no local memory)
BT_MP3_HD double cos_pi(double x) {
#if defined(__CUDA_ARCH__)
  return cospi(x);
#else
  return std::cos(3.14159265358979323846 * x);
#endif
}
BT_MP3_HD double sin_pi(double x) {
#if defined(__CUDA_ARCH__)
  return sinpi(x);
#else
  return std::sin(3.14159265358979323846 * x);
#endif
}

BT_MP3_HD float transform_table_value(int i) {
  if (i < 36 * 18) return static_cast<float>(cos_pi((2 * (i / 18) + 1 + 18) * (2 * (i % 18) + 1) / 72.0));
  i -= 36 * 18;
  if (i < 12 * 6) return static_cast<float>(cos_pi((2 * (i / 6) + 1 + 6) * (2 * (i % 6) + 1) / 24.0));
  i -= 12 * 6;
  const int bt = i / 36, n = i % 36;
  if (bt == 2) return n < 12 ? static_cast<float>(sin_pi((n + 0.5) / 12)) : 0.f;
  if (bt == 1 && n >= 18) return n < 24 ? 1.f : n < 30 ? static_cast<float>(sin_pi((n - 18 + 0.5) / 12)) : 0.f;
  if (bt == 3 && n < 18) return n < 6 ? 0.f : n < 12 ? static_cast<float>(sin_pi((n - 6 + 0.5) / 12)) : 1.f;
  return static_cast<float>(sin_pi((n + 0.5) / 36));
}

// Windowed IMDCT value n (0..35) of subband sb from its 18 aliased lines X (tt: the transform tables)
BT_MP3_HD float imdct_value(const float* X, const GranuleRec& r, int sb, int n, const float* tt) {
  const bool short_sb = r.short_blocks && !(r.mixed && sb < 2);
  const float* cos36 = tt;
  const float* cos12 = tt + 36 * 18;
  const float* win = tt + 36 * 18 + 12 * 6;
  if (!short_sb) {
    const float w = win[(r.short_blocks ? 0 : r.block_type) * 36 + n];
    float s = 0.f;
    for (int k = 0; k < 18; ++k) s += X[k] * cos36[n * 18 + k];
    return s * w;
  }
  float s = 0.f;
  for (int w = 0; w < 3; ++w) {
    const int m = n - 6 - 6 * w;
    if (m < 0 || m >= 12) continue;
    float y = 0.f;
    for (int k = 0; k < 6; ++k) y += X[3 * k + w] * cos12[m * 6 + k];
    s += y * win[2 * 36 + m];
  }
  return s;
}

// ---- polyphase synthesis ---------------------------------------------------------------------------------------------
// D[i] * 65536 for i = 0 .. 256 (Table 3-B.3 of the standard); D[512 - i] = D[i] when 64 divides i, else -D[i]
BT_MP3_TABLE(int32_t, kWindowHalf, 257, {
      0, -1, -1, -1, -1, -1, -1, -2, -2, -2, -2, -3, -3, -4, -4, -5, -5, -6, -7, -7, -8, -9, -10, -11, -13, -14, -16,
      -17, -19, -21, -24, -26, -29, -31, -35, -38, -41, -45, -49, -53, -58, -63, -68, -73, -79, -85, -91, -97, -104,
      -111, -117, -125, -132, -139, -147, -154, -161, -169, -176, -183, -190, -196, -202, -208, 213, 218, 222, 225, 227,
      228, 228, 227, 224, 221, 215, 208, 200, 189, 177, 163, 146, 127, 106, 83, 57, 29, -2, -36, -72, -111, -153, -197,
      -244, -294, -347, -401, -459, -519, -581, -645, -711, -779, -848, -919, -991, -1064, -1137, -1210, -1283, -1356,
      -1428, -1498, -1567, -1634, -1698, -1759, -1817, -1870, -1919, -1962, -2001, -2032, -2057, -2075, -2085, -2087,
      -2080, -2063, 2037, 2000, 1952, 1893, 1822, 1739, 1644, 1535, 1414, 1280, 1131, 970, 794, 605, 402, 185, -45, -288,
      -545, -814, -1095, -1388, -1692, -2006, -2330, -2663, -3004, -3351, -3705, -4063, -4425, -4788, -5153, -5517,
      -5879, -6237, -6589, -6935, -7271, -7597, -7910, -8209, -8491, -8755, -8998, -9219, -9416, -9585, -9727, -9838,
      -9916, -9959, -9966, -9935, -9863, -9750, -9592, -9389, -9139, -8840, -8492, -8092, -7640, -7134, 6574, 5959, 5288,
      4561, 3776, 2935, 2037, 1082, 70, -998, -2122, -3300, -4533, -5818, -7154, -8540, -9975, -11455, -12980, -14548,
      -16155, -17799, -19478, -21189, -22929, -24694, -26482, -28289, -30112, -31947, -33791, -35640, -37489, -39336,
      -41176, -43006, -44821, -46617, -48390, -50137, -51853, -53534, -55178, -56778, -58333, -59838, -61289, -62684,
      -64019, -65290, -66494, -67629, -68692, -69679, -70590, -71420, -72169, -72835, -73415, -73908, -74313, -74630,
      -74856, -74992, 75038})
BT_MP3_HD int32_t window_half(int i) { return BT_MP3_AT(kWindowHalf)[i]; }

BT_MP3_HD float synth_window(int i) {
  const int32_t v = i <= 256 ? window_half(i) : ((512 - i) % 64 == 0 ? window_half(512 - i) : -window_half(512 - i));
  return static_cast<float>(v) * (1.f / 65536.f);
}

BT_MP3_HD float synth_cos(int i, int k) {  // N[i][k] = cos((16 + i)(2k + 1) pi / 64), i < 64, k < 32
  return static_cast<float>(cos_pi((16 + i) * (2 * k + 1) / 64.0));
}

// Subband sample of subband sb at time slot `slot` of granule g (slot < 0: the slots of granule g - 1) of channel c
// (blocks: [granule][channels][32][36]): the slot's block value plus the previous granule's tail (zeros before the
// first granule), then frequency inversion.
BT_MP3_HD float slot_sample(const float* blocks, int nch, int c, int64_t g, int slot, int sb) {
  if (slot < 0) {
    --g;
    slot += kSlots;
  }
  if (g < 0) return 0.f;
  float v = blocks[((g * nch + c) * 32 + sb) * kBlock + slot];
  if (g > 0) v += blocks[(((g - 1) * nch + c) * 32 + sb) * kBlock + 18 + slot];
  return ((sb & 1) && (slot & 1)) ? -v : v;
}

// V[i] of one time slot: sum over k of N[i][k] S[k] (ncos: N, [64][32])
BT_MP3_HD float matrix_value(const float* S, const float* ncos, int i) {
  float v = 0.f;
  for (int k = 0; k < 32; ++k) v += ncos[i * 32 + k] * S[k];
  return v;
}

// PCM sample j of time slot u (V: [slots][64], slot u and the 15 before it; win: D[0 .. 511])
BT_MP3_HD float window_sum(const float* V, const float* win, int u, int j) {
  float v = 0.f;
  for (int i = 0; i < 8; ++i) {
    v += V[(u - 2 * i) * 64 + j] * win[64 * i + j];
    v += V[(u - 2 * i - 1) * 64 + 32 + j] * win[64 * i + 32 + j];
  }
  return v;
}

// The mono mix of bt_stage_wav_files: the channels summed in float64, one division, one rounding to fp32
BT_MP3_HD float mono_sample(float s0, float s1, int nch) {
  return nch == 1 ? s0 : static_cast<float>((static_cast<double>(s0) + static_cast<double>(s1)) / 2);
}

// ---- per-lane steps of the hybrid kernel --------------------------------------------------------------------------
// Line i of both channels dequantised into x[c * 576 + i]; bound[0]: the last nonzero line of the right channel's long
// part, bound[1 + w]: the last short band of window w with a nonzero right-channel line (atomic maxima).
BT_MP3_HD void atomic_max_int(int* p, int v) {
#if defined(__CUDA_ARCH__)
  atomicMax(p, v);
#else
  if (v > *p) *p = v;
#endif
}

BT_MP3_HD void hybrid_requant(const GranuleRec* recs, int nch, int ri, int i, float* x, int* bound) {
  for (int c = 0; c < nch; ++c) {
    const GranuleRec& r = recs[c];
    int win, pos;
    const int band = band_of(r, ri, i, &win, &pos);
    const int q = r.lines[i];
    x[c * kLines + i] = requant(q, gain_quarters(r, band, win));
    if (c == 1 && q != 0) atomic_max_int(win < 0 ? &bound[0] : &bound[1 + win], win < 0 ? i : band);
  }
}

// Intensity stereo with ratio = tan(p pi / 12): left = l ratio / (1 + ratio) = l sin / (sin + cos), right = l cos /
// (sin + cos), in float64 for p = 0 .. 6
BT_MP3_TABLE(double, kIsLeft, 7, {0.0, 0.2113248654051871, 0.3660254037844386, 0.5, 0.6339745962155612,
                                  0.788675134594813, 1.0})
BT_MP3_TABLE(double, kIsRight, 7, {1.0, 0.7886751345948129, 0.6339745962155614, 0.5, 0.3660254037844388,
                                   0.21132486540518702, 0.0})

// M/S and intensity stereo of line i in place (header: the frame's header word)
BT_MP3_HD void hybrid_stereo(const GranuleRec* recs, int nch, int ri, uint32_t header, int i, float* x,
                             const int* bound) {
  if (nch != 2 || ((header >> 6) & 3) != 1) return;
  const int ext = (header >> 4) & 3;
  const GranuleRec& r = recs[1];
  int win, pos;
  const int band = band_of(r, ri, i, &win, &pos);
  bool intensity = false;
  if (ext & 1) {
    if (win >= 0) {
      intensity = band > bound[1 + win];
    } else {
      const bool short_nz = r.short_blocks && (bound[1] >= 0 || bound[2] >= 0 || bound[3] >= 0);
      intensity = !short_nz && sfb_long(ri, band) > bound[0];
    }
  }
  const int p = intensity ? is_pos(r, band, win) : 7;
  const float l = x[i], rr = x[kLines + i];
  if (p != 7) {
    x[i] = static_cast<float>(l * BT_MP3_AT(kIsLeft)[p]);
    x[kLines + i] = static_cast<float>(l * BT_MP3_AT(kIsRight)[p]);
  } else if (ext & 2) {
    const float k = 0.70710678118654752f;
    x[i] = (l + rr) * k;
    x[kLines + i] = (l - rr) * k;
  }
}

// ---- per-thread step of the granules kernel ------------------------------------------------------------------------
// Both granules of channel ch of one frame into recs[gr * nch + ch]: false when malformed
BT_MP3_HD bool decode_frame_channel(const uint8_t* main, int64_t main_bytes, int64_t main_start, uint32_t header,
                                    const uint8_t* side, int nch, int ch, int ri, const uint32_t* lut,
                                    GranuleRec* recs) {
  Header h;
  if (!parse_header(header, &h) || h.channels != nch || rate_index(h.sample_rate) != ri) return false;
  if (main_start < -511) return false;  // main_data_begin reaches 511 bytes back at most: the entry is outside its stream
  int64_t bit = 8 * main_start;
  bool ok = true;
  for (int gr = 0; gr < 2; ++gr) {
    for (int c = 0; c < nch; ++c) {
      Granule g;
      int scfsi, mdb;
      parse_side(side, nch, gr, c, ri, &g, &scfsi, &mdb);
      if (c == ch && ok)
        ok = decode_granule(main, main_bytes, bit, g, scfsi, gr, ri, &recs[c], lut, &recs[gr * nch + c]);
      bit += g.part2_3;
    }
  }
  return ok;
}

}  // namespace mp3
}  // namespace bt
