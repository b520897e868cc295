// FLAC (RFC 9639) frame parsing and decoding, shared by the host staging of bt_stage_flac_files, the decode kernels of
// bt_flac_decode and the host test hook bt_debug_flac_decode_host: one __host__ __device__ implementation, so the CPU tests
// hold the device's arithmetic to the test encoder.
//
// Conventions a misreading would hide (RFC 9639 sections in parentheses):
//  - residuals are zigzag folded: u even -> u / 2, u odd -> -(u + 1) / 2 (9.2.7.1);
//  - side = left - right; left/side rebuilds right = left - side, side/right left = side + right (9.1.3 / 4.2);
//  - mid/side: mid = (mid << 1) | (side & 1), left = (mid + side) >> 1, right = (mid - side) >> 1;
//  - LPC: s[i] = e[i] + ((sum_j c[j] * s[i - 1 - j]) >> shift), c[0] on the newest sample; a negative shift is refused;
//  - the first residual partition holds (block size >> partition order) - predictor order residuals (9.2.7).
#pragma once
#include <cstdint>

#include "../../include/beatthis.h"

#if defined(__CUDACC__)
#define BT_HD __host__ __device__ __forceinline__
#else
#define BT_HD inline
#endif

namespace bt {
namespace flac {

// Frame-header CRC-8 (polynomial x^8 + x^2 + x + 1, init 0) and frame CRC-16 (x^16 + x^15 + x^2 + 1, init 0), bitwise.
BT_HD uint8_t crc8_byte(uint8_t crc, uint8_t b) {
  crc ^= b;
  for (int k = 0; k < 8; ++k) crc = static_cast<uint8_t>((crc & 0x80) ? (crc << 1) ^ 0x07 : crc << 1);
  return crc;
}
BT_HD uint16_t crc16_byte_slow(uint16_t crc, uint8_t b) {
  crc ^= static_cast<uint16_t>(b) << 8;
  for (int k = 0; k < 8; ++k) crc = static_cast<uint16_t>((crc & 0x8000) ? (crc << 1) ^ 0x8005 : crc << 1);
  return crc;
}
// table[b] = crc16_byte_slow(0, b): crc' = (crc << 8) ^ table[(crc >> 8) ^ b]
BT_HD uint16_t crc16_byte(const uint16_t* table, uint16_t crc, uint8_t b) {
  return static_cast<uint16_t>((crc << 8) ^ table[((crc >> 8) ^ b) & 0xFF]);
}

BT_HD int clz8(uint32_t b) {  // leading zeros of a non-zero byte
  int n = 0;
  while (!(b & 0x80)) { b <<= 1; ++n; }
  return n;
}

// MSB-first bit reader over bytes [0, nbytes) of p.  A read past the end sets `bad` and returns 0: every read of a
// frame is bounded by the frame's own span.
struct Bits {
  const uint8_t* p;
  int64_t nbits;
  int64_t pos;
  bool bad;

  BT_HD uint64_t read(int n) {  // n <= 64
    if (n == 0) return 0;
    if (pos + n > nbits) { bad = true; pos = nbits; return 0; }
    uint64_t v = 0;
    while (n > 0) {
      const int off = static_cast<int>(pos & 7);
      const int take = n < 8 - off ? n : 8 - off;
      const uint32_t b = p[pos >> 3];
      v = (v << take) | ((b >> (8 - off - take)) & ((1u << take) - 1));
      pos += take;
      n -= take;
    }
    return v;
  }
  BT_HD int64_t read_signed(int n) {  // two's complement, n <= 33 (a side channel of 32-bit audio)
    if (n == 0) return 0;
    const uint64_t v = read(n);
    return static_cast<int64_t>(v << (64 - n)) >> (64 - n);
  }
  // zeros before the next 1 bit (consumed), at most `limit` of them; more sets `bad`
  BT_HD uint64_t unary(uint64_t limit) {
    uint64_t q = 0;
    for (;;) {
      if (pos >= nbits) { bad = true; return 0; }
      const int off = static_cast<int>(pos & 7);
      const uint32_t b = (static_cast<uint32_t>(p[pos >> 3]) << off) & 0xFF;
      if (b == 0) {
        q += 8 - off;
        pos += 8 - off;
      } else {
        const int z = clz8(b);
        q += z;
        pos += z + 1;
        if (q > limit) { bad = true; return 0; }
        return q;
      }
      if (q > limit) { bad = true; return 0; }
    }
  }
};

// What a frame header says (9.1).  number: the frame number (fixed block size) or first sample (variable).
struct Header {
  int block_size;
  int sample_rate;  // 0: from STREAMINFO
  int assignment;   // 0..7 independent (channels - 1), 8 left/side, 9 side/right, 10 mid/side
  int channels;
  int bits;         // 0: from STREAMINFO
  int variable;     // blocking strategy bit
  int64_t number;
  int length;       // header bytes, CRC-8 included
};

// The sample rates of header codes 0..11 (0: from STREAMINFO)
BT_HD int coded_rate(int code) {
  switch (code) {
    case 1: return 88200;
    case 2: return 176400;
    case 3: return 192000;
    case 4: return 8000;
    case 5: return 16000;
    case 6: return 22050;
    case 7: return 24000;
    case 8: return 32000;
    case 9: return 44100;
    case 10: return 48000;
    case 11: return 96000;
    default: return 0;
  }
}

// Parses and checks the frame header at p[0 .. avail): sync code, reserved bits and values, the coded number (up to the
// 7-byte form) and CRC-8.  False when any of them fails.
BT_HD bool parse_header(const uint8_t* p, int64_t avail, Header* h) {
  if (avail < 6 || p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return false;
  h->variable = p[1] & 1;
  const int bs_code = p[2] >> 4, sr_code = p[2] & 15;
  const int ch_code = p[3] >> 4, sz_code = (p[3] >> 1) & 7;
  if (bs_code == 0 || sr_code == 15 || ch_code > 10 || sz_code == 3 || (p[3] & 1)) return false;
  // coded number: UTF-8 style, 1..7 bytes
  int64_t pos = 4;
  const uint32_t b0 = p[pos++];
  int extra;
  uint64_t v;
  if (b0 < 0x80) { extra = 0; v = b0; }
  else if ((b0 & 0xE0) == 0xC0) { extra = 1; v = b0 & 0x1F; }
  else if ((b0 & 0xF0) == 0xE0) { extra = 2; v = b0 & 0x0F; }
  else if ((b0 & 0xF8) == 0xF0) { extra = 3; v = b0 & 0x07; }
  else if ((b0 & 0xFC) == 0xF8) { extra = 4; v = b0 & 0x03; }
  else if ((b0 & 0xFE) == 0xFC) { extra = 5; v = b0 & 0x01; }
  else if (b0 == 0xFE) { extra = 6; v = 0; }
  else return false;
  if (pos + extra > avail) return false;
  for (int k = 0; k < extra; ++k) {
    const uint32_t b = p[pos++];
    if ((b & 0xC0) != 0x80) return false;
    v = (v << 6) | (b & 0x3F);
  }
  if (!h->variable && extra > 5) return false;  // frame numbers have 31 bits at most
  h->number = static_cast<int64_t>(v);
  int bs;
  if (bs_code == 1) bs = 192;
  else if (bs_code <= 5) bs = 576 << (bs_code - 2);
  else if (bs_code == 6) { if (pos + 1 > avail) return false; bs = p[pos] + 1; pos += 1; }
  else if (bs_code == 7) { if (pos + 2 > avail) return false; bs = ((p[pos] << 8) | p[pos + 1]) + 1; pos += 2; }
  else bs = 256 << (bs_code - 8);
  int sr;
  if (sr_code < 12) sr = coded_rate(sr_code);
  else if (sr_code == 12) { if (pos + 1 > avail) return false; sr = p[pos] * 1000; pos += 1; }
  else {
    if (pos + 2 > avail) return false;
    sr = (p[pos] << 8) | p[pos + 1];
    if (sr_code == 14) sr *= 10;
    pos += 2;
  }
  if (pos + 1 > avail) return false;
  uint8_t crc = 0;
  for (int64_t k = 0; k < pos; ++k) crc = crc8_byte(crc, p[k]);
  if (crc != p[pos]) return false;
  h->block_size = bs;
  h->sample_rate = sr;
  h->assignment = ch_code;
  h->channels = ch_code < 8 ? ch_code + 1 : 2;
  h->bits = sz_code == 0 ? 0 : sz_code == 1 ? 8 : sz_code == 2 ? 12 : sz_code == 7 ? 32 : 8 + 4 * (sz_code - 2);
  h->length = static_cast<int>(pos + 1);
  return true;
}

// Reads a residual of bs - order values (9.2.7) and rebuilds the samples out[order .. bs) with `predict(i)` (the
// prediction of sample i from out[i - order .. i)), wrapping in 64 bits.  False on a reserved coding method, a partition
// order the block size does not divide into at least `order` samples, or a read past the frame.
template <class Predict>
BT_HD bool residual(Bits& br, int bs, int order, int64_t* out, Predict predict) {
  const int method = static_cast<int>(br.read(2));
  if (method > 1) return false;
  const int pbits = method ? 5 : 4, escape = (1 << pbits) - 1;
  const int porder = static_cast<int>(br.read(4));
  if (br.bad || (bs & ((1 << porder) - 1)) != 0) return false;
  const int psize = bs >> porder;
  if (psize < order) return false;
  int i = order;
  for (int part = 0; part < (1 << porder); ++part) {
    const int end = i + psize - (part == 0 ? order : 0);
    const int k = static_cast<int>(br.read(pbits));
    if (br.bad) return false;
    if (k == escape) {
      const int w = static_cast<int>(br.read(5));
      for (; i < end; ++i) {
        const int64_t e = br.read_signed(w);
        out[i] = static_cast<int64_t>(static_cast<uint64_t>(e) + static_cast<uint64_t>(predict(i)));
      }
    } else {
      for (; i < end; ++i) {
        const uint64_t q = br.unary(0xFFFFFFFFull);
        const uint64_t u = (q << k) | br.read(k);
        const int64_t e = static_cast<int64_t>(u >> 1) ^ -static_cast<int64_t>(u & 1);
        out[i] = static_cast<int64_t>(static_cast<uint64_t>(e) + static_cast<uint64_t>(predict(i)));
      }
    }
    if (br.bad) return false;
  }
  return true;
}

// One subframe (9.2) of bs samples of `ss` bits into out[0 .. bs).  coef: 32 int32 slots at stride cs (LPC
// coefficients).  False when the subframe is malformed.
BT_HD bool subframe(Bits& br, int bs, int ss, int64_t* out, int32_t* coef, int cs) {
  const int hdr = static_cast<int>(br.read(8));
  if (br.bad || (hdr & 0x80)) return false;
  const int type = (hdr >> 1) & 63;
  int wasted = 0;
  if (hdr & 1) wasted = 1 + static_cast<int>(br.unary(31));
  ss -= wasted;
  if (br.bad || ss < 1) return false;
  if (type == 0) {  // CONSTANT
    const int64_t v = br.read_signed(ss);
    for (int i = 0; i < bs; ++i) out[i] = v;
  } else if (type == 1) {  // VERBATIM
    for (int i = 0; i < bs; ++i) out[i] = br.read_signed(ss);
  } else if (type >= 8 && type <= 12) {  // FIXED, order 0..4
    const int order = type - 8;
    if (order > bs) return false;
    for (int i = 0; i < order; ++i) out[i] = br.read_signed(ss);
    if (br.bad) return false;
    bool ok;
    switch (order) {
      case 0: ok = residual(br, bs, 0, out, [](int) { return int64_t{0}; }); break;
      case 1: ok = residual(br, bs, 1, out, [&](int i) { return out[i - 1]; }); break;
      case 2: ok = residual(br, bs, 2, out, [&](int i) { return 2 * out[i - 1] - out[i - 2]; }); break;
      case 3:
        ok = residual(br, bs, 3, out, [&](int i) { return 3 * out[i - 1] - 3 * out[i - 2] + out[i - 3]; });
        break;
      default:
        ok = residual(br, bs, 4, out,
                      [&](int i) { return 4 * out[i - 1] - 6 * out[i - 2] + 4 * out[i - 3] - out[i - 4]; });
        break;
    }
    if (!ok) return false;
  } else if (type >= 32) {  // LPC, order 1..32
    const int order = type - 31;
    if (order > bs) return false;
    for (int i = 0; i < order; ++i) out[i] = br.read_signed(ss);
    const int precision = static_cast<int>(br.read(4)) + 1;
    const int shift = static_cast<int>(br.read_signed(5));
    if (br.bad || precision == 16 || shift < 0) return false;
    for (int j = 0; j < order; ++j) coef[j * cs] = static_cast<int32_t>(br.read_signed(precision));
    if (br.bad) return false;
    const bool ok = residual(br, bs, order, out, [&](int i) {
      uint64_t acc = 0;
      for (int j = 0; j < order; ++j)
        acc += static_cast<uint64_t>(static_cast<int64_t>(coef[j * cs]) * out[i - 1 - j]);
      return static_cast<int64_t>(acc) >> shift;
    });
    if (!ok) return false;
  } else {
    return false;  // reserved subframe type
  }
  if (br.bad) return false;
  if (wasted)
    for (int i = 0; i < bs; ++i) out[i] = static_cast<int64_t>(static_cast<uint64_t>(out[i]) << wasted);
  return true;
}

// Decodes one frame of `len` bytes at f: checks CRC-16 (crc16: the byte table), that its header gives `bs` samples,
// `channels` channels and `bits` bits (0 in the header: from STREAMINFO), decodes every subframe and undoes the channel
// decorrelation.  Channel c's sample t goes to out[c * stride + t].  False when the frame is malformed.
BT_HD bool decode_frame(const uint8_t* f, int64_t len, int bs, int channels, int bits, const uint16_t* crc16,
                        int64_t* out, int64_t stride, int32_t* coef, int cs) {
  if (len < 8) return false;
  uint16_t crc = 0;
  for (int64_t k = 0; k < len - 2; ++k) crc = crc16_byte(crc16, crc, f[k]);
  if (crc != ((f[len - 2] << 8) | f[len - 1])) return false;
  Header h;
  if (!parse_header(f, len - 2, &h) || h.block_size != bs || h.channels != channels || (h.bits && h.bits != bits))
    return false;
  Bits br{f, (len - 2) * 8, static_cast<int64_t>(h.length) * 8, false};
  for (int c = 0; c < channels; ++c) {
    const bool side = (h.assignment == 8 || h.assignment == 10) ? c == 1 : h.assignment == 9 ? c == 0 : false;
    if (!subframe(br, bs, bits + (side ? 1 : 0), out + c * stride, coef, cs)) return false;
  }
  // the bits up to the CRC are zero padding to the byte boundary
  if (br.bad || (br.nbits - br.pos) >= 8) return false;
  int64_t* a = out;
  int64_t* b = out + stride;
  if (h.assignment == 8) {
    for (int i = 0; i < bs; ++i) b[i] = a[i] - b[i];
  } else if (h.assignment == 9) {
    for (int i = 0; i < bs; ++i) a[i] += b[i];
  } else if (h.assignment == 10) {
    for (int i = 0; i < bs; ++i) {
      const int64_t mid = static_cast<int64_t>(static_cast<uint64_t>(a[i]) << 1) | (b[i] & 1), side = b[i];
      a[i] = (mid + side) >> 1;
      b[i] = (mid - side) >> 1;
    }
  }
  return true;
}

// Sample t of a decoded stream as the outputs hold it.  Mono: value * 2^-(bits-1) in float64, summed over channels in
// channel order, one division by the channel count, one fp32 rounding (host_stage.cpp's mix_pcm_t); one channel is a
// single multiply and rounding.  Channels: each value * 2^-(bits-1) in float64.
BT_HD double scale_of(int bits) { return 1.0 / static_cast<double>(int64_t{1} << (bits - 1)); }
BT_HD float mono_sample(const int64_t* x, int64_t stride, int channels, double scale) {
  if (channels == 1) return static_cast<float>(static_cast<double>(x[0]) * scale);
  double acc = static_cast<double>(x[0]) * scale;
  for (int c = 1; c < channels; ++c) acc += static_cast<double>(x[c * stride]) * scale;
  return static_cast<float>(acc / static_cast<double>(channels));
}

}  // namespace flac
}  // namespace bt
