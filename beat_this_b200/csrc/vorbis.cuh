// Vorbis I audio decoding (the Xiph.Org Vorbis I specification), shared by the device kernels (kernels_vorbis.cu), the
// host staging and the host test hook (api_vorbis.cu).  Every step is a __host__ __device__ function of one "lane" (a
// thread on the device, a loop index on the host), so the host hook runs the kernels' own arithmetic.
//
// A staged file is its audio packets back to back, a packet table (bt_vorbis_packet, include/beatthis.h) and its decode
// tables: the setup header turned into fixed-size records (Tables, Codebook, Floor1, Residue, Mapping, Mode) followed by
// every codebook's decode tree and expanded VQ vectors, all 32-bit words.  The host reads each packet's type, mode and
// window flags to fill the table, so the device needs no state carried from one packet to the next.
//
// Scratch of one packet of block size n and one channel (bt_vorbis_decode keeps it in the ctx):
//   n floats        its spectrum (the first n / 2), then its windowed IMDCT output (all n)
//   n / 2 bytes     residue classifications
//   kFloorWords     floor1 posts: the "nonzero" flag and the decoded Y values
// 4.5 n + 264 bytes per packet and channel, about 9.3 bytes per output sample and channel at blocks 256 / 2048.
#pragma once

#include <cmath>
#include <cstdint>

#include "../../include/beatthis.h"
#include "fft.cuh"

#if defined(__CUDACC__)
#define BT_VB_HD __host__ __device__ __forceinline__
#else
#define BT_VB_HD inline
#endif

namespace bt {
namespace vorbis {

constexpr int kMaxChannels = 8;
constexpr int kMaxPosts = 65;        // floor1 X values (libvorbis's limit as well)
constexpr int kFloorWords = 66;      // per packet and channel: nonzero flag, Y[65]
constexpr int kMinLog2 = 6, kMaxLog2 = 13;  // block sizes 64 .. 8192
constexpr uint32_t kLeaf = 0x80000000u;     // a tree child that is an entry (low bits), not a node
constexpr int64_t kMaxTableWords = int64_t(1) << 24;  // decode tables of one file: 64 MB at most

// ---- the decode tables of one file ------------------------------------------------------------------------------------
struct Tables {
  int32_t channels, blocksize[2];
  int32_t n_codebooks, n_floors, n_residues, n_mappings, n_modes, mode_bits;
  int32_t codebooks, floors, residues, mappings, modes;  // word offsets of the record arrays
  int32_t words;                                          // the tables' size in words
};

struct Codebook {
  int32_t dimensions, entries, lookup;  // lookup: 0 scalar only, 1 or 2 VQ
  int32_t tree;                         // word offset of the tree: node k is words [tree + 2k, tree + 2k + 2)
  int32_t vq;                           // word offset of entries x dimensions floats (lookup 1, 2)
  int32_t used;                         // used entries (0: the book decodes nothing)
};

struct Floor1 {
  int32_t partitions, multiplier, values, classes;
  int32_t partition_class[31];
  int32_t class_dim[16], class_sub[16], class_master[16], sub_book[16][8];  // book -1: none
  int32_t x[kMaxPosts], sorted[kMaxPosts], low[kMaxPosts], high[kMaxPosts];
};

struct Residue {
  int32_t type, begin, end, partition_size, classifications, classbook;
  int32_t books[64][8];  // -1: no book in that pass
};

struct Mapping {
  int32_t submaps, coupling_steps;
  int32_t mux[kMaxChannels], submap_floor[16], submap_residue[16];
  int32_t magnitude[256], angle[256];
};

struct Mode {
  int32_t blockflag, mapping;
};

template <class T>
BT_VB_HD const T* rec(const uint32_t* t, int32_t at, int i) {
  return reinterpret_cast<const T*>(t + at) + i;
}

BT_VB_HD int ilog(uint32_t v) {
  int r = 0;
  while (v) {
    ++r;
    v >>= 1;
  }
  return r;
}

// ---- bits: LSB first within each byte, little-endian fields ----------------------------------------------------------
struct Bits {
  const uint8_t* p;
  int64_t n_bits, pos;
  bool eop;
  BT_VB_HD uint32_t read(int n) {  // n <= 32; past the end of the packet: eop, and the value is 0
    if (pos + n > n_bits) {
      eop = true;
      pos = n_bits;
      return 0;
    }
    uint32_t v = 0;
    for (int i = 0; i < n;) {
      const int64_t at = pos + i;
      const int b = static_cast<int>(at & 7), take = (8 - b) < (n - i) ? (8 - b) : (n - i);
      v |= ((static_cast<uint32_t>(p[at >> 3]) >> b) & ((1u << take) - 1)) << i;
      i += take;
    }
    pos += n;
    return v;
  }
};

// One codeword of book `cb`: its entry, -1 at the end of the packet, -2 for a codeword the book does not have.
BT_VB_HD int32_t decode_entry(const uint32_t* t, const Codebook& cb, Bits& b) {
  if (cb.used == 0) return -2;
  uint32_t node = 0;
  for (int depth = 0; depth < 33; ++depth) {
    if (b.pos >= b.n_bits) {
      b.eop = true;
      return -1;
    }
    const uint32_t bit = (b.p[b.pos >> 3] >> (b.pos & 7)) & 1;
    ++b.pos;
    const uint32_t c = t[cb.tree + 2 * node + bit];
    if (c & kLeaf) return static_cast<int32_t>(c & ~kLeaf);
    if (c == 0) return -2;
    node = c;
  }
  return -2;
}

// ---- floor1 packet decode: lane = packet; writes out[0] (nonzero) and out[1 + i] (Y[i]).  Returns 1, 0 at the end of
// the packet (which makes every floor of the packet unused) or -2 for a codeword a book does not have. ----------------
BT_VB_HD int floor1_decode(const uint32_t* t, const Tables& T, const Floor1& f, Bits& b, int32_t* out) {
  out[0] = static_cast<int32_t>(b.read(1));
  if (b.eop) return 0;
  if (!out[0]) return 1;
  const int range = f.multiplier == 1 ? 256 : f.multiplier == 2 ? 128 : f.multiplier == 3 ? 86 : 64;
  const int rb = ilog(range - 1);
  out[1] = static_cast<int32_t>(b.read(rb));
  out[2] = static_cast<int32_t>(b.read(rb));
  int off = 2;
  for (int i = 0; i < f.partitions; ++i) {
    const int cls = f.partition_class[i];
    const int cdim = f.class_dim[cls], cbits = f.class_sub[cls], csub = (1 << cbits) - 1;
    int32_t cval = 0;
    if (cbits > 0) {
      cval = decode_entry(t, *rec<Codebook>(t, T.codebooks, f.class_master[cls]), b);
      if (cval < 0) return cval == -1 ? 0 : -2;
    }
    for (int j = 0; j < cdim; ++j) {
      const int book = f.sub_book[cls][cval & csub];
      cval >>= cbits;
      int32_t y = 0;
      if (book >= 0) {
        y = decode_entry(t, *rec<Codebook>(t, T.codebooks, book), b);
        if (y < 0) return y == -1 ? 0 : -2;
      }
      out[1 + off++] = y;
    }
  }
  return b.eop ? 0 : 1;
}

// value k of residue vector v += x: type 2 (interleaved) spreads one vector over the submap's channels
BT_VB_HD void add_value(float* spec, int stride, uint32_t chans, int nch, bool interleaved, int v, int k, float x) {
  const int j = interleaved ? k % nch : v;
  spec[((chans >> (4 * j)) & 15) * stride + (interleaved ? k / nch : k)] += x;
}

// ---- residue packet decode --------------------------------------------------------------------------------------------
// The vectors of one submap: its nch channels, channel j of the submap being (chans >> 4j) & 15, each a vector of n2
// values at spec + channel * stride (type 2: one interleaved vector of nch x n2 values); `skip` a bit mask of the
// submap's channels not to decode.  cls: n2 x nch bytes of scratch.
// Returns 0, or -2 for a codeword a book does not have (an end of packet just ends the decode).
BT_VB_HD int residue_decode(const uint32_t* t, const Tables& T, const Residue& r, Bits& b, float* spec, int stride,
                            uint32_t chans, int nch, uint32_t skip, int n2, uint8_t* cls) {
  const bool interleaved = r.type == 2;
  const int nv = interleaved ? 1 : nch;
  const int size = interleaved ? n2 * nch : n2;  // at most 8 x 4096: the indices below are 32-bit
  if (interleaved) skip = (skip == (1u << nch) - 1) ? 1u : 0u;
  const int lb = r.begin < size ? r.begin : size, le = r.end < size ? r.end : size;
  const int psize = r.partition_size, parts = (le - lb) / psize;
  if (le - lb <= 0 || parts == 0) return 0;
  const Codebook& ccb = *rec<Codebook>(t, T.codebooks, r.classbook);
  const int cpw = ccb.dimensions;
  for (int pass = 0; pass < 8; ++pass) {
    int pc = 0;
    while (pc < parts) {
      if (pass == 0) {
        for (int v = 0; v < nv; ++v) {
          if (skip >> v & 1) continue;
          int32_t temp = decode_entry(t, ccb, b);
          if (temp < 0) return temp == -1 ? 0 : -2;
          for (int i = cpw - 1; i >= 0; --i) {
            if (pc + i < parts) cls[v * n2 + pc + i] = static_cast<uint8_t>(temp % r.classifications);
            temp /= r.classifications;
          }
        }
      }
      for (int i = 0; i < cpw && pc < parts; ++i, ++pc) {
        for (int v = 0; v < nv; ++v) {
          if (skip >> v & 1) continue;
          const int book = r.books[cls[v * n2 + pc]][pass];
          if (book < 0) continue;
          const Codebook& cb = *rec<Codebook>(t, T.codebooks, book);
          const float* vq = reinterpret_cast<const float*>(t + cb.vq);
          const int d = cb.dimensions;
          const int off = lb + pc * psize;
          if (r.type == 0) {
            const int step = psize / d;
            for (int j = 0; j < step; ++j) {
              const int32_t e = decode_entry(t, cb, b);
              if (e < 0) return e == -1 ? 0 : -2;
              for (int k = 0; k < d; ++k) add_value(spec, stride, chans, nch, interleaved, v, off + j + k * step, vq[static_cast<int64_t>(e) * d + k]);
            }
          } else {
            for (int j = 0; j < psize;) {
              const int32_t e = decode_entry(t, cb, b);
              if (e < 0) return e == -1 ? 0 : -2;
              for (int k = 0; k < d; ++k, ++j) add_value(spec, stride, chans, nch, interleaved, v, off + j, vq[static_cast<int64_t>(e) * d + k]);
            }
          }
        }
      }
    }
  }
  return 0;
}

// ---- floor1 curve -----------------------------------------------------------------------------------------------------
BT_VB_HD int render_point(int x0, int y0, int x1, int y1, int x) {
  const int dy = y1 - y0, adx = x1 - x0, ady = dy < 0 ? -dy : dy;
  const int off = ady * (x - x0) / adx;
  return dy < 0 ? y0 - off : y0 + off;
}

// Step 2 of floor1 (amplitude value synthesis) of one channel: final Y and "used" flags of every post, from the
// decoded Y values y[0 .. values).  One lane per channel.
BT_VB_HD void floor1_step2(const Floor1& f, const int32_t* y, int32_t* fy, int32_t* used) {
  const int range = f.multiplier == 1 ? 256 : f.multiplier == 2 ? 128 : f.multiplier == 3 ? 86 : 64;
  fy[0] = y[0];
  fy[1] = y[1];
  used[0] = used[1] = 1;
  for (int i = 2; i < f.values; ++i) {
    const int lo = f.low[i], hi = f.high[i];
    const int pred = render_point(f.x[lo], fy[lo], f.x[hi], fy[hi], f.x[i]);
    const int val = y[i], highroom = range - pred, lowroom = pred;
    const int room = (highroom < lowroom ? highroom : lowroom) * 2;
    if (val != 0) {
      used[lo] = used[hi] = used[i] = 1;
      if (val >= room)
        fy[i] = highroom > lowroom ? val - lowroom + pred : pred - val + highroom - 1;
      else
        fy[i] = (val & 1) ? pred - (val + 1) / 2 : pred + val / 2;
    } else {
      used[i] = 0;
      fy[i] = pred;
    }
  }
}

// The line of render_line from (x0, y0) to (x1, y1) at x0 <= x < x1, in closed form: after k steps the error term has
// wrapped floor(k * ady / adx) times.
BT_VB_HD int render_at(int x0, int y0, int x1, int y1, int x) {
  const int dy = y1 - y0, adx = x1 - x0;
  const int base = dy / adx, ady = (dy < 0 ? -dy : dy) - (base < 0 ? -base : base) * adx;
  const int k = x - x0;
  const int extra = static_cast<int>(static_cast<int64_t>(k) * ady / adx);
  return y0 + k * base + (dy < 0 ? -extra : extra);
}

// The floor value at x from the used posts in X order: px[0 .. np), py (already multiplied), dB: the inverse dB table.
BT_VB_HD float floor_at(const int32_t* px, const int32_t* py, int np, int x, const float* dB) {
  int lo = 0, hi = np - 1;  // the last post with px <= x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (px[mid] <= x) lo = mid;
    else hi = mid - 1;
  }
  const int y = lo + 1 < np ? render_at(px[lo], py[lo], px[lo + 1], py[lo + 1], x) : py[lo];
  return dB[y < 0 ? 0 : y > 255 ? 255 : y];
}

// Inverse square-polar coupling of one value pair (magnitude m, angle a).
BT_VB_HD void uncouple(float& m, float& a) {
  const float M = m, A = a;
  if (M > 0) {
    if (A > 0) { m = M; a = M - A; }
    else { a = M; m = M + A; }
  } else {
    if (A > 0) { m = M; a = M + A; }
    else { a = M; m = M - A; }
  }
}

// ---- the IMDCT: y[n] = sum_k X[k] cos(2 pi / N (n + 1/2 + N/4)(k + 1/2)), n < N, through an N/4-point complex FFT ---
// With M = N/2 and H = N/4: v[k] = (X[2k] + i X[M-1-2k]) e^{-i pi (k + 1/4) / M}, V = FFT_H(v), W[k] = V[k] e^{-i pi k/M};
// the DCT-IV u of X is u[2k] = Re W[k], u[M-1-2k] = -Im W[k], and y unfolds it: y[n] = u[n + M/2] (n + M/2 < M),
// -u[3M/2 - 1 - n] (< 2M), -u[n - 3M/2].
// Signal tables of block size n = 2^b, at float2 signal_at(b): pre twiddles e^{-i pi (k + 1/4) / M} (H), post
// twiddles e^{-i pi k / M} (H), FFT twiddles e^{-2 pi i m / H} (H / 2), then the rising window slope of length n / 2
// (n / 4 float2): 7 n / 8 float2.  The 256 floats of the floor1 inverse dB table follow the last block size's.
BT_VB_HD int64_t signal_at(int b) { return 7 * ((int64_t(1) << (b - 3)) - 8); }
constexpr int64_t kDbAt = 7 * ((int64_t(1) << (kMaxLog2 + 1 - 3)) - 8);  // float2 offset of the dB table
constexpr int64_t kSignalFloats = 2 * kDbAt + 256;

// butterfly j of the radix-R Stockham pass after Ns points of an H-point FFT, `in` to `out`; tw: e^{-2 pi i m / H}
template <int R>
BT_VB_HD void stockham(const float2* in, float2* out, int j, int Ns, int H, const float2* tw) {
  float2 v[8];
  const int k = j & (Ns - 1), step = H / (Ns * R);
#pragma unroll
  for (int r = 0; r < R; ++r) {
    v[r] = in[j + r * (H / R)];
    if (r) {
      const int m = k * r * step;
      const float2 w = tw[m & (H / 2 - 1)];
      v[r] = cmul(v[r], (m & (H / 2)) ? make_float2(-w.x, -w.y) : w);
    }
  }
  if constexpr (R == 8) {
    dft8(v);
  } else if constexpr (R == 4) {
    dft4(v[0], v[1], v[2], v[3]);
  } else {
    const float2 t = v[0];
    v[0] = cadd(t, v[1]);
    v[1] = csub(t, v[1]);
  }
  const int d = (j - k) * R + k;
#pragma unroll
  for (int r = 0; r < R; ++r) out[d + r * Ns] = v[r];
}

// radix of pass q of an H-point FFT (8 while 8 divides what is left, then 4 or 2) and the points before it
BT_VB_HD int pass_radix(int H, int Ns) {
  const int left = H / Ns;
  return left % 8 == 0 ? 8 : left;
}

// u[2k] and u[M-1-2k] from V[k]
BT_VB_HD void post_twiddle(const float2* V, const float2* s, int n, int k, float* u) {
  const int M = n / 2;
  const float2 w = cmul(V[k], s[n / 4 + k]);
  u[2 * k] = w.x;
  u[M - 1 - 2 * k] = -w.y;
}

// The windowed IMDCT value n of a block: u its DCT-IV, the window from the block flags (spec 4.3.1).
BT_VB_HD float windowed(const float* u, int n, int i, int long_block, int prev, int next, int b0,
                        const float* slope_short, const float* slope_long) {
  const int M = n / 2;
  const int m = i + M / 2;
  const float y = m < M ? u[m] : m < 2 * M ? -u[2 * M - 1 - m] : -u[m - 2 * M];
  const bool left_short = long_block && !prev, right_short = long_block && !next;
  float w;
  if (i < M) {
    const int ls = left_short ? n / 4 - b0 / 4 : 0, le = left_short ? n / 4 + b0 / 4 : M;
    const float* sl = left_short ? slope_short : slope_long;
    w = i < ls ? 0.f : i >= le ? 1.f : sl[i - ls];
  } else {
    const int rs = right_short ? 3 * n / 4 - b0 / 4 : M, re = right_short ? 3 * n / 4 + b0 / 4 : n;
    const float* sl = right_short ? slope_short : slope_long;
    const int len = re - rs;
    w = i < rs ? 1.f : i >= re ? 0.f : sl[len - 1 - (i - rs)];
  }
  return y * w;
}


// ---- one stream of a decode call --------------------------------------------------------------------------------------
struct StreamDev {
  const uint8_t* bytes;             // its packet bytes
  const uint32_t* tables;           // its decode tables
  const bt_vorbis_packet* packets;  // its packet table
  float* spec;                      // scratch: channels x block_samples floats ...
  int32_t* floors;                  // ... channels x n_packets x kFloorWords words ...
  uint8_t* cls;                     // ... channels x block_samples / 2 bytes
  int64_t byte_count, table_words, n_packets, block_samples, skip, n_samples, out_off;
  int32_t channels;
};

BT_VB_HD int block_size(const StreamDev& s, const bt_vorbis_packet& e) {
  return reinterpret_cast<const Tables*>(s.tables)->blocksize[e.blockflag ? 1 : 0];
}

// The packet-decode lane of packet p: its entry checked against its stream and the one before, then floors, nonzero
// propagation and residues into the packet's scratch.  BT_OK or BT_ERR_IO.
BT_VB_HD int decode_packet(const StreamDev& s, int64_t p) {
  const uint32_t* t = s.tables;
  const Tables& T = *reinterpret_cast<const Tables*>(t);
  if (s.table_words < static_cast<int64_t>(sizeof(Tables) / 4) || T.words > s.table_words) return BT_ERR_IO;
  const bt_vorbis_packet& e = s.packets[p];
  const int nch = s.channels;
  if (e.mode >= T.n_modes || nch != T.channels) return BT_ERR_IO;
  const Mode& mo = *rec<Mode>(t, T.modes, e.mode);
  const int n = T.blocksize[mo.blockflag];
  if (e.blockflag != mo.blockflag || e.bytes < 0 || e.byte_offset < 0 || e.byte_offset + e.bytes > s.byte_count ||
      e.block_offset < 0 || e.block_offset + n > s.block_samples)
    return BT_ERR_IO;
  if (p == 0 ? (e.block_offset != 0 || e.end_sample != 0)
             : (e.block_offset != s.packets[p - 1].block_offset + block_size(s, s.packets[p - 1]) ||
                e.end_sample != s.packets[p - 1].end_sample + block_size(s, s.packets[p - 1]) / 4 + n / 4))
    return BT_ERR_IO;
  float* spec = s.spec + e.block_offset * nch;
  int32_t* fl = s.floors + p * nch * kFloorWords;
  for (int c = 0; c < nch; ++c)
    for (int i = 0; i < n / 2; ++i) spec[c * n + i] = 0.f;
  Bits b{s.bytes + e.byte_offset, 8 * static_cast<int64_t>(e.bytes), 0, false};
  b.read(1 + T.mode_bits + (mo.blockflag ? 2 : 0));
  const Mapping& m = *rec<Mapping>(t, T.mappings, mo.mapping);
  uint32_t nonzero = 0;
  for (int c = 0; c < nch; ++c) {
    const Floor1& f = *rec<Floor1>(t, T.floors, m.submap_floor[m.mux[c]]);
    const int r = floor1_decode(t, T, f, b, fl + c * kFloorWords);
    if (r < 0) return BT_ERR_IO;
    if (r == 0) {  // the packet ends in the floors: every channel's output is zero
      for (int k = 0; k < nch; ++k) fl[k * kFloorWords] = 0;
      return BT_OK;
    }
    if (fl[c * kFloorWords]) nonzero |= 1u << c;
  }
  for (int i = 0; i < m.coupling_steps; ++i)
    if ((nonzero >> m.magnitude[i] | nonzero >> m.angle[i]) & 1) nonzero |= (1u << m.magnitude[i]) | (1u << m.angle[i]);
  for (int sm = 0; sm < m.submaps; ++sm) {
    uint32_t chans = 0, skip = 0;
    int k = 0;
    for (int c = 0; c < nch; ++c)
      if (m.mux[c] == sm) {
        chans |= static_cast<uint32_t>(c) << (4 * k);
        if (!(nonzero >> c & 1)) skip |= 1u << k;
        ++k;
      }
    if (k == 0) continue;
    const Residue& r = *rec<Residue>(t, T.residues, m.submap_residue[sm]);
    if (residue_decode(t, T, r, b, spec, n, chans, k, skip, n / 2, s.cls + e.block_offset * nch / 2) < 0)
      return BT_ERR_IO;
  }
  return BT_OK;
}

// ---- the block lanes --------------------------------------------------------------------------------------------------
struct BlockGeom {
  int n, prev, next, blockflag, mapping;
};

BT_VB_HD BlockGeom block_geom(const StreamDev& s, int64_t p) {
  const Tables& T = *reinterpret_cast<const Tables*>(s.tables);
  const bt_vorbis_packet& e = s.packets[p];
  const Mode& mo = *rec<Mode>(s.tables, T.modes, e.mode);
  return BlockGeom{T.blocksize[mo.blockflag], e.prev_long, e.next_long, mo.blockflag, mo.mapping};
}

// floor curves of a packet's channels: the used posts in X order, Y multiplied
struct BlockShared {
  int32_t fy[kMaxChannels][kMaxPosts], used[kMaxChannels][kMaxPosts];
  int32_t px[kMaxChannels][kMaxPosts], py[kMaxChannels][kMaxPosts];
  int32_t np[kMaxChannels];  // 0: the floor is unused and the channel's output is zero
};

// lane = channel: floor1 step 2 and the used posts in X order
BT_VB_HD void block_floor(const StreamDev& s, int64_t p, const BlockGeom& g, int c, BlockShared* sh) {
  const Tables& T = *reinterpret_cast<const Tables*>(s.tables);
  const Mapping& m = *rec<Mapping>(s.tables, T.mappings, g.mapping);
  const Floor1& f = *rec<Floor1>(s.tables, T.floors, m.submap_floor[m.mux[c]]);
  const int32_t* fl = s.floors + (p * s.channels + c) * kFloorWords;
  sh->np[c] = 0;
  if (!fl[0]) return;
  floor1_step2(f, fl + 1, sh->fy[c], sh->used[c]);
  int k = 0;
  for (int i = 0; i < f.values; ++i) {
    const int j = f.sorted[i];
    if (!sh->used[c][j]) continue;
    sh->px[c][k] = f.x[j];
    sh->py[c][k] = sh->fy[c][j] * f.multiplier;
    ++k;
  }
  sh->np[c] = k;
}

// lane = spectral line i: inverse coupling of every step, in reverse order
BT_VB_HD void block_couple(const StreamDev& s, int64_t p, const BlockGeom& g, int i) {
  const Tables& T = *reinterpret_cast<const Tables*>(s.tables);
  const Mapping& m = *rec<Mapping>(s.tables, T.mappings, g.mapping);
  float* spec = s.spec + s.packets[p].block_offset * s.channels;
  for (int k = m.coupling_steps - 1; k >= 0; --k) uncouple(spec[m.magnitude[k] * g.n + i], spec[m.angle[k] * g.n + i]);
}

BT_VB_HD const float2* sig(const float* tables, int n) {
  return reinterpret_cast<const float2*>(tables) + signal_at(ilog(static_cast<uint32_t>(n)) - 1);
}

// floor x residue at line i of channel c
BT_VB_HD float block_line(const StreamDev& s, int64_t p, const BlockGeom& g, int c, const BlockShared* sh,
                          const float* tables, int i) {
  const float* spec = s.spec + s.packets[p].block_offset * s.channels + c * g.n;
  const float* dB = tables + 2 * kDbAt;
  return spec[i] * floor_at(sh->px[c], sh->py[c], sh->np[c], i, dB);
}

// lane = k < n / 4: the pre-twiddled FFT input v[k] of channel c
BT_VB_HD void block_pre(const StreamDev& s, int64_t p, const BlockGeom& g, int c, const BlockShared* sh,
                        const float* tables, int k, float2* v) {
  const int M = g.n / 2;
  if (sh->np[c] == 0) {
    v[k] = make_float2(0.f, 0.f);
    return;
  }
  v[k] = cmul(make_float2(block_line(s, p, g, c, sh, tables, 2 * k), block_line(s, p, g, c, sh, tables, M - 1 - 2 * k)),
              sig(tables, g.n)[k]);
}

// lane = butterfly j of the radix-R pass after Ns points of the n / 4-point FFT
BT_VB_HD void block_pass(const float2* in, float2* out, int j, int Ns, int R, const BlockGeom& g, const float* tables) {
  const int H = g.n / 4;
  const float2* tw = sig(tables, g.n) + 2 * H;
  if (R == 8) stockham<8>(in, out, j, Ns, H, tw);
  else if (R == 4) stockham<4>(in, out, j, Ns, H, tw);
  else stockham<2>(in, out, j, Ns, H, tw);
}

// lane = i < n: the windowed IMDCT value i of channel c (u: its DCT-IV) into the packet's scratch
BT_VB_HD void block_out(const StreamDev& s, int64_t p, const BlockGeom& g, int c, const BlockShared* sh,
                        const float* tables, const float* u, int i) {
  const Tables& T = *reinterpret_cast<const Tables*>(s.tables);
  float* out = s.spec + s.packets[p].block_offset * s.channels + c * g.n;
  const int b0 = T.blocksize[0];
  const float* own = reinterpret_cast<const float*>(sig(tables, g.n) + g.n / 2 + g.n / 8);
  const float* shrt = reinterpret_cast<const float*>(sig(tables, b0) + b0 / 2 + b0 / 8);
  out[i] = sh->np[c] == 0 ? 0.f : windowed(u, g.n, i, g.blockflag, g.prev, g.next, b0, shrt, own);
}

// ---- output: lane = output sample t --------------------------------------------------------------------------------
// Overlap-add of the packet whose returned samples hold t and the one before it.
BT_VB_HD float output_sample(const StreamDev& s, int64_t t, int c) {
  const int64_t td = t + s.skip;
  int64_t lo = 1, hi = s.n_packets;  // the first packet p >= 1 with end_sample > td
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (s.packets[mid].end_sample > td) hi = mid;
    else lo = mid + 1;
  }
  if (lo >= s.n_packets) return 0.f;
  const bt_vorbis_packet &a = s.packets[lo - 1], &b = s.packets[lo];
  const int na = block_size(s, a), nb = block_size(s, b);
  const int64_t d = td - a.end_sample, ia = na / 2 + d, ib = nb / 4 - na / 4 + d;
  const float va = ia < na ? s.spec[a.block_offset * s.channels + c * na + ia] : 0.f;
  const float vb = ib >= 0 ? s.spec[b.block_offset * s.channels + c * nb + ib] : 0.f;
  return va + vb;
}

BT_VB_HD float output_mono(const StreamDev& s, int64_t t) {
  double acc = 0;
  for (int c = 0; c < s.channels; ++c) acc += static_cast<double>(output_sample(s, t, c));
  return static_cast<float>(acc / s.channels);
}

}  // namespace vorbis
}  // namespace bt
