// C ABI (include/beatthis.h): native MP3 input -- bt_mp3_probe and bt_stage_mp3_files on the host, bt_mp3_decode on
// the device (kernels_mp3.cu), and the host test hook bt_debug_mp3_decode_host.  Header parsing, the Huffman walk and
// the filter banks are mp3.cuh's, shared by all of them.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <vector>

#include "api_internal.h"
#include "host_pool.h"
#include "mp3.cuh"

namespace {

using bt::mp3::Header;

// ---- Huffman lookup tables (ISO/IEC 11172-3 Table 3-B.7) --------------------------------------------------------------
// Per code table: the code lengths hlen and code words hcod of the symbols (x, y) in row order.
struct CodeTable {
  int size;
  std::vector<int> hlen, hcod;
};

std::vector<CodeTable> code_tables();  // below: tables 1, 2, 3, 5 .. 13, 15, 16, 24, count1 A and B

struct Code {
  int len;
  uint32_t code;
  int sym;
};

// Nested lookup levels of `codes` (all longer than `used` bits, sharing their first `used` bits) at lut[base ..
// base + 2^bits); returns false when the tables do not fit.
bool fill_level(std::vector<uint32_t>& lut, uint32_t base, int bits, int used, const std::vector<Code>& codes) {
  std::vector<std::vector<Code>> sub(1u << bits);
  for (const Code& c : codes) {
    const int rel = c.len - used;
    const uint32_t relcode = c.code & ((1u << rel) - 1);
    if (rel <= bits) {
      const uint32_t first = relcode << (bits - rel);
      for (uint32_t k = 0; k < (1u << (bits - rel)); ++k)
        lut[base + first + k] = 0x80000000u | (static_cast<uint32_t>(rel) << 16) | static_cast<uint32_t>(c.sym);
    } else {
      sub[relcode >> (rel - bits)].push_back(c);
    }
  }
  for (uint32_t k = 0; k < (1u << bits); ++k) {
    if (sub[k].empty()) continue;
    int longest = 0;
    for (const Code& c : sub[k]) longest = std::max(longest, c.len - used - bits);
    const int nb = std::min(longest, bt::mp3::kFirstBits);
    const uint32_t at = static_cast<uint32_t>(lut.size());
    if (at + (1u << nb) > static_cast<uint32_t>(bt::mp3::kLutEntries)) return false;
    lut.resize(at + (1u << nb), 0);
    lut[base + k] = (static_cast<uint32_t>(nb) << 24) | at;
    if (!fill_level(lut, at, nb, used + bits, sub[k])) return false;
  }
  return true;
}

// The lookup tables of mp3.cuh: kLutEntries entries, then the first entry of each of the 34 table slots.
const std::vector<uint32_t>& huffman_lut() {
  static const std::vector<uint32_t> lut = [] {
    std::vector<uint32_t> t(1, 0);  // entry 0: never a valid start
    std::vector<uint32_t> start(34, 0);
    const std::vector<CodeTable> ct = code_tables();
    const int ids[17] = {1, 2, 3, 5, 6, 7, 8, 9, 10, 11, 12, 13, 15, 16, 24, 32, 33};
    for (int j = 0; j < 17; ++j) {
      std::vector<Code> codes;
      for (size_t i = 0; i < ct[j].hlen.size(); ++i) {
        const int x = static_cast<int>(i) / ct[j].size, y = static_cast<int>(i) % ct[j].size;
        codes.push_back({ct[j].hlen[i], static_cast<uint32_t>(ct[j].hcod[i]), ids[j] >= 32 ? static_cast<int>(i)
                                                                                             : (x << 4) | y});
      }
      const uint32_t at = static_cast<uint32_t>(t.size());
      t.resize(at + (1u << bt::mp3::kFirstBits), 0);
      if (!fill_level(t, at, bt::mp3::kFirstBits, 0, codes)) { t.clear(); break; }
      start[ids[j]] = at;
    }
    for (int k = 16; k < 24; ++k) start[k] = start[16];
    for (int k = 24; k < 32; ++k) start[k] = start[24];
    t.resize(bt::mp3::kLutEntries, 0);
    t.insert(t.end(), start.begin(), start.end());
    return t;
  }();
  return lut;
}

// The float tables of the hybrid and synthesis kernels (mp3.cuh, kFloatTables), computed once in float64
const std::vector<float>& float_tables() {
  static const std::vector<float> t = [] {
    std::vector<float> v(bt::mp3::kFloatTables);
    for (int i = 0; i < bt::mp3::kTransformTable; ++i) v[i] = bt::mp3::transform_table_value(i);
    for (int i = 0; i < 512; ++i) v[bt::mp3::kWindowAt + i] = bt::mp3::synth_window(i);
    for (int i = 0; i < 64 * 32; ++i) v[bt::mp3::kCosAt + i] = bt::mp3::synth_cos(i / 32, i % 32);
    return v;
  }();
  return t;
}

// ---- the header walk --------------------------------------------------------------------------------------------------
uint32_t be32(const uint8_t* p) {
  return (static_cast<uint32_t>(p[0]) << 24) | (static_cast<uint32_t>(p[1]) << 16) | (static_cast<uint32_t>(p[2]) << 8) |
         p[3];
}

bool header_at(const uint8_t* b, int64_t end, int64_t p, Header* h) {
  return p >= 0 && p + 4 <= end && bt::mp3::parse_header(be32(b + p), h);
}

bool same_stream(const Header& a, const Header& b) { return a.sample_rate == b.sample_rate && a.channels == b.channels; }

// A frame that starts a stream at p: a header followed by two more consistent headers, each at the length the one
// before gives (or by `end` after the first or the second).  Three chained headers leave a chance match in other
// compressed data negligible.
bool confirmed(const uint8_t* b, int64_t end, int64_t p, Header* h) {
  if (!header_at(b, end, p, h) || p + h->length > end) return false;
  Header n = *h;
  int64_t q = p;
  for (int k = 0; k < 2; ++k) {
    q += n.length;
    if (q == end) return true;
    Header m;
    if (!header_at(b, end, q, &m) || !same_stream(*h, m) || q + m.length > end) return k > 0 && q + 4 > end;
    n = m;
  }
  return true;
}

// End of the audio region: before a trailing ID3v1 tag and an APEv2 tag (footer "APETAGEX", size at 12, header flag)
int64_t audio_end(const uint8_t* b, int64_t n) {
  if (n >= 128 && memcmp(b + n - 128, "TAG", 3) == 0) n -= 128;
  if (n >= 32 && memcmp(b + n - 32, "APETAGEX", 8) == 0) {
    const uint8_t* f = b + n - 32;
    const int64_t size = f[12] | (f[13] << 8) | (f[14] << 16) | (static_cast<int64_t>(f[15]) << 24);
    const bool has_header = f[23] & 0x80;
    const int64_t cut = size + (has_header ? 32 : 0);
    if (cut <= n) n -= cut;
  }
  return n;
}

struct Walk {
  int rc = BT_ERR_FORMAT;
  bool lost_sync = false;
  int64_t first = 0, end = 0;  // the frames' byte range
  std::vector<int64_t> offsets;  // every audio frame (a Xing / Info frame excluded)
  int sample_rate = 0, channels = 0;
  bool gapless = false;
  int64_t delay = 0, padding = 0;
};

// Xing / Info frame at p (header h): its frame count and LAME-style tag (delay, padding), if any
bool xing(const uint8_t* b, int64_t p, const Header& h, int64_t* frames, int64_t* delay, int64_t* padding, bool* tag) {
  const int64_t x = p + 4 + (h.crc ? 2 : 0) + h.side_bytes;
  if (x + 8 > p + h.length || (memcmp(b + x, "Xing", 4) != 0 && memcmp(b + x, "Info", 4) != 0)) return false;
  const uint32_t flags = be32(b + x + 4);
  int64_t q = x + 8;
  *frames = -1;
  if (flags & 1) {
    if (q + 4 > p + h.length) return true;
    *frames = be32(b + q);
    q += 4;
  }
  q += (flags & 2 ? 4 : 0) + (flags & 4 ? 100 : 0) + (flags & 8 ? 4 : 0);
  *tag = false;
  if (q + 24 <= p + h.length && (memcmp(b + q, "LAME", 4) == 0 || memcmp(b + q, "Lavf", 4) == 0 ||
                                 memcmp(b + q, "Lavc", 4) == 0)) {
    const uint8_t* d = b + q + 21;
    *delay = (d[0] << 4) | (d[1] >> 4);
    *padding = ((d[1] & 15) << 8) | d[2];
    *tag = true;
  }
  return true;
}

Walk walk(const uint8_t* b, int64_t n) {
  Walk w;
  int64_t pos = 0;
  if (n >= 10 && memcmp(b, "ID3", 3) == 0)
    pos = 10 + ((b[6] & 0x7F) << 21 | (b[7] & 0x7F) << 14 | (b[8] & 0x7F) << 7 | (b[9] & 0x7F)) + ((b[5] & 0x10) ? 10 : 0);
  const int64_t end = audio_end(b, n);
  Header h;
  while (pos < end && !confirmed(b, end, pos, &h)) ++pos;
  if (pos >= end) return w;
  const Header first = h;
  w.sample_rate = h.sample_rate;
  w.channels = h.channels;
  w.first = pos;
  int64_t xing_frames = -1;
  bool tag = false;
  if (xing(b, pos, h, &xing_frames, &w.delay, &w.padding, &tag)) pos += h.length;
  while (pos + 4 <= end) {
    if (!header_at(b, end, pos, &h)) {
      // trailing bytes are ignored unless a further frame follows: then sync was lost inside the stream
      Header m;
      for (int64_t q = pos + 1; q < end; ++q)
        if (confirmed(b, end, q, &m) && same_stream(first, m)) {
          w.lost_sync = true;
          break;
        }
      break;
    }
    if (!same_stream(first, h)) return w;  // rate or channels change: refused
    if (pos + h.length > end) break;       // a truncated last frame is dropped
    w.offsets.push_back(pos);
    pos += h.length;
  }
  w.end = pos;
  if (w.offsets.empty()) return w;
  const int64_t N = static_cast<int64_t>(w.offsets.size());
  w.gapless = tag && xing_frames == N;
  w.rc = BT_OK;
  return w;
}

void fill_info(const Walk& w, bt_mp3_info* info) {
  const int64_t N = static_cast<int64_t>(w.offsets.size());
  info->sample_rate = w.sample_rate;
  info->channels = w.channels;
  info->n_frames = N;
  info->gapless = w.gapless;
  info->skip = w.gapless ? w.delay + 529 : 0;
  info->padding = w.gapless ? w.padding : 0;
  const int64_t stop = w.gapless ? std::min<int64_t>(1152 * N, 1152 * N - w.padding + 529) : 1152 * N;
  info->n_samples = std::max<int64_t>(0, stop - info->skip);
  info->frames_offset = w.first;
  info->frames_bytes = w.end - w.first;
  info->max_frames = N;
  info->main_bytes = w.end - w.first;
}

int check_streams(const bt_mp3_stream* s, int32_t n) {
  for (int32_t i = 0; i < n; ++i)
    if (s[i].byte_offset < 0 || s[i].byte_count < 0 || s[i].frame_offset < 0 || s[i].n_frames < 0 || s[i].skip < 0 ||
        s[i].n_samples < 0 || s[i].out_offset < 0 || s[i].channels < 1 || s[i].channels > 2 ||
        (s[i].sample_rate != 32000 && s[i].sample_rate != 44100 && s[i].sample_rate != 48000))
      return 1;
  return 0;
}

}  // namespace

extern "C" {

int bt_mp3_probe(const char* path, bt_mp3_info* info) {
  if (!path || !info) return BT_ERR_ARG;
  memset(info, 0, sizeof(*info));
  std::vector<uint8_t> b;
  if (!bt::read_whole_file(path, &b)) return BT_ERR_IO;
  const Walk w = walk(b.data(), static_cast<int64_t>(b.size()));
  if (w.rc != BT_OK) return w.rc;
  fill_info(w, info);
  return BT_OK;
}

int bt_stage_mp3_files(const char* const* paths, const bt_mp3_info* infos, int32_t n_files, uint8_t* bytes_dst,
                       const int64_t* byte_offsets, bt_mp3_frame* frames_dst, const int64_t* frame_offsets,
                       int64_t* main_bytes, int64_t* n_frames, int32_t n_threads, int32_t* status) {
  if (n_files <= 0) return BT_OK;
  if (!paths || !infos || !bytes_dst || !byte_offsets || !frames_dst || !frame_offsets || !main_bytes || !n_frames)
    return BT_ERR_ARG;
  std::atomic<int> failed{0};
  bt::run_pool(static_cast<size_t>(n_files), n_threads, [&](size_t i) {
    const bt_mp3_info& in = infos[i];
    n_frames[i] = main_bytes[i] = 0;
    int rc = BT_ERR_IO;
    std::vector<uint8_t> b;
    if (bt::read_whole_file(paths[i], &b)) {
      const Walk w = walk(b.data(), static_cast<int64_t>(b.size()));
      const int64_t N = static_cast<int64_t>(w.offsets.size());
      if (w.rc == BT_OK && !w.lost_sync && N == in.n_frames && N <= in.max_frames && w.first == in.frames_offset) {
        uint8_t* dst = bytes_dst + byte_offsets[i];
        bt_mp3_frame* fr = frames_dst + frame_offsets[i];
        int64_t at = 0;
        rc = BT_OK;
        for (int64_t k = 0; k < N && rc == BT_OK; ++k) {
          const int64_t p = w.offsets[k];
          Header h;
          bt::mp3::parse_header(be32(b.data() + p), &h);
          const int64_t side = p + 4 + (h.crc ? 2 : 0);
          const int64_t body = side + h.side_bytes;
          const int64_t len = p + h.length - body;
          if (len < 0 || at + len > in.main_bytes) { rc = BT_ERR_IO; break; }
          bt_mp3_frame f{};
          f.header = be32(b.data() + p);
          memcpy(f.side_info, b.data() + side, static_cast<size_t>(h.side_bytes));
          const int mdb = (f.side_info[0] << 1) | (f.side_info[1] >> 7);
          f.main_start = at - mdb;
          f.first_sample = 1152 * k;
          f.main_bytes = static_cast<int32_t>(len);
          fr[k] = f;
          memcpy(dst + at, b.data() + body, static_cast<size_t>(len));
          at += len;
        }
        if (rc == BT_OK) {
          n_frames[i] = N;
          main_bytes[i] = at;
        }
      }
    }
    if (rc != BT_OK) {
      n_frames[i] = main_bytes[i] = 0;
      failed.fetch_add(1);
    }
    if (status) status[i] = rc;
  });
  return failed.load() ? BT_ERR_IO : BT_OK;
}

int bt_mp3_decode(bt_ctx* c, const uint8_t* bytes_dev, const bt_mp3_frame* frames_dev,
                  const bt_mp3_stream* streams_host, int32_t n_streams, int32_t mode, void* out_dev, int32_t* status_dev,
                  void* stream) {
  static const char* fn = "bt_mp3_decode";
  if (!c) return BT_ERR_ARG;
  if (n_streams < 0 || n_streams > 65535) return fail(c, BT_ERR_ARG, "%s: need 0 <= n_streams <= 65535", fn);
  if (mode != BT_MP3_MONO_F32 && mode != BT_MP3_CHANNELS_F64) return fail(c, BT_ERR_ARG, "%s: unknown mode %d", fn, mode);
  if (n_streams == 0) return BT_OK;
  if (!bytes_dev || !frames_dev || !streams_host || !out_dev || !status_dev)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  if (check_streams(streams_host, n_streams))
    return fail(c, BT_ERR_ARG, "%s: a stream has a negative count or offset, channels outside 1..2 or a sample rate "
                "other than 32000, 44100 or 48000", fn);
  const std::vector<uint32_t>& lut = huffman_lut();
  if (lut.size() != static_cast<size_t>(bt::mp3::kLutEntries + 34) || lut[bt::mp3::kLutEntries + 1] == 0)
    return fail(c, BT_ERR_STATE, "%s: the Huffman lookup tables do not fit", fn);
  const size_t per_gran = sizeof(bt::mp3::GranuleRec) + sizeof(float) * 32 * bt::mp3::kBlock;
  int64_t grans = 0, max_frames = 0, max_out = 0;
  for (int32_t i = 0; i < n_streams; ++i) {
    grans += 2 * streams_host[i].n_frames * streams_host[i].channels;
    max_frames = std::max(max_frames, streams_host[i].n_frames);
    if (streams_host[i].n_samples > 0)  // granules that hold output samples, decoded or zero-filled
      max_out = std::max(max_out, (streams_host[i].skip + streams_host[i].n_samples + bt::mp3::kLines - 1) / bt::mp3::kLines);
  }
  cudaStream_t st;
  int r = enter(c, fn, stream, &st);
  if (r != BT_OK) return r;
  const size_t bytes = per_gran * static_cast<size_t>(std::max<int64_t>(grans, 1));
  BT_CUDA(c, c->mp3_ws.reserve(bytes, bytes + bytes / 4));
  std::vector<Mp3StreamDev> sd(n_streams);
  char* recs = c->mp3_ws.get();
  float* blocks = reinterpret_cast<float*>(recs + sizeof(bt::mp3::GranuleRec) * static_cast<size_t>(std::max<int64_t>(grans, 1)));
  for (int32_t i = 0; i < n_streams; ++i) {
    const bt_mp3_stream& s = streams_host[i];
    sd[i] = Mp3StreamDev{bytes_dev + s.byte_offset, frames_dev + s.frame_offset, recs, blocks, s.byte_count, s.n_frames,
                         s.skip, s.n_samples, s.out_offset, s.channels, bt::mp3::rate_index(s.sample_rate)};
    const int64_t g = 2 * s.n_frames * s.channels;
    recs += sizeof(bt::mp3::GranuleRec) * g;
    blocks += static_cast<int64_t>(32) * bt::mp3::kBlock * g;
  }
  const Mp3StreamDev* d[1];
  if ((r = stage(c, st, {{sd.data(), sd.size()}}, d)) != BT_OK) return r;
  const uint32_t* dl[1];
  if ((r = stage(c, st, {{lut.data(), lut.size()}}, dl)) != BT_OK) return r;
  const std::vector<float>& ft = float_tables();
  const float* dt[1];
  if ((r = stage(c, st, {{ft.data(), ft.size()}}, dt)) != BT_OK) return r;
  if (max_frames > 0) {
    launch_mp3_granules(d[0], n_streams, max_frames, dl[0], status_dev, st);
    BT_LAUNCHED(c, "mp3_granules", st);
    launch_mp3_hybrid(d[0], n_streams, max_frames, dt[0], status_dev, st);
    BT_LAUNCHED(c, "mp3_hybrid", st);
  }
  if (max_out > 0) {  // also for streams without frames (a failed staging): their output is zero-filled
    launch_mp3_synth(d[0], n_streams, max_out, dt[0], mode, out_dev, status_dev, st);
    BT_LAUNCHED(c, "mp3_synth", st);
  }
  return BT_OK;
}

int bt_debug_mp3_decode_host(const uint8_t* bytes_host, const bt_mp3_frame* frames_host,
                             const bt_mp3_stream* streams_host, int32_t n_streams, int32_t mode, void* out_host,
                             int32_t* status_host) {
  namespace m = bt::mp3;
  if (n_streams < 0) return BT_ERR_ARG;
  if (n_streams == 0) return BT_OK;
  if (!bytes_host || !frames_host || !streams_host || !out_host || !status_host || check_streams(streams_host, n_streams) ||
      (mode != BT_MP3_MONO_F32 && mode != BT_MP3_CHANNELS_F64))
    return BT_ERR_ARG;
  const std::vector<uint32_t>& lut = huffman_lut();
  if (lut.size() != static_cast<size_t>(m::kLutEntries + 34)) return BT_ERR_STATE;
  const std::vector<float>& ft = float_tables();
  const float* tt = ft.data();
  const float* win = ft.data() + m::kWindowAt;
  const float* ncos = ft.data() + m::kCosAt;
  for (int32_t si = 0; si < n_streams; ++si) {
    const bt_mp3_stream& s = streams_host[si];
    const int nch = s.channels, ri = m::rate_index(s.sample_rate);
    const int64_t G = 2 * s.n_frames;
    std::vector<m::GranuleRec> recs(static_cast<size_t>(G * nch));
    std::vector<float> blocks(static_cast<size_t>(G * nch * 32 * m::kBlock));
    const uint8_t* main = bytes_host + s.byte_offset;
    for (int64_t f = 0; f < s.n_frames && status_host[si] == BT_OK; ++f) {
      const bt_mp3_frame& fr = frames_host[s.frame_offset + f];
      for (int ch = 0; ch < nch; ++ch)
        if (!m::decode_frame_channel(main, s.byte_count, fr.main_start, fr.header, fr.side_info, nch, ch, ri,
                                     lut.data(), recs.data() + f * 2 * nch))
          status_host[si] = BT_ERR_IO;
    }
    std::vector<float> x(2 * m::kLines), y(2 * m::kLines);
    for (int64_t g = 0; status_host[si] == BT_OK && g < G; ++g) {
      const m::GranuleRec* r = recs.data() + g * nch;
      const uint32_t header = frames_host[s.frame_offset + g / 2].header;
      int bound[4] = {-1, -1, -1, -1};
      for (int i = 0; i < m::kLines; ++i) m::hybrid_requant(r, nch, ri, i, x.data(), bound);
      for (int i = 0; i < m::kLines; ++i) m::hybrid_stereo(r, nch, ri, header, i, x.data(), bound);
      for (int c = 0; c < nch; ++c)
        for (int i = 0; i < m::kLines; ++i) y[c * m::kLines + i] = x[c * m::kLines + m::reorder_src(r[c], ri, i)];
      for (int c = 0; c < nch; ++c)
        for (int i = 0; i < m::kLines; ++i) x[c * m::kLines + i] = m::antialias(y.data() + c * m::kLines, r[c], i);
      for (int c = 0; c < nch; ++c)
        for (int o = 0; o < 32 * m::kBlock; ++o)
          blocks[((g * nch + c) * 32 + o / m::kBlock) * m::kBlock + o % m::kBlock] =
              m::imdct_value(x.data() + c * m::kLines + 18 * (o / m::kBlock), r[c], o / m::kBlock, o % m::kBlock, tt);
    }
    std::vector<float> S(33 * 32), V(33 * 64), pcm(2 * m::kLines);
    const int64_t G_out = (s.skip + s.n_samples + m::kLines - 1) / m::kLines;  // granules holding output samples
    for (int64_t g = 0; g < G_out; ++g) {
      const int64_t first = g * m::kLines - s.skip;
      if (first >= s.n_samples || first + m::kLines <= 0) continue;
      const bool ok = status_host[si] == BT_OK && g < G;
      for (int c = 0; ok && c < nch; ++c) {
        for (int e = 0; e < 33 * 32; ++e) S[e] = m::slot_sample(blocks.data(), nch, c, g, e / 32 - 15, e % 32);
        for (int e = 0; e < 33 * 64; ++e) V[e] = m::matrix_value(S.data() + (e / 64) * 32, ncos, e % 64);
        for (int e = 0; e < m::kLines; ++e) pcm[c * m::kLines + e] = m::window_sum(V.data(), win, 15 + e / 32, e % 32);
      }
      for (int e = 0; e < m::kLines; ++e) {
        const int64_t t = first + e;
        if (t < 0 || t >= s.n_samples) continue;
        if (mode == BT_MP3_MONO_F32) {
          static_cast<float*>(out_host)[s.out_offset + t] =
              ok ? m::mono_sample(pcm[e], pcm[m::kLines + e], nch) : 0.f;
        } else {
          for (int c = 0; c < nch; ++c)
            static_cast<double*>(out_host)[s.out_offset + t * nch + c] = ok ? static_cast<double>(pcm[c * m::kLines + e]) : 0.0;
        }
      }
    }
  }
  return BT_OK;
}

}  // extern "C"

namespace {

// ISO/IEC 11172-3 Table 3-B.7: hlen and hcod of every big-values table in row order of (x, y); count1 tables A and B
// by the value vwxy.
std::vector<CodeTable> code_tables() {
  return {
      // table 1
      {2,
       {1, 3, 2, 3},
       {1, 1, 1, 0}},
      // table 2
      {3,
       {1, 3, 6, 3, 3, 5, 5, 5, 6},
       {1, 2, 1, 3, 1, 1, 3, 2, 0}},
      // table 3
      {3,
       {2, 2, 6, 3, 2, 5, 5, 5, 6},
       {3, 2, 1, 1, 1, 1, 3, 2, 0}},
      // table 5
      {4,
       {1, 3, 6, 7, 3, 3, 6, 7, 6, 6, 7, 8, 7, 6, 7, 8},
       {1, 2, 6, 5, 3, 1, 4, 4, 7, 5, 7, 1, 6, 1, 1, 0}},
      // table 6
      {4,
       {3, 3, 5, 7, 3, 2, 4, 5, 4, 4, 5, 6, 6, 5, 6, 7},
       {7, 3, 5, 1, 6, 2, 3, 2, 5, 4, 4, 1, 3, 3, 2, 0}},
      // table 7
      {6,
       {1, 3, 6, 8, 8, 9, 3, 4, 6, 7, 7, 8, 6, 5, 7, 8, 8, 9, 7, 7, 8, 9, 9, 9, 7, 7, 8, 9, 9, 10, 8, 8, 9, 10, 10,
        10},
       {1, 2, 10, 19, 16, 10, 3, 3, 7, 10, 5, 3, 11, 4, 13, 17, 8, 4, 12, 11, 18, 15, 11, 2, 7, 6, 9, 14, 3, 1, 6,
        4, 5, 3, 2, 0}},
      // table 8
      {6,
       {2, 3, 6, 8, 8, 9, 3, 2, 4, 8, 8, 8, 6, 4, 6, 8, 8, 9, 8, 8, 8, 9, 9, 10, 8, 7, 8, 9, 10, 10, 9, 8, 9, 9, 11,
        11},
       {3, 4, 6, 18, 12, 5, 5, 1, 2, 16, 9, 3, 7, 3, 5, 14, 7, 3, 19, 17, 15, 13, 10, 4, 13, 5, 8, 11, 5, 1, 12, 4,
        4, 1, 1, 0}},
      // table 9
      {6,
       {3, 3, 5, 6, 8, 9, 3, 3, 4, 5, 6, 8, 4, 4, 5, 6, 7, 8, 6, 5, 6, 7, 7, 8, 7, 6, 7, 7, 8, 9, 8, 7, 8, 8, 9, 9},
       {7, 5, 9, 14, 15, 7, 6, 4, 5, 5, 6, 7, 7, 6, 8, 8, 8, 5, 15, 6, 9, 10, 5, 1, 11, 7, 9, 6, 4, 1, 14, 4, 6, 2,
        6, 0}},
      // table 10
      {8,
       {1, 3, 6, 8, 9, 9, 9, 10, 3, 4, 6, 7, 8, 9, 8, 8, 6, 6, 7, 8, 9, 10, 9, 9, 7, 7, 8, 9, 10, 10, 9, 10, 8, 8,
        9, 10, 10, 10, 10, 10, 9, 9, 10, 10, 11, 11, 10, 11, 8, 8, 9, 10, 10, 10, 11, 11, 9, 8, 9, 10, 10,
        11, 11, 11},
       {1, 2, 10, 23, 35, 30, 12, 17, 3, 3, 8, 12, 18, 21, 12, 7, 11, 9, 15, 21, 32, 40, 19, 6, 14, 13, 22, 34, 46,
        23, 18, 7, 20, 19, 33, 47, 27, 22, 9, 3, 31, 22, 41, 26, 21, 20, 5, 3, 14, 13, 10, 11, 16, 6, 5, 1,
        9, 8, 7, 8, 4, 4, 2, 0}},
      // table 11
      {8,
       {2, 3, 5, 7, 8, 9, 8, 9, 3, 3, 4, 6, 8, 8, 7, 8, 5, 5, 6, 7, 8, 9, 8, 8, 7, 6, 7, 9, 8, 10, 8, 9, 8, 8, 8, 9,
        9, 10, 9, 10, 8, 8, 9, 10, 10, 11, 10, 11, 8, 7, 7, 8, 9, 10, 10, 10, 8, 7, 8, 9, 10, 10, 10, 10},
       {3, 4, 10, 24, 34, 33, 21, 15, 5, 3, 4, 10, 32, 17, 11, 10, 11, 7, 13, 18, 30, 31, 20, 5, 25, 11, 19, 59, 27,
        18, 12, 5, 35, 33, 31, 58, 30, 16, 7, 5, 28, 26, 32, 19, 17, 15, 8, 14, 14, 12, 9, 13, 14, 9, 4, 1,
        11, 4, 6, 6, 6, 3, 2, 0}},
      // table 12
      {8,
       {4, 3, 5, 7, 8, 9, 9, 9, 3, 3, 4, 5, 7, 7, 8, 8, 5, 4, 5, 6, 7, 8, 7, 8, 6, 5, 6, 6, 7, 8, 8, 8, 7, 6, 7, 7,
        8, 8, 8, 9, 8, 7, 8, 8, 8, 9, 8, 9, 8, 7, 7, 8, 8, 9, 9, 10, 9, 8, 8, 9, 9, 9, 9, 10},
       {9, 6, 16, 33, 41, 39, 38, 26, 7, 5, 6, 9, 23, 16, 26, 11, 17, 7, 11, 14, 21, 30, 10, 7, 17, 10, 15, 12, 18,
        28, 14, 5, 32, 13, 22, 19, 18, 16, 9, 5, 40, 17, 31, 29, 17, 13, 4, 2, 27, 12, 11, 15, 10, 7, 4, 1,
        27, 12, 8, 12, 6, 3, 1, 0}},
      // table 13
      {16,
       {1, 4, 6, 7, 8, 9, 9, 10, 9, 10, 11, 11, 12, 12, 13, 13, 3, 4, 6, 7, 8, 8, 9, 9, 9, 9, 10, 10, 11, 12, 12,
        12, 6, 6, 7, 8, 9, 9, 10, 10, 9, 10, 10, 11, 11, 12, 13, 13, 7, 7, 8, 9, 9, 10, 10, 10, 10, 11, 11,
        11, 11, 12, 13, 13, 8, 7, 9, 9, 10, 10, 11, 11, 10, 11, 11, 12, 12, 13, 13, 14, 9, 8, 9, 10, 10, 10,
        11, 11, 11, 11, 12, 11, 13, 13, 14, 14, 9, 9, 10, 10, 11, 11, 11, 11, 11, 12, 12, 12, 13, 13, 14,
        14, 10, 9, 10, 11, 11, 11, 12, 12, 12, 12, 13, 13, 13, 14, 16, 16, 9, 8, 9, 10, 10, 11, 11, 12, 12,
        12, 12, 13, 13, 14, 15, 15, 10, 9, 10, 10, 11, 11, 11, 13, 12, 13, 13, 14, 14, 14, 16, 15, 10, 10,
        10, 11, 11, 12, 12, 13, 12, 13, 14, 13, 14, 15, 16, 17, 11, 10, 10, 11, 12, 12, 12, 12, 13, 13, 13,
        14, 15, 15, 15, 16, 11, 11, 11, 12, 12, 13, 12, 13, 14, 14, 15, 15, 15, 16, 16, 16, 12, 11, 12, 13,
        13, 13, 14, 14, 14, 14, 14, 15, 16, 15, 16, 16, 13, 12, 12, 13, 13, 13, 15, 14, 14, 17, 15, 15, 15,
        17, 16, 16, 12, 12, 13, 14, 14, 14, 15, 14, 15, 15, 16, 16, 19, 18, 19, 16},
       {1, 5, 14, 21, 34, 51, 46, 71, 42, 52, 68, 52, 67, 44, 43, 19, 3, 4, 12, 19, 31, 26, 44, 33, 31, 24, 32, 24,
        31, 35, 22, 14, 15, 13, 23, 36, 59, 49, 77, 65, 29, 40, 30, 40, 27, 33, 42, 16, 22, 20, 37, 61, 56,
        79, 73, 64, 43, 76, 56, 37, 26, 31, 25, 14, 35, 16, 60, 57, 97, 75, 114, 91, 54, 73, 55, 41, 48, 53,
        23, 24, 58, 27, 50, 96, 76, 70, 93, 84, 77, 58, 79, 29, 74, 49, 41, 17, 47, 45, 78, 74, 115, 94, 90,
        79, 69, 83, 71, 50, 59, 38, 36, 15, 72, 34, 56, 95, 92, 85, 91, 90, 86, 73, 77, 65, 51, 44, 43, 42,
        43, 20, 30, 44, 55, 78, 72, 87, 78, 61, 46, 54, 37, 30, 20, 16, 53, 25, 41, 37, 44, 59, 54, 81, 66,
        76, 57, 54, 37, 18, 39, 11, 35, 33, 31, 57, 42, 82, 72, 80, 47, 58, 55, 21, 22, 26, 38, 22, 53, 25,
        23, 38, 70, 60, 51, 36, 55, 26, 34, 23, 27, 14, 9, 7, 34, 32, 28, 39, 49, 75, 30, 52, 48, 40, 52,
        28, 18, 17, 9, 5, 45, 21, 34, 64, 56, 50, 49, 45, 31, 19, 12, 15, 10, 7, 6, 3, 48, 23, 20, 39, 36,
        35, 53, 21, 16, 23, 13, 10, 6, 1, 4, 2, 16, 15, 17, 27, 25, 20, 29, 11, 17, 12, 16, 8, 1, 1, 0, 1}},
      // table 15
      {16,
       {3, 4, 5, 7, 7, 8, 9, 9, 9, 10, 10, 11, 11, 11, 12, 13, 4, 3, 5, 6, 7, 7, 8, 8, 8, 9, 9, 10, 10, 10, 11, 11,
        5, 5, 5, 6, 7, 7, 8, 8, 8, 9, 9, 10, 10, 11, 11, 11, 6, 6, 6, 7, 7, 8, 8, 9, 9, 9, 10, 10, 10, 11,
        11, 11, 7, 6, 7, 7, 8, 8, 9, 9, 9, 9, 10, 10, 10, 11, 11, 11, 8, 7, 7, 8, 8, 8, 9, 9, 9, 9, 10, 10,
        11, 11, 11, 12, 9, 7, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10, 11, 11, 12, 12, 9, 8, 8, 9, 9, 9, 9, 10, 10,
        10, 10, 10, 11, 11, 11, 12, 9, 8, 8, 9, 9, 9, 9, 10, 10, 10, 10, 11, 11, 12, 12, 12, 9, 8, 9, 9, 9,
        9, 10, 10, 10, 11, 11, 11, 11, 12, 12, 12, 10, 9, 9, 9, 10, 10, 10, 10, 10, 11, 11, 11, 11, 12, 13,
        12, 10, 9, 9, 9, 10, 10, 10, 10, 11, 11, 11, 11, 12, 12, 12, 13, 11, 10, 9, 10, 10, 10, 11, 11, 11,
        11, 11, 11, 12, 12, 13, 13, 11, 10, 10, 10, 10, 11, 11, 11, 11, 12, 12, 12, 12, 12, 13, 13, 12, 11,
        11, 11, 11, 11, 11, 11, 12, 12, 12, 12, 13, 13, 12, 13, 12, 11, 11, 11, 11, 11, 11, 12, 12, 12, 12,
        12, 13, 13, 13, 13},
       {7, 12, 18, 53, 47, 76, 124, 108, 89, 123, 108, 119, 107, 81, 122, 63, 13, 5, 16, 27, 46, 36, 61, 51, 42, 70,
        52, 83, 65, 41, 59, 36, 19, 17, 15, 24, 41, 34, 59, 48, 40, 64, 50, 78, 62, 80, 56, 33, 29, 28, 25,
        43, 39, 63, 55, 93, 76, 59, 93, 72, 54, 75, 50, 29, 52, 22, 42, 40, 67, 57, 95, 79, 72, 57, 89, 69,
        49, 66, 46, 27, 77, 37, 35, 66, 58, 52, 91, 74, 62, 48, 79, 63, 90, 62, 40, 38, 125, 32, 60, 56, 50,
        92, 78, 65, 55, 87, 71, 51, 73, 51, 70, 30, 109, 53, 49, 94, 88, 75, 66, 122, 91, 73, 56, 42, 64,
        44, 21, 25, 90, 43, 41, 77, 73, 63, 56, 92, 77, 66, 47, 67, 48, 53, 36, 20, 71, 34, 67, 60, 58, 49,
        88, 76, 67, 106, 71, 54, 38, 39, 23, 15, 109, 53, 51, 47, 90, 82, 58, 57, 48, 72, 57, 41, 23, 27,
        62, 9, 86, 42, 40, 37, 70, 64, 52, 43, 70, 55, 42, 25, 29, 18, 11, 11, 118, 68, 30, 55, 50, 46, 74,
        65, 49, 39, 24, 16, 22, 13, 14, 7, 91, 44, 39, 38, 34, 63, 52, 45, 31, 52, 28, 19, 14, 8, 9, 3, 123,
        60, 58, 53, 47, 43, 32, 22, 37, 24, 17, 12, 15, 10, 2, 1, 71, 37, 34, 30, 28, 20, 17, 26, 21, 16,
        10, 6, 8, 6, 2, 0}},
      // table 16
      {16,
       {1, 4, 6, 8, 9, 9, 10, 10, 11, 11, 11, 12, 12, 12, 13, 9, 3, 4, 6, 7, 8, 9, 9, 9, 10, 10, 10, 11, 12, 11, 12,
        8, 6, 6, 7, 8, 9, 9, 10, 10, 11, 10, 11, 11, 11, 12, 12, 9, 8, 7, 8, 9, 9, 10, 10, 10, 11, 11, 12,
        12, 12, 13, 13, 10, 9, 8, 9, 9, 10, 10, 11, 11, 11, 12, 12, 12, 13, 13, 13, 9, 9, 8, 9, 9, 10, 11,
        11, 12, 11, 12, 12, 13, 13, 13, 14, 10, 10, 9, 9, 10, 11, 11, 11, 11, 12, 12, 12, 12, 13, 13, 14,
        10, 10, 9, 10, 10, 11, 11, 11, 12, 12, 13, 13, 13, 13, 15, 15, 10, 10, 10, 10, 11, 11, 11, 12, 12,
        13, 13, 13, 13, 14, 14, 14, 10, 11, 10, 10, 11, 11, 12, 12, 13, 13, 13, 13, 14, 13, 14, 13, 11, 11,
        11, 10, 11, 12, 12, 12, 12, 13, 14, 14, 14, 15, 15, 14, 10, 12, 11, 11, 11, 12, 12, 13, 14, 14, 14,
        14, 14, 14, 13, 14, 11, 12, 12, 12, 12, 12, 13, 13, 13, 13, 15, 14, 14, 14, 14, 16, 11, 14, 12, 12,
        12, 13, 13, 14, 14, 14, 16, 15, 15, 15, 17, 15, 11, 13, 13, 11, 12, 14, 14, 13, 14, 14, 15, 16, 15,
        17, 15, 14, 11, 9, 8, 8, 9, 9, 10, 10, 10, 11, 11, 11, 11, 11, 11, 11, 8},
       {1, 5, 14, 44, 74, 63, 110, 93, 172, 149, 138, 242, 225, 195, 376, 17, 3, 4, 12, 20, 35, 62, 53, 47, 83, 75,
        68, 119, 201, 107, 207, 9, 15, 13, 23, 38, 67, 58, 103, 90, 161, 72, 127, 117, 110, 209, 206, 16,
        45, 21, 39, 69, 64, 114, 99, 87, 158, 140, 252, 212, 199, 387, 365, 26, 75, 36, 68, 65, 115, 101,
        179, 164, 155, 264, 246, 226, 395, 382, 362, 9, 66, 30, 59, 56, 102, 185, 173, 265, 142, 253, 232,
        400, 388, 378, 445, 16, 111, 54, 52, 100, 184, 178, 160, 133, 257, 244, 228, 217, 385, 366, 715, 10,
        98, 48, 91, 88, 165, 157, 148, 261, 248, 407, 397, 372, 380, 889, 884, 8, 85, 84, 81, 159, 156, 143,
        260, 249, 427, 401, 392, 383, 727, 713, 708, 7, 154, 76, 73, 141, 131, 256, 245, 426, 406, 394, 384,
        735, 359, 710, 352, 11, 139, 129, 67, 125, 247, 233, 229, 219, 393, 743, 737, 720, 885, 882, 439, 4,
        243, 120, 118, 115, 227, 223, 396, 746, 742, 736, 721, 712, 706, 223, 436, 6, 202, 224, 222, 218,
        216, 389, 386, 381, 364, 888, 443, 707, 440, 437, 1728, 4, 747, 211, 210, 208, 370, 379, 734, 723,
        714, 1735, 883, 877, 876, 3459, 865, 2, 377, 369, 102, 187, 726, 722, 358, 711, 709, 866, 1734, 871,
        3458, 870, 434, 0, 12, 10, 7, 11, 10, 17, 11, 9, 13, 12, 10, 7, 5, 3, 1, 3}},
      // table 24
      {16,
       {4, 4, 6, 7, 8, 9, 9, 10, 10, 11, 11, 11, 11, 11, 12, 9, 4, 4, 5, 6, 7, 8, 8, 9, 9, 9, 10, 10, 10, 10, 10, 8,
        6, 5, 6, 7, 7, 8, 8, 9, 9, 9, 9, 10, 10, 10, 11, 7, 7, 6, 7, 7, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10, 10,
        7, 8, 7, 7, 8, 8, 8, 8, 9, 9, 9, 10, 10, 10, 10, 11, 7, 9, 7, 8, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10,
        10, 10, 7, 9, 8, 8, 8, 8, 9, 9, 9, 9, 10, 10, 10, 10, 10, 11, 7, 10, 8, 8, 8, 9, 9, 9, 9, 10, 10,
        10, 10, 10, 11, 11, 8, 10, 9, 9, 9, 9, 9, 9, 9, 9, 10, 10, 10, 10, 11, 11, 8, 10, 9, 9, 9, 9, 9, 9,
        10, 10, 10, 10, 10, 11, 11, 11, 8, 11, 9, 9, 9, 9, 10, 10, 10, 10, 10, 10, 11, 11, 11, 11, 8, 11,
        10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 11, 11, 11, 11, 8, 11, 10, 10, 10, 10, 10, 10, 10, 10, 10, 11,
        11, 11, 11, 11, 8, 11, 10, 10, 10, 10, 10, 10, 10, 11, 11, 11, 11, 11, 11, 11, 8, 12, 10, 10, 10,
        10, 10, 10, 11, 11, 11, 11, 11, 11, 11, 11, 8, 8, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 8, 8, 8, 8, 4},
       {15, 13, 46, 80, 146, 262, 248, 434, 426, 669, 653, 649, 621, 517, 1032, 88, 14, 12, 21, 38, 71, 130, 122,
        216, 209, 198, 327, 345, 319, 297, 279, 42, 47, 22, 41, 74, 68, 128, 120, 221, 207, 194, 182, 340,
        315, 295, 541, 18, 81, 39, 75, 70, 134, 125, 116, 220, 204, 190, 178, 325, 311, 293, 271, 16, 147,
        72, 69, 135, 127, 118, 112, 210, 200, 188, 352, 323, 306, 285, 540, 14, 263, 66, 129, 126, 119, 114,
        214, 202, 192, 180, 341, 317, 301, 281, 262, 12, 249, 123, 121, 117, 113, 215, 206, 195, 185, 347,
        330, 308, 291, 272, 520, 10, 435, 115, 111, 109, 211, 203, 196, 187, 353, 332, 313, 298, 283, 531,
        381, 17, 427, 212, 208, 205, 201, 193, 186, 177, 169, 320, 303, 286, 268, 514, 377, 16, 335, 199,
        197, 191, 189, 181, 174, 333, 321, 305, 289, 275, 521, 379, 371, 11, 668, 184, 183, 179, 175, 344,
        331, 314, 304, 290, 277, 530, 383, 373, 366, 10, 652, 346, 171, 168, 164, 318, 309, 299, 287, 276,
        263, 513, 375, 368, 362, 6, 648, 322, 316, 312, 307, 302, 292, 284, 269, 261, 512, 376, 370, 364,
        359, 4, 620, 300, 296, 294, 288, 282, 273, 266, 515, 380, 374, 369, 365, 361, 357, 2, 1033, 280,
        278, 274, 267, 264, 259, 382, 378, 372, 367, 363, 360, 358, 356, 0, 43, 20, 19, 17, 15, 13, 11, 9,
        7, 6, 4, 7, 5, 3, 1, 3}},
      // count1 A
      {16, {1, 4, 4, 5, 4, 6, 5, 6, 4, 5, 5, 6, 5, 6, 6, 6}, {1, 5, 4, 5, 6, 5, 4, 4, 7, 3, 6, 0, 7, 2, 3, 1}},
      // count1 B
      {16, {4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4}, {15, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1, 0}},
  };
}

}  // namespace
