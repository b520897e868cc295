// C ABI (include/beatthis.h): native Ogg Vorbis input -- bt_vorbis_probe and bt_stage_vorbis_files on the host,
// bt_vorbis_decode on the device (kernels_vorbis.cu), and the host test hook bt_debug_vorbis_decode_host.  The Ogg
// page walk, the header parser and the decode-table builder are here; the packet arithmetic is vorbis.cuh's.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <vector>

#include "api_internal.h"
#include "host_pool.h"
#include "vorbis.cuh"

namespace {

namespace vb = bt::vorbis;

// ---- Ogg pages --------------------------------------------------------------------------------------------------------
// CRC-32 of Ogg: polynomial 0x04C11DB7, initial value 0, not reflected, no final xor
const uint32_t* ogg_crc_table() {
  static uint32_t t[256];
  static const bool done = [] {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t r = i << 24;
      for (int k = 0; k < 8; ++k) r = (r & 0x80000000u) ? (r << 1) ^ 0x04C11DB7u : r << 1;
      t[i] = r;
    }
    return true;
  }();
  (void)done;
  return t;
}

uint32_t le32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | (static_cast<uint32_t>(p[3]) << 24); }

struct Packet {
  int64_t off, len;  // in Walk::data
  int page;          // the page it completes on
};

struct Walk {
  int rc = BT_ERR_FORMAT;
  bool audio_bad = false;           // a CRC, sequence or continuation error after the headers
  std::vector<uint8_t> data;        // every completed packet, back to back
  std::vector<Packet> packets;      // headers first
  std::vector<int64_t> granule;     // per page
};

// The pages of a file from byte 0 and their packets.  A partial last page, and a packet continued into it, are dropped.
// Errors up to the page that completes the third packet (the setup header) are BT_ERR_FORMAT; later ones set audio_bad
// when check_audio is set (the probe leaves the audio pages' CRCs to staging).
Walk walk_pages(const uint8_t* b, int64_t n, bool check_audio) {
  Walk w;
  const uint32_t* crc_t = ogg_crc_table();
  int64_t pos = 0;
  uint32_t serial = 0, seq0 = 0;
  bool open = false, eos = false;
  int64_t open_at = 0;
  for (int page = 0;; ++page) {
    if (pos + 27 > n || memcmp(b + pos, "OggS", 4) != 0) {
      if (page == 0) return w;
      break;
    }
    const uint8_t* h = b + pos;
    const int nseg = h[26];
    if (pos + 27 + nseg > n) break;
    int64_t body = 0;
    for (int s = 0; s < nseg; ++s) body += h[27 + s];
    if (pos + 27 + nseg + body > n) break;  // a file cut inside this page
    const bool in_headers = w.packets.size() < 3;
    bool bad = false;
    if (page == 0) {
      serial = le32(h + 14);
      seq0 = le32(h + 18);
    } else if (le32(h + 14) != serial) {
      return w;  // a second logical stream: multiplexed or chained
    }
    if (h[4] != 0 || (page > 0 && (h[5] & 2)) || eos) return w;  // another version, or a stream after the last page
    eos = (h[5] & 4) != 0;
    if (in_headers || check_audio) {
      uint32_t crc = 0;
      for (int64_t i = 0; i < 27 + nseg + body; ++i) {
        const uint8_t v = (i >= 22 && i < 26) ? 0 : h[i];
        crc = (crc << 8) ^ crc_t[((crc >> 24) ^ v) & 0xFF];
      }
      bad = bad || crc != le32(h + 22) || le32(h + 18) != seq0 + static_cast<uint32_t>(page);
    }
    if (((h[5] & 1) != 0) != open) bad = true;  // a continued page without an open packet, or the reverse
    if (bad) {
      if (in_headers) return w;
      w.audio_bad = true;
    }
    w.granule.push_back(static_cast<int64_t>(le32(h + 6)) | (static_cast<int64_t>(le32(h + 10)) << 32));
    int64_t at = pos + 27 + nseg;
    if (!(h[5] & 1)) open_at = static_cast<int64_t>(w.data.size());  // a packet left open before is dropped
    for (int s = 0; s < nseg; ++s) {
      const int lace = h[27 + s];
      w.data.insert(w.data.end(), b + at, b + at + lace);
      at += lace;
      if (lace < 255) {
        w.packets.push_back({open_at, static_cast<int64_t>(w.data.size()) - open_at, page});
        open_at = static_cast<int64_t>(w.data.size());
        open = false;
      } else {
        open = true;
      }
    }
    pos = at;
  }
  if (open) w.data.resize(static_cast<size_t>(open_at));  // a packet not completed by the last whole page
  w.rc = BT_OK;
  return w;
}

// ---- header bits ------------------------------------------------------------------------------------------------------
struct Reader {
  vb::Bits b;
  Reader(const uint8_t* p, int64_t len) : b{p, 8 * len, 0, false} {}
  uint32_t operator()(int n) { return b.read(n); }
};

double float32_unpack(uint32_t x) {
  const double mantissa = static_cast<double>(x & 0x1FFFFF);
  const int exponent = static_cast<int>((x & 0x7FE00000u) >> 21);
  return std::ldexp((x & 0x80000000u) ? -mantissa : mantissa, exponent - 788);
}

// the largest r with r^dim <= entries
int64_t lookup1_values(int64_t entries, int64_t dim) {
  int64_t r = static_cast<int64_t>(std::floor(std::exp(std::log(static_cast<double>(entries)) / dim)));
  auto pw = [&](int64_t v) {  // v^dim, saturating above entries
    int64_t p = 1;
    for (int64_t i = 0; i < dim; ++i) {
      p *= v;
      if (p > entries) return entries + 1;
    }
    return p;
  };
  while (r > 0 && pw(r) > entries) --r;
  while (pw(r + 1) <= entries) ++r;
  return r;
}

struct Setup {
  int channels = 0, rate = 0, bs[2] = {0, 0};
  std::vector<uint32_t> words;  // the decode tables (vorbis.cuh)
};

// Codewords of the lengths (0: unused), the specification's assignment (each entry takes the lowest codeword of its
// length that no earlier one prefixes or is prefixed by): false for an over-full list.
bool codewords(const std::vector<int>& len, std::vector<uint32_t>* code) {
  uint32_t marker[33] = {0};
  code->assign(len.size(), 0);
  for (size_t i = 0; i < len.size(); ++i) {
    const int L = len[i];
    if (L <= 0) continue;
    uint32_t entry = marker[L];
    if (L < 32 && (entry >> L)) return false;
    (*code)[i] = entry;
    for (int j = L; j > 0; --j) {
      if (marker[j] & 1) {
        if (j == 1) marker[1]++;
        else marker[j] = marker[j - 1] << 1;
        break;
      }
      marker[j]++;
    }
    for (int j = L + 1; j < 33; ++j) {
      if ((marker[j] >> 1) == entry) {
        entry = marker[j];
        marker[j] = marker[j - 1] << 1;
      } else {
        break;
      }
    }
  }
  return true;
}

// The setup of a stream from its three header packets, or BT_ERR_FORMAT.
int parse_setup(const uint8_t* id, int64_t id_len, const uint8_t* cm, int64_t cm_len, const uint8_t* su, int64_t su_len,
                Setup* S) {
  if (id_len < 30 || id[0] != 1 || memcmp(id + 1, "vorbis", 6) != 0) return BT_ERR_FORMAT;
  if (le32(id + 7) != 0) return BT_ERR_FORMAT;
  S->channels = id[11];
  S->rate = static_cast<int>(le32(id + 12));
  S->bs[0] = id[28] & 15;
  S->bs[1] = id[28] >> 4;
  if (S->channels < 1 || S->channels > vb::kMaxChannels || S->rate <= 0 || le32(id + 12) > 0x7FFFFFFFu ||
      S->bs[0] < vb::kMinLog2 || S->bs[1] > vb::kMaxLog2 || S->bs[0] > S->bs[1] || !(id[29] & 1))
    return BT_ERR_FORMAT;
  S->bs[0] = 1 << S->bs[0];
  S->bs[1] = 1 << S->bs[1];
  if (cm_len < 7 || cm[0] != 3 || memcmp(cm + 1, "vorbis", 6) != 0) return BT_ERR_FORMAT;
  if (su_len < 7 || su[0] != 5 || memcmp(su + 1, "vorbis", 6) != 0) return BT_ERR_FORMAT;
  Reader r(su + 7, su_len - 7);
  const int ch = S->channels;
  std::vector<uint32_t>& W = S->words;
  auto alloc = [&](int64_t words) -> int64_t {
    const int64_t at = static_cast<int64_t>(W.size());
    if (at + words > vb::kMaxTableWords) return -1;
    W.resize(static_cast<size_t>(at + words), 0);
    return at;
  };
  const int64_t words_T = (sizeof(vb::Tables) + 3) / 4;
  alloc(words_T);
  vb::Tables T{};
  T.channels = ch;
  T.blocksize[0] = S->bs[0];
  T.blocksize[1] = S->bs[1];
  // codebooks
  T.n_codebooks = static_cast<int32_t>(r(8)) + 1;
  const int64_t cb_at = alloc(T.n_codebooks * static_cast<int64_t>(sizeof(vb::Codebook) / 4));
  T.codebooks = static_cast<int32_t>(cb_at);
  std::vector<vb::Codebook> books(T.n_codebooks);
  for (int i = 0; i < T.n_codebooks; ++i) {
    if (r(24) != 0x564342 || r.b.eop) return BT_ERR_FORMAT;
    vb::Codebook& cb = books[i];
    cb.dimensions = static_cast<int32_t>(r(16));
    cb.entries = static_cast<int32_t>(r(24));
    if (cb.dimensions == 0 || cb.entries == 0 || r.b.eop) return BT_ERR_FORMAT;
    std::vector<int> len(cb.entries, 0);
    if (!r(1)) {
      const bool sparse = r(1);
      for (int e = 0; e < cb.entries && !r.b.eop; ++e)
        if (!sparse || r(1)) len[e] = static_cast<int>(r(5)) + 1;
    } else {
      int e = 0, L = static_cast<int>(r(5)) + 1;
      while (e < cb.entries && !r.b.eop) {
        const int64_t num = r(vb::ilog(static_cast<uint32_t>(cb.entries - e)));
        if (e + num > cb.entries || L > 32) return BT_ERR_FORMAT;
        for (int64_t k = 0; k < num; ++k) len[e + k] = L;
        e += static_cast<int>(num);
        ++L;
      }
    }
    if (r.b.eop) return BT_ERR_FORMAT;
    std::vector<uint32_t> code;
    if (!codewords(len, &code)) return BT_ERR_FORMAT;
    cb.used = 0;
    for (int e = 0; e < cb.entries; ++e) cb.used += len[e] > 0;
    // the decode tree: node k's children at words [tree + 2k, tree + 2k + 2), 0 absent, kLeaf | entry, or a node
    std::vector<uint32_t> tree(2, 0);
    for (int e = 0; e < cb.entries; ++e) {
      if (len[e] == 0) continue;
      uint32_t node = 0;
      for (int d = len[e] - 1; d >= 0; --d) {
        const size_t at = 2 * node + ((code[e] >> d) & 1);
        if (d == 0) {
          tree[at] = vb::kLeaf | static_cast<uint32_t>(e);
        } else {
          if (tree[at] == 0) {
            tree[at] = static_cast<uint32_t>(tree.size() / 2);
            tree.resize(tree.size() + 2, 0);
          }
          node = tree[at];
        }
      }
    }
    const int64_t tree_at = alloc(static_cast<int64_t>(tree.size()));
    if (tree_at < 0) return BT_ERR_FORMAT;
    std::copy(tree.begin(), tree.end(), W.begin() + tree_at);
    cb.tree = static_cast<int32_t>(tree_at);
    cb.lookup = static_cast<int32_t>(r(4));
    cb.vq = 0;
    if (cb.lookup == 1 || cb.lookup == 2) {
      const double mn = float32_unpack(r(32)), delta = float32_unpack(r(32));
      const int vbits = static_cast<int>(r(4)) + 1;
      const bool seq = r(1);
      const int64_t nv = cb.lookup == 1 ? lookup1_values(cb.entries, cb.dimensions)
                                        : static_cast<int64_t>(cb.entries) * cb.dimensions;
      if (nv <= 0 || nv > vb::kMaxTableWords) return BT_ERR_FORMAT;
      std::vector<uint32_t> mult(static_cast<size_t>(nv));
      for (int64_t k = 0; k < nv && !r.b.eop; ++k) mult[k] = r(vbits);
      if (r.b.eop) return BT_ERR_FORMAT;
      const int64_t vq_at = alloc(static_cast<int64_t>(cb.entries) * cb.dimensions);
      if (vq_at < 0) return BT_ERR_FORMAT;
      cb.vq = static_cast<int32_t>(vq_at);
      for (int64_t e = 0; e < cb.entries; ++e) {
        double last = 0;
        int64_t div = 1;
        for (int j = 0; j < cb.dimensions; ++j) {
          const int64_t off = cb.lookup == 1 ? (e / div) % nv : e * cb.dimensions + j;
          const double v = mult[off] * delta + mn + last;
          if (seq) last = v;
          const float f = static_cast<float>(v);
          memcpy(&W[vq_at + e * cb.dimensions + j], &f, 4);
          if (cb.lookup == 1) div *= nv;
          if (div > cb.entries) div = cb.entries + 1;  // keeps (e / div) at 0 without overflowing
        }
      }
    } else if (cb.lookup != 0) {
      return BT_ERR_FORMAT;
    }
  }
  // time-domain transforms: placeholders that must be zero
  const int n_time = static_cast<int>(r(6)) + 1;
  for (int i = 0; i < n_time; ++i)
    if (r(16) != 0) return BT_ERR_FORMAT;
  // floors
  T.n_floors = static_cast<int32_t>(r(6)) + 1;
  const int64_t fl_at = alloc(T.n_floors * static_cast<int64_t>(sizeof(vb::Floor1) / 4));
  if (fl_at < 0) return BT_ERR_FORMAT;
  T.floors = static_cast<int32_t>(fl_at);
  std::vector<vb::Floor1> floors(T.n_floors);
  for (auto& f : floors) {
    if (r(16) != 1) return BT_ERR_FORMAT;  // floor 0 is not decoded; other types do not exist
    f.partitions = static_cast<int32_t>(r(5));
    int max_class = -1;
    for (int i = 0; i < f.partitions; ++i) {
      f.partition_class[i] = static_cast<int32_t>(r(4));
      max_class = std::max(max_class, f.partition_class[i]);
    }
    f.classes = max_class + 1;
    for (int c = 0; c < f.classes; ++c) {
      f.class_dim[c] = static_cast<int32_t>(r(3)) + 1;
      f.class_sub[c] = static_cast<int32_t>(r(2));
      f.class_master[c] = 0;
      if (f.class_sub[c]) {
        f.class_master[c] = static_cast<int32_t>(r(8));
        if (f.class_master[c] >= T.n_codebooks) return BT_ERR_FORMAT;
      }
      for (int j = 0; j < 8; ++j) f.sub_book[c][j] = -1;
      for (int j = 0; j < (1 << f.class_sub[c]); ++j) {
        f.sub_book[c][j] = static_cast<int32_t>(r(8)) - 1;
        if (f.sub_book[c][j] >= T.n_codebooks) return BT_ERR_FORMAT;
      }
    }
    f.multiplier = static_cast<int32_t>(r(2)) + 1;
    const int rb = static_cast<int>(r(4));
    f.x[0] = 0;
    f.x[1] = 1 << rb;
    f.values = 2;
    for (int i = 0; i < f.partitions; ++i)
      for (int j = 0; j < f.class_dim[f.partition_class[i]]; ++j) {
        if (f.values >= vb::kMaxPosts) return BT_ERR_FORMAT;
        f.x[f.values++] = static_cast<int32_t>(r(rb));
      }
    if (r.b.eop) return BT_ERR_FORMAT;
    for (int i = 0; i < f.values; ++i) {
      f.sorted[i] = i;
      for (int j = 0; j < i; ++j)
        if (f.x[j] == f.x[i]) return BT_ERR_FORMAT;  // X values are unique
    }
    std::stable_sort(f.sorted, f.sorted + f.values, [&](int a, int b) { return f.x[a] < f.x[b]; });
    for (int i = 2; i < f.values; ++i) {
      int lo = 0, hi = 1;
      for (int j = 0; j < i; ++j) {
        if (f.x[j] < f.x[i] && f.x[j] > f.x[lo]) lo = j;
        if (f.x[j] > f.x[i] && f.x[j] < f.x[hi]) hi = j;
      }
      f.low[i] = lo;
      f.high[i] = hi;
    }
  }
  // residues
  T.n_residues = static_cast<int32_t>(r(6)) + 1;
  const int64_t re_at = alloc(T.n_residues * static_cast<int64_t>(sizeof(vb::Residue) / 4));
  if (re_at < 0) return BT_ERR_FORMAT;
  T.residues = static_cast<int32_t>(re_at);
  std::vector<vb::Residue> residues(T.n_residues);
  for (auto& q : residues) {
    q.type = static_cast<int32_t>(r(16));
    if (q.type > 2) return BT_ERR_FORMAT;
    q.begin = static_cast<int32_t>(r(24));
    q.end = static_cast<int32_t>(r(24));
    q.partition_size = static_cast<int32_t>(r(24)) + 1;
    q.classifications = static_cast<int32_t>(r(6)) + 1;
    q.classbook = static_cast<int32_t>(r(8));
    if (q.classbook >= T.n_codebooks || q.end < q.begin) return BT_ERR_FORMAT;
    int cascade[64];
    for (int c = 0; c < q.classifications; ++c) {
      cascade[c] = static_cast<int>(r(3));
      if (r(1)) cascade[c] |= static_cast<int>(r(5)) << 3;
    }
    for (int c = 0; c < 64; ++c)
      for (int p = 0; p < 8; ++p) q.books[c][p] = -1;
    for (int c = 0; c < q.classifications; ++c)
      for (int p = 0; p < 8; ++p)
        if (cascade[c] >> p & 1) {
          const int bk = static_cast<int>(r(8));
          if (bk >= T.n_codebooks || books[bk].lookup == 0 || q.partition_size % books[bk].dimensions != 0)
            return BT_ERR_FORMAT;  // residue books are VQ books whose vectors tile a partition
          q.books[c][p] = bk;
        }
  }
  // mappings
  T.n_mappings = static_cast<int32_t>(r(6)) + 1;
  const int64_t ma_at = alloc(T.n_mappings * static_cast<int64_t>(sizeof(vb::Mapping) / 4));
  if (ma_at < 0) return BT_ERR_FORMAT;
  T.mappings = static_cast<int32_t>(ma_at);
  std::vector<vb::Mapping> maps(T.n_mappings);
  for (auto& m : maps) {
    if (r(16) != 0) return BT_ERR_FORMAT;
    m.submaps = r(1) ? static_cast<int32_t>(r(4)) + 1 : 1;
    m.coupling_steps = r(1) ? static_cast<int32_t>(r(8)) + 1 : 0;
    const int cb = vb::ilog(static_cast<uint32_t>(ch - 1));
    for (int s = 0; s < m.coupling_steps; ++s) {
      m.magnitude[s] = static_cast<int32_t>(r(cb));
      m.angle[s] = static_cast<int32_t>(r(cb));
      if (m.magnitude[s] == m.angle[s] || m.magnitude[s] >= ch || m.angle[s] >= ch) return BT_ERR_FORMAT;
    }
    if (r(2) != 0) return BT_ERR_FORMAT;
    for (int c = 0; c < vb::kMaxChannels; ++c) m.mux[c] = 0;
    if (m.submaps > 1)
      for (int c = 0; c < ch; ++c) {
        m.mux[c] = static_cast<int32_t>(r(4));
        if (m.mux[c] >= m.submaps) return BT_ERR_FORMAT;
      }
    for (int s = 0; s < m.submaps; ++s) {
      r(8);
      m.submap_floor[s] = static_cast<int32_t>(r(8));
      m.submap_residue[s] = static_cast<int32_t>(r(8));
      if (m.submap_floor[s] >= T.n_floors || m.submap_residue[s] >= T.n_residues) return BT_ERR_FORMAT;
    }
  }
  // modes
  T.n_modes = static_cast<int32_t>(r(6)) + 1;
  const int64_t mo_at = alloc(T.n_modes * static_cast<int64_t>(sizeof(vb::Mode) / 4));
  if (mo_at < 0) return BT_ERR_FORMAT;
  T.modes = static_cast<int32_t>(mo_at);
  std::vector<vb::Mode> modes(T.n_modes);
  for (auto& m : modes) {
    m.blockflag = static_cast<int32_t>(r(1));
    if (r(16) != 0 || r(16) != 0) return BT_ERR_FORMAT;
    m.mapping = static_cast<int32_t>(r(8));
    if (m.mapping >= T.n_mappings) return BT_ERR_FORMAT;
  }
  if (r(1) != 1 || r.b.eop) return BT_ERR_FORMAT;
  T.mode_bits = vb::ilog(static_cast<uint32_t>(T.n_modes - 1));
  T.words = static_cast<int32_t>(W.size());
  memcpy(W.data(), &T, sizeof(T));
  memcpy(W.data() + T.codebooks, books.data(), books.size() * sizeof(vb::Codebook));
  memcpy(W.data() + T.floors, floors.data(), floors.size() * sizeof(vb::Floor1));
  memcpy(W.data() + T.residues, residues.data(), residues.size() * sizeof(vb::Residue));
  memcpy(W.data() + T.mappings, maps.data(), maps.size() * sizeof(vb::Mapping));
  memcpy(W.data() + T.modes, modes.data(), modes.size() * sizeof(vb::Mode));
  return BT_OK;
}

// ---- the audio packets ------------------------------------------------------------------------------------------------
struct Stream {
  int rc = BT_ERR_FORMAT;
  bool audio_bad = false;
  Setup setup;
  Walk w;
  std::vector<bt_vorbis_packet> table;
  int64_t packet_bytes = 0, block_samples = 0, skip = 0, n_samples = 0;
};

// The whole file: pages, headers, and the packet table (offsets into w.data until staging packs them).  An audio
// packet that is empty, not an audio packet or too short to hold its mode and window flags is dropped (the
// specification's decoder ignores it).
Stream read_stream(const uint8_t* b, int64_t n, bool check_audio) {
  Stream s;
  s.w = walk_pages(b, n, check_audio);
  if (s.w.rc != BT_OK || s.w.packets.size() < 3) return s;
  const Walk& w = s.w;
  const uint8_t* d = w.data.data();
  if (parse_setup(d + w.packets[0].off, w.packets[0].len, d + w.packets[1].off, w.packets[1].len,
                  d + w.packets[2].off, w.packets[2].len, &s.setup) != BT_OK)
    return s;
  const vb::Tables& T = *reinterpret_cast<const vb::Tables*>(s.setup.words.data());
  const vb::Mode* modes = vb::rec<vb::Mode>(s.setup.words.data(), T.modes, 0);
  std::vector<int> page_of;
  int64_t end = 0, prev_n = 0;
  for (size_t k = 3; k < w.packets.size(); ++k) {
    const Packet& p = w.packets[k];
    if (p.len == 0) continue;
    vb::Bits bits{d + p.off, 8 * p.len, 0, false};
    if (bits.read(1) != 0) continue;
    bt_vorbis_packet e{};
    e.mode = static_cast<uint8_t>(bits.read(T.mode_bits));
    if (e.mode < T.n_modes && modes[e.mode].blockflag) {
      e.blockflag = 1;
      e.prev_long = static_cast<uint8_t>(bits.read(1));
      e.next_long = static_cast<uint8_t>(bits.read(1));
    }
    if (bits.eop) continue;
    const int64_t bn = T.blocksize[e.blockflag];
    e.byte_offset = p.off;
    e.bytes = static_cast<int32_t>(p.len);
    e.block_offset = s.block_samples;
    end += s.table.empty() ? 0 : prev_n / 4 + bn / 4;
    e.end_sample = end;
    s.table.push_back(e);
    page_of.push_back(p.page);
    s.block_samples += bn;
    s.packet_bytes += p.len;
    prev_n = bn;
  }
  // trims by the granule positions: the first audio page's gives the granule of decoded sample 0, the last page's
  // the end of the output
  int64_t base = 0, g_end = -1;
  bool first = true;
  for (size_t k = 0; k < s.table.size(); ++k) {
    const int pg = page_of[k];
    if (k + 1 < s.table.size() && page_of[k + 1] == pg) continue;  // not the last packet completed on its page
    const int64_t g = w.granule[pg];
    if (g == -1) continue;
    if (first) base = g - s.table[k].end_sample;
    first = false;
    g_end = g;
  }
  s.skip = std::max<int64_t>(0, -base);
  const int64_t total = s.table.empty() ? 0 : s.table.back().end_sample;
  const int64_t stop = g_end < 0 ? total : std::min(total, g_end - base);
  s.n_samples = std::max<int64_t>(0, stop - s.skip);
  s.audio_bad = w.audio_bad;
  s.rc = BT_OK;
  return s;
}

void fill_info(const Stream& s, bt_vorbis_info* info) {
  info->sample_rate = s.setup.rate;
  info->channels = s.setup.channels;
  info->blocksize0 = s.setup.bs[0];
  info->blocksize1 = s.setup.bs[1];
  info->n_packets = static_cast<int64_t>(s.table.size());
  info->packet_bytes = s.packet_bytes;
  info->table_bytes = 4 * static_cast<int64_t>(s.setup.words.size());
  info->skip = s.skip;
  info->n_samples = s.n_samples;
}

int check_streams(const bt_vorbis_stream* s, int32_t n) {
  for (int32_t i = 0; i < n; ++i)
    if (s[i].byte_offset < 0 || s[i].byte_count < 0 || s[i].table_offset < 0 || s[i].table_offset % 4 != 0 ||
        s[i].table_bytes < 0 || s[i].packet_offset < 0 || s[i].n_packets < 0 || s[i].block_samples < 0 ||
        s[i].skip < 0 || s[i].n_samples < 0 || s[i].out_offset < 0 || s[i].channels < 1 ||
        s[i].channels > vb::kMaxChannels || s[i].sample_rate <= 0)
      return 1;
  return 0;
}

// The signal tables of every block size and the floor1 inverse dB table (vorbis.cuh), computed once in float64.
const std::vector<float>& signal_tables() {
  static const std::vector<float> t = [] {
    std::vector<float> v(vb::kSignalFloats);
    const double pi = 3.14159265358979323846;
    for (int b = vb::kMinLog2; b <= vb::kMaxLog2; ++b) {
      const int n = 1 << b, M = n / 2, H = n / 4;
      float* s = v.data() + 2 * vb::signal_at(b);
      for (int k = 0; k < H; ++k) {
        const double a = -pi * (k + 0.25) / M, c = -pi * k / M;
        s[2 * k] = static_cast<float>(std::cos(a));
        s[2 * k + 1] = static_cast<float>(std::sin(a));
        s[2 * (H + k)] = static_cast<float>(std::cos(c));
        s[2 * (H + k) + 1] = static_cast<float>(std::sin(c));
      }
      for (int m = 0; m < H / 2; ++m) {
        const double a = -2 * pi * m / H;
        s[2 * (2 * H + m)] = static_cast<float>(std::cos(a));
        s[2 * (2 * H + m) + 1] = static_cast<float>(std::sin(a));
      }
      float* slope = s + 2 * (2 * H + H / 2);
      for (int i = 0; i < M; ++i) {
        const double x = std::sin((i + 0.5) / M * pi / 2);
        slope[i] = static_cast<float>(std::sin(pi / 2 * x * x));
      }
    }
    for (int i = 0; i < 256; ++i) v[2 * vb::kDbAt + i] = static_cast<float>(std::pow(10.0, 7.0 * (i - 255) / 256.0));
    return v;
  }();
  return t;
}

}  // namespace

extern "C" {

int bt_vorbis_probe(const char* path, bt_vorbis_info* info) {
  if (!path || !info) return BT_ERR_ARG;
  memset(info, 0, sizeof(*info));
  std::vector<uint8_t> b;
  if (!bt::read_whole_file(path, &b)) return BT_ERR_IO;
  const Stream s = read_stream(b.data(), static_cast<int64_t>(b.size()), false);
  if (s.rc != BT_OK) return s.rc;
  fill_info(s, info);
  return BT_OK;
}

int bt_stage_vorbis_files(const char* const* paths, const bt_vorbis_info* infos, int32_t n_files, uint8_t* bytes_dst,
                          const int64_t* byte_offsets, bt_vorbis_packet* packets_dst, const int64_t* packet_offsets,
                          int64_t* packet_bytes, int64_t* n_packets, int64_t* block_samples, int32_t n_threads,
                          int32_t* status) {
  if (n_files <= 0) return BT_OK;
  if (!paths || !infos || !bytes_dst || !byte_offsets || !packets_dst || !packet_offsets || !packet_bytes ||
      !n_packets || !block_samples)
    return BT_ERR_ARG;
  std::atomic<int> failed{0};
  bt::run_pool(static_cast<size_t>(n_files), n_threads, [&](size_t i) {
    const bt_vorbis_info& in = infos[i];
    n_packets[i] = packet_bytes[i] = block_samples[i] = 0;
    int rc = BT_ERR_IO;
    std::vector<uint8_t> b;
    if (bt::read_whole_file(paths[i], &b)) {
      const Stream s = read_stream(b.data(), static_cast<int64_t>(b.size()), true);
      const int64_t N = static_cast<int64_t>(s.table.size());
      if (s.rc == BT_OK && !s.audio_bad && N <= in.n_packets && s.packet_bytes <= in.packet_bytes &&
          4 * static_cast<int64_t>(s.setup.words.size()) == in.table_bytes && s.setup.channels == in.channels &&
          s.setup.rate == in.sample_rate && s.skip == in.skip && s.n_samples == in.n_samples) {
        uint8_t* dst = bytes_dst + byte_offsets[i];
        bt_vorbis_packet* pk = packets_dst + packet_offsets[i];
        int64_t at = 0;
        for (int64_t k = 0; k < N; ++k) {
          bt_vorbis_packet e = s.table[k];
          memcpy(dst + at, s.w.data.data() + e.byte_offset, static_cast<size_t>(e.bytes));
          e.byte_offset = at;
          at += e.bytes;
          pk[k] = e;
        }
        memcpy(dst + (in.packet_bytes + 3) / 4 * 4, s.setup.words.data(), static_cast<size_t>(in.table_bytes));
        n_packets[i] = N;
        packet_bytes[i] = at;
        block_samples[i] = s.block_samples;
        rc = BT_OK;
      }
    }
    if (rc != BT_OK) failed.fetch_add(1);
    if (status) status[i] = rc;
  });
  return failed.load() ? BT_ERR_IO : BT_OK;
}

int bt_vorbis_decode(bt_ctx* c, const uint8_t* bytes_dev, const bt_vorbis_packet* packets_dev,
                     const bt_vorbis_stream* streams_host, int32_t n_streams, int32_t mode, void* out_dev,
                     int32_t* status_dev, void* stream) {
  static const char* fn = "bt_vorbis_decode";
  if (!c) return BT_ERR_ARG;
  if (n_streams < 0 || n_streams > 65535) return fail(c, BT_ERR_ARG, "%s: need 0 <= n_streams <= 65535", fn);
  if (mode != BT_VORBIS_MONO_F32 && mode != BT_VORBIS_CHANNELS_F64)
    return fail(c, BT_ERR_ARG, "%s: unknown mode %d", fn, mode);
  if (n_streams == 0) return BT_OK;
  if (!bytes_dev || !packets_dev || !streams_host || !out_dev || !status_dev)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  if (check_streams(streams_host, n_streams))
    return fail(c, BT_ERR_ARG, "%s: a stream has a negative count or offset, a table offset that is not a multiple of 4, "
                "channels outside 1..8 or a sample rate <= 0", fn);
  int64_t spec = 0, cls = 0, floors = 0, max_packets = 0, max_out = 0;
  for (int32_t i = 0; i < n_streams; ++i) {
    const bt_vorbis_stream& s = streams_host[i];
    spec += s.channels * s.block_samples;
    cls += s.channels * s.block_samples / 2;
    floors += s.channels * s.n_packets * vb::kFloorWords;
    max_packets = std::max(max_packets, s.n_packets);
    if (s.n_samples > 0) max_out = std::max(max_out, s.n_samples);
  }
  cudaStream_t st;
  int r = enter(c, fn, stream, &st);
  if (r != BT_OK) return r;
  const size_t bytes = 4 * static_cast<size_t>(spec + floors) + static_cast<size_t>(cls) + 16;
  BT_CUDA(c, c->vorbis_ws.reserve(bytes, bytes + bytes / 4));
  std::vector<vb::StreamDev> sd(n_streams);
  float* sp = reinterpret_cast<float*>(c->vorbis_ws.get());
  int32_t* fl = reinterpret_cast<int32_t*>(sp + spec);
  uint8_t* cl = reinterpret_cast<uint8_t*>(fl + floors);
  for (int32_t i = 0; i < n_streams; ++i) {
    const bt_vorbis_stream& s = streams_host[i];
    sd[i] = vb::StreamDev{bytes_dev + s.byte_offset, reinterpret_cast<const uint32_t*>(bytes_dev + s.table_offset),
                            packets_dev + s.packet_offset, sp, fl, cl, s.byte_count, s.table_bytes / 4, s.n_packets,
                            s.block_samples, s.skip, s.n_samples, s.out_offset, s.channels};
    sp += s.channels * s.block_samples;
    cl += s.channels * s.block_samples / 2;
    fl += s.channels * s.n_packets * vb::kFloorWords;
  }
  const vb::StreamDev* d[1];
  if ((r = stage(c, st, {{sd.data(), sd.size()}}, d)) != BT_OK) return r;
  const std::vector<float>& tt = signal_tables();
  const float* dt[1];
  if ((r = stage(c, st, {{tt.data(), tt.size()}}, dt)) != BT_OK) return r;
  if (max_packets > 0) {
    launch_vorbis_packets(d[0], n_streams, max_packets, status_dev, st);
    BT_LAUNCHED(c, "vorbis_packets", st);
    launch_vorbis_blocks(d[0], n_streams, max_packets, dt[0], status_dev, st);
    BT_LAUNCHED(c, "vorbis_blocks", st);
  }
  if (max_out > 0) {  // also for streams that are not decoded: their output is zero-filled
    launch_vorbis_output(d[0], n_streams, max_out, mode, out_dev, status_dev, st);
    BT_LAUNCHED(c, "vorbis_output", st);
  }
  return BT_OK;
}

int bt_debug_vorbis_decode_host(const uint8_t* bytes_host, const bt_vorbis_packet* packets_host,
                                const bt_vorbis_stream* streams_host, int32_t n_streams, int32_t mode, void* out_host,
                                int32_t* status_host) {
  if (n_streams < 0) return BT_ERR_ARG;
  if (n_streams == 0) return BT_OK;
  if (!bytes_host || !packets_host || !streams_host || !out_host || !status_host ||
      check_streams(streams_host, n_streams) || (mode != BT_VORBIS_MONO_F32 && mode != BT_VORBIS_CHANNELS_F64))
    return BT_ERR_ARG;
  const std::vector<float>& tt = signal_tables();
  for (int32_t si = 0; si < n_streams; ++si) {
    const bt_vorbis_stream& s = streams_host[si];
    const int nch = s.channels;
    std::vector<float> spec(static_cast<size_t>(nch * s.block_samples));
    std::vector<int32_t> fl(static_cast<size_t>(nch * s.n_packets * vb::kFloorWords));
    std::vector<uint8_t> cl(static_cast<size_t>(nch * s.block_samples / 2 + 1));
    vb::StreamDev sd{bytes_host + s.byte_offset, reinterpret_cast<const uint32_t*>(bytes_host + s.table_offset),
                       packets_host + s.packet_offset, spec.data(), fl.data(), cl.data(), s.byte_count,
                       s.table_bytes / 4, s.n_packets, s.block_samples, s.skip, s.n_samples, s.out_offset, nch};
    if (status_host[si] == BT_OK)
      for (int64_t p = 0; p < s.n_packets && status_host[si] == BT_OK; ++p)
        status_host[si] = vb::decode_packet(sd, p);
    if (status_host[si] == BT_OK) {
      vb::BlockShared sh;
      std::vector<float2> buf[2] = {std::vector<float2>(2048), std::vector<float2>(2048)};
      for (int64_t p = 0; p < s.n_packets; ++p) {
        const vb::BlockGeom g = vb::block_geom(sd, p);
        for (int c = 0; c < nch; ++c) vb::block_floor(sd, p, g, c, &sh);
        for (int i = 0; i < g.n / 2; ++i) vb::block_couple(sd, p, g, i);
        for (int c = 0; c < nch; ++c) {
          for (int k = 0; k < g.n / 4; ++k) vb::block_pre(sd, p, g, c, &sh, tt.data(), k, buf[0].data());
          int cur = 0;
          for (int Ns = 1; Ns < g.n / 4;) {
            const int R = vb::pass_radix(g.n / 4, Ns);
            for (int j = 0; j < g.n / 4 / R; ++j) vb::block_pass(buf[cur].data(), buf[cur ^ 1].data(), j, Ns, R, g, tt.data());
            cur ^= 1;
            Ns *= R;
          }
          float* u = reinterpret_cast<float*>(buf[cur ^ 1].data());
          for (int k = 0; k < g.n / 4; ++k) vb::post_twiddle(buf[cur].data(), vb::sig(tt.data(), g.n), g.n, k, u);
          for (int i = 0; i < g.n; ++i) vb::block_out(sd, p, g, c, &sh, tt.data(), u, i);
        }
      }
    }
    for (int64_t t = 0; t < s.n_samples; ++t) {
      const bool ok = status_host[si] == BT_OK && s.n_packets > 0;
      if (mode == BT_VORBIS_MONO_F32) {
        static_cast<float*>(out_host)[s.out_offset + t] = ok ? vb::output_mono(sd, t) : 0.f;
      } else {
        for (int c = 0; c < nch; ++c)
          static_cast<double*>(out_host)[s.out_offset + t * nch + c] = ok ? static_cast<double>(vb::output_sample(sd, t, c)) : 0.0;
      }
    }
  }
  return BT_OK;
}

}  // extern "C"
