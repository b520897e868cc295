// C ABI (include/beatthis.h): native FLAC input -- bt_flac_probe and bt_stage_flac_files on the host,
// bt_flac_decode on the device (kernels_flac.cu), and the host test hook bt_debug_flac_decode_host.  The frame parsing
// and decoding are flac.cuh's, shared by all three.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <cstring>
#include <vector>

#include "api_internal.h"
#include "flac.cuh"
#include "host_pool.h"

namespace {

using bt::flac::Header;

bool read_all(int fd, uint8_t* dst, int64_t n, int64_t at) {
  int64_t got = 0;
  while (got < n) {
    const ssize_t r = pread(fd, dst + got, static_cast<size_t>(n - got), at + got);
    if (r <= 0) return false;
    got += r;
  }
  return true;
}

uint32_t be(const uint8_t* p, int n) {
  uint32_t v = 0;
  for (int k = 0; k < n; ++k) v = (v << 8) | p[k];
  return v;
}

// A header that may continue a stream: STREAMINFO's channels, bits, rate and block-size limit, the stream's blocking
// strategy and the expected frame or sample number.
bool continues(const Header& h, const bt_flac_info& in, int variable, int64_t number) {
  return h.variable == variable && h.number == number && h.channels == in.channels &&
         (h.bits == 0 || h.bits == in.bits_per_sample) && (h.sample_rate == 0 || h.sample_rate == in.sample_rate) &&
         h.block_size <= in.max_block;
}

// Frame table of one file's frame bytes b[0 .. n): BT_OK or BT_ERR_IO.
int scan_frames(const uint8_t* b, int64_t n, const bt_flac_info& in, bt_flac_frame* out, int64_t cap, int64_t* n_frames,
                int64_t* n_samples) {
  Header h;
  if (!bt::flac::parse_header(b, n, &h) || !continues(h, in, h.variable, 0)) return BT_ERR_IO;
  const int variable = h.variable;
  int64_t pos = 0, first = 0, count = 0;
  for (;;) {
    const int64_t next_number = variable ? first + h.block_size : h.number + 1;
    Header nh{};
    int64_t q = pos + h.length;
    bool found = false;
    while (q + 1 < n) {
      const void* ff = memchr(b + q, 0xFF, static_cast<size_t>(n - 1 - q));
      if (!ff) break;
      q = static_cast<const uint8_t*>(ff) - b;
      if (b[q + 1] == (0xF8 | variable) && bt::flac::parse_header(b + q, n - q, &nh) &&
          continues(nh, in, variable, next_number)) {
        found = true;
        break;
      }
      ++q;
    }
    const int64_t end = found ? q : n;
    if (count >= cap || end - pos > INT32_MAX) return BT_ERR_IO;
    out[count++] = bt_flac_frame{pos, first, static_cast<int32_t>(end - pos), h.block_size};
    first += h.block_size;
    if (!found) break;
    pos = q;
    h = nh;
  }
  if (in.total_samples > 0 && first != in.total_samples) return BT_ERR_IO;
  *n_frames = count;
  *n_samples = first;
  return BT_OK;
}

// Host tables of one bt_flac_decode call, checked.
int check_streams(const bt_flac_stream* s, int32_t n, int32_t mode) {
  if (mode != BT_FLAC_MONO_F32 && mode != BT_FLAC_CHANNELS_F64) return 1;
  for (int32_t i = 0; i < n; ++i)
    if (s[i].byte_offset < 0 || s[i].byte_count < 0 || s[i].frame_offset < 0 || s[i].n_frames < 0 ||
        s[i].n_samples < 0 || s[i].out_offset < 0 || s[i].channels < 1 || s[i].channels > 8 ||
        s[i].bits_per_sample < 4 || s[i].bits_per_sample > 32)
      return 2;
  return 0;
}

std::vector<uint16_t> crc16_table() {
  std::vector<uint16_t> t(256);
  for (int b = 0; b < 256; ++b) t[b] = bt::flac::crc16_byte_slow(0, static_cast<uint8_t>(b));
  return t;
}

}  // namespace

extern "C" {

int bt_flac_probe(const char* path, bt_flac_info* info) {
  if (!path || !info) return BT_ERR_ARG;
  memset(info, 0, sizeof(*info));
  const int fd = open(path, O_RDONLY);
  if (fd < 0) return BT_ERR_IO;
  struct stat sb;
  if (fstat(fd, &sb) != 0) { close(fd); return BT_ERR_IO; }
  const int64_t size = sb.st_size;
  int rc = BT_ERR_FORMAT;
  uint8_t h[10];
  int64_t pos = 0;
  if (size >= 10 && read_all(fd, h, 10, 0) && memcmp(h, "ID3", 3) == 0)  // ID3v2: 10 bytes, syncsafe size, footer
    pos = 10 + ((h[6] & 0x7F) << 21 | (h[7] & 0x7F) << 14 | (h[8] & 0x7F) << 7 | (h[9] & 0x7F)) + ((h[5] & 0x10) ? 10 : 0);
  uint8_t m[4];
  if (pos + 4 <= size && read_all(fd, m, 4, pos) && memcmp(m, "fLaC", 4) == 0) {
    pos += 4;
    bool first = true, done = false;
    while (!done && pos + 4 <= size) {
      uint8_t bh[4];
      if (!read_all(fd, bh, 4, pos)) break;
      const bool last = bh[0] & 0x80;
      const int type = bh[0] & 0x7F;
      const int64_t len = be(bh + 1, 3);
      if (type == 127 || (first != (type == 0)) || pos + 4 + len > size) break;
      if (type == 0) {
        uint8_t si[34];
        if (len != 34 || !read_all(fd, si, 34, pos + 4)) break;
        info->min_block = static_cast<int32_t>(be(si, 2));
        info->max_block = static_cast<int32_t>(be(si + 2, 2));
        info->sample_rate = static_cast<int32_t>(be(si + 10, 3) >> 4);
        info->channels = ((si[12] >> 1) & 7) + 1;
        info->bits_per_sample = (((si[12] & 1) << 4) | (si[13] >> 4)) + 1;
        info->total_samples = (static_cast<int64_t>(si[13] & 15) << 32) | be(si + 14, 4);
        memcpy(info->md5, si + 18, 16);
        if (info->bits_per_sample < 4 || info->max_block < 1 || info->sample_rate < 1) break;
      }
      first = false;
      done = last;
      pos += 4 + len;
    }
    if (done) {
      info->frames_offset = pos;
      info->frames_bytes = size - pos;
      info->max_frames = info->total_samples > 0
                             ? (info->total_samples + std::max(info->min_block, 16) - 1) / std::max(info->min_block, 16) + 1
                             : info->frames_bytes / 10 + 1;
      rc = BT_OK;
    }
  }
  close(fd);
  if (rc != BT_OK) {
    memset(info, 0, sizeof(*info));
  }
  return rc;
}

int bt_stage_flac_files(const char* const* paths, const bt_flac_info* infos, int32_t n_files, uint8_t* bytes_dst,
                        const int64_t* byte_offsets, bt_flac_frame* frames_dst, const int64_t* frame_offsets,
                        int64_t* n_frames, int64_t* n_samples, int32_t n_threads, int32_t* status) {
  if (n_files <= 0) return BT_OK;
  if (!paths || !infos || !bytes_dst || !byte_offsets || !frames_dst || !frame_offsets || !n_frames || !n_samples)
    return BT_ERR_ARG;
  std::atomic<int> failed{0};
  bt::run_pool(static_cast<size_t>(n_files), n_threads, [&](size_t i) {
    const bt_flac_info& in = infos[i];
    n_frames[i] = n_samples[i] = 0;
    int rc = BT_ERR_IO;
    const int fd = open(paths[i], O_RDONLY);
    if (fd >= 0) {
      uint8_t* b = bytes_dst + byte_offsets[i];
      if (in.frames_bytes > 0 && in.max_frames > 0 && read_all(fd, b, in.frames_bytes, in.frames_offset))
        rc = scan_frames(b, in.frames_bytes, in, frames_dst + frame_offsets[i], in.max_frames, &n_frames[i],
                         &n_samples[i]);
      close(fd);
    }
    if (rc != BT_OK) {
      n_frames[i] = n_samples[i] = 0;
      failed.fetch_add(1);
    }
    if (status) status[i] = rc;
  });
  return failed.load() ? BT_ERR_IO : BT_OK;
}

int bt_flac_decode(bt_ctx* c, const uint8_t* bytes_dev, const bt_flac_frame* frames_dev,
                   const bt_flac_stream* streams_host, int32_t n_streams, int32_t mode, void* out_dev,
                   int32_t* status_dev, void* stream) {
  static const char* fn = "bt_flac_decode";
  if (!c) return BT_ERR_ARG;
  if (n_streams < 0 || n_streams > 65535) return fail(c, BT_ERR_ARG, "%s: need 0 <= n_streams <= 65535", fn);
  if (mode != BT_FLAC_MONO_F32 && mode != BT_FLAC_CHANNELS_F64) return fail(c, BT_ERR_ARG, "%s: unknown mode %d", fn, mode);
  if (n_streams == 0) return BT_OK;
  if (!bytes_dev || !frames_dev || !streams_host || !out_dev || !status_dev)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  if (check_streams(streams_host, n_streams, mode))
    return fail(c, BT_ERR_ARG, "%s: a stream has a negative count or offset, or channels / bits outside 1..8 / 4..32", fn);
  int64_t scratch = 0, max_frames = 0, max_samples = 0;
  for (int32_t i = 0; i < n_streams; ++i) {
    scratch += streams_host[i].n_samples * streams_host[i].channels;
    max_frames = std::max(max_frames, streams_host[i].n_frames);
    max_samples = std::max(max_samples, streams_host[i].n_samples);
  }
  cudaStream_t st;
  int r = enter(c, fn, stream, &st);
  if (r != BT_OK) return r;
  const size_t bytes = sizeof(int64_t) * static_cast<size_t>(std::max<int64_t>(scratch, 1));
  BT_CUDA(c, c->flac_ws.reserve(bytes, bytes + bytes / 4));
  std::vector<FlacStreamDev> sd(n_streams);
  int64_t so = 0;
  for (int32_t i = 0; i < n_streams; ++i) {
    const bt_flac_stream& s = streams_host[i];
    sd[i] = FlacStreamDev{bytes_dev + s.byte_offset, frames_dev + s.frame_offset, c->flac_ws.get() + so, s.byte_count,
                          s.n_frames, s.n_samples, s.out_offset, s.channels, s.bits_per_sample};
    so += s.n_samples * s.channels;
  }
  const FlacStreamDev* d[1];
  if ((r = stage(c, st, {{sd.data(), sd.size()}}, d)) != BT_OK) return r;
  if (max_frames > 0) {
    launch_flac_frames(d[0], n_streams, max_frames, status_dev, st);
    BT_LAUNCHED(c, "flac_frames", st);
  }
  if (max_samples > 0) {
    launch_flac_output(d[0], n_streams, max_samples, mode, out_dev, status_dev, st);
    BT_LAUNCHED(c, "flac_output", st);
  }
  return BT_OK;
}

int bt_debug_flac_decode_host(const uint8_t* bytes_host, const bt_flac_frame* frames_host,
                              const bt_flac_stream* streams_host, int32_t n_streams, int32_t mode, void* out_host,
                              int32_t* status_host) {
  if (n_streams < 0) return BT_ERR_ARG;
  if (n_streams == 0) return BT_OK;
  if (!bytes_host || !frames_host || !streams_host || !out_host || !status_host ||
      check_streams(streams_host, n_streams, mode))
    return BT_ERR_ARG;
  const std::vector<uint16_t> crc16 = crc16_table();
  int32_t coef[32];
  for (int32_t i = 0; i < n_streams; ++i) {
    const bt_flac_stream& s = streams_host[i];
    std::vector<int64_t> x(static_cast<size_t>(s.n_samples * s.channels));
    for (int64_t k = 0; k < s.n_frames && status_host[i] == BT_OK; ++k) {
      const bt_flac_frame fr = frames_host[s.frame_offset + k];
      const bool ok = fr.offset >= 0 && fr.bytes > 0 && fr.offset <= s.byte_count - fr.bytes && fr.block_size >= 1 &&
                      fr.first_sample >= 0 && fr.first_sample <= s.n_samples - fr.block_size &&
                      bt::flac::decode_frame(bytes_host + s.byte_offset + fr.offset, fr.bytes, fr.block_size, s.channels,
                                             s.bits_per_sample, crc16.data(), x.data() + fr.first_sample, s.n_samples,
                                             coef, 1);
      if (!ok) status_host[i] = BT_ERR_IO;
    }
    const bool ok = status_host[i] == BT_OK;
    const double scale = bt::flac::scale_of(s.bits_per_sample);
    for (int64_t t = 0; t < s.n_samples; ++t) {
      if (mode == BT_FLAC_MONO_F32) {
        static_cast<float*>(out_host)[s.out_offset + t] =
            ok ? bt::flac::mono_sample(x.data() + t, s.n_samples, s.channels, scale) : 0.f;
      } else {
        for (int ch = 0; ch < s.channels; ++ch)
          static_cast<double*>(out_host)[s.out_offset + t * s.channels + ch] =
              ok ? static_cast<double>(x[ch * s.n_samples + t]) * scale : 0.0;
      }
    }
  }
  return BT_OK;
}

}  // extern "C"
