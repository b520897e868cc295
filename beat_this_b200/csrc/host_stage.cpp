// Host side of Audio2Frames.signal2spect (reference beat_this/inference.py:269-277) and of load_audio for RIFF/WAVE
// files (reference beat_this/preprocessing.py:6-24): channel mix in the reference's arithmetic + cast to fp32, many
// clips at once on a pool of host threads, written straight into ONE (pinned) buffer that is then copied to the device.
// No CUDA in this file; every function is thread-safe.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/beatthis.h"
#include "host_pool.h"

namespace {

struct Piece { int32_t clip; int64_t lo, hi; };  // frames [lo, hi) of one clip

std::vector<Piece> split_pieces(const int64_t* frames, int32_t n, int64_t grain) {
  std::vector<Piece> v;
  for (int32_t i = 0; i < n; ++i)
    for (int64_t lo = 0; lo < frames[i]; lo += grain) v.push_back({i, lo, std::min(frames[i], lo + grain)});
  return v;
}

using bt::run_pool;

// mean over channels exactly as numpy's signal.mean(1) computes it for `ch` < 8 channels (sequential sum in the
// array's own floating type, one division), then the fp32 cast of torch.tensor(signal, dtype=float32)
// (inference.py:270-271,276).
// Acc = the array's own type for ndarray input (numpy reduces float32 in float32), double for files (load_audio
// returns float64 whatever the file holds, preprocessing.py:6-10).
template <typename T, typename Acc>
inline void mix_float(const T* src, int32_t ch, int64_t lo, int64_t hi, float* dst) {
  if (ch == 1) {
    for (int64_t t = lo; t < hi; ++t) dst[t] = static_cast<float>(src[t]);
    return;
  }
  const Acc n = static_cast<Acc>(ch);
  for (int64_t t = lo; t < hi; ++t) {
    const T* f = src + t * ch;
    Acc acc = static_cast<Acc>(f[0]);
    for (int32_t c = 1; c < ch; ++c) acc += static_cast<Acc>(f[c]);
    dst[t] = static_cast<float>(acc / n);
  }
}

// integer PCM: value / 2^(bits-1) in float64 (what soundfile / torchaudio hand to load_audio), float64 channel mean
template <int BPS>
inline int32_t pcm_value(const uint8_t* s) {
  if constexpr (BPS == 1) return static_cast<int32_t>(s[0]) - 128;  // 8-bit WAV is unsigned
  else if constexpr (BPS == 2) return static_cast<int16_t>(s[0] | (s[1] << 8));
  else if constexpr (BPS == 3) return (static_cast<int32_t>(s[0] | (s[1] << 8) | (s[2] << 16)) << 8) >> 8;
  else return static_cast<int32_t>(static_cast<uint32_t>(s[0]) | (static_cast<uint32_t>(s[1]) << 8) |
                                   (static_cast<uint32_t>(s[2]) << 16) | (static_cast<uint32_t>(s[3]) << 24));
}
template <int BPS>
inline void mix_pcm_t(const uint8_t* src, int32_t ch, int64_t lo, int64_t hi, float* dst) {
  constexpr double scale = BPS == 1 ? 1.0 / 128.0 : BPS == 2 ? 1.0 / 32768.0 : BPS == 3 ? 1.0 / 8388608.0 : 1.0 / 2147483648.0;
  if (ch == 1) {  // value * 2^-k is exact in float64 and (for <= 24 bits) in float32: one multiply, one rounding
    for (int64_t t = lo; t < hi; ++t) dst[t] = static_cast<float>(static_cast<double>(pcm_value<BPS>(src + t * BPS)) * scale);
    return;
  }
  const int64_t stride = static_cast<int64_t>(BPS) * ch;
  const double n = static_cast<double>(ch);
  for (int64_t t = lo; t < hi; ++t) {
    const uint8_t* f = src + t * stride;
    double acc = static_cast<double>(pcm_value<BPS>(f)) * scale;
    for (int32_t c = 1; c < ch; ++c) acc += static_cast<double>(pcm_value<BPS>(f + c * BPS)) * scale;
    dst[t] = static_cast<float>(acc / n);
  }
}
inline void mix_pcm(const uint8_t* src, int32_t bytes_per_sample, int32_t ch, int64_t lo, int64_t hi, float* dst) {
  switch (bytes_per_sample) {
    case 1: mix_pcm_t<1>(src, ch, lo, hi, dst); break;
    case 2: mix_pcm_t<2>(src, ch, lo, hi, dst); break;
    case 3: mix_pcm_t<3>(src, ch, lo, hi, dst); break;
    default: mix_pcm_t<4>(src, ch, lo, hi, dst); break;
  }
}

uint32_t rd32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | (static_cast<uint32_t>(p[3]) << 24); }
uint16_t rd16(const uint8_t* p) { return static_cast<uint16_t>(p[0] | (p[1] << 8)); }

}  // namespace

extern "C" {

int bt_stage_audio(const void* const* signals, const int32_t* dtypes, const int64_t* frames, const int32_t* channels,
                   int32_t n_clips, float* dst, const int64_t* dst_offsets, int32_t n_threads) {
  if (n_clips <= 0) return BT_OK;
  if (!signals || !dtypes || !frames || !channels || !dst || !dst_offsets) return BT_ERR_ARG;
  for (int32_t i = 0; i < n_clips; ++i) {
    if (!signals[i] && frames[i] > 0) return BT_ERR_ARG;
    if (channels[i] < 1 || frames[i] < 0) return BT_ERR_ARG;
    if (dtypes[i] != BT_SIG_F32 && dtypes[i] != BT_SIG_F64 && dtypes[i] != BT_SIG_I16) return BT_ERR_ARG;
  }
  const std::vector<Piece> pieces = split_pieces(frames, n_clips, 1 << 17);
  run_pool(pieces.size(), n_threads, [&](size_t k) {
    const Piece& p = pieces[k];
    float* out = dst + dst_offsets[p.clip];
    const int32_t ch = channels[p.clip];
    switch (dtypes[p.clip]) {
      case BT_SIG_F32: mix_float<float, float>(static_cast<const float*>(signals[p.clip]), ch, p.lo, p.hi, out); break;
      case BT_SIG_F64: mix_float<double, double>(static_cast<const double*>(signals[p.clip]), ch, p.lo, p.hi, out); break;
      default: mix_pcm(static_cast<const uint8_t*>(signals[p.clip]), 2, ch, p.lo, p.hi, out); break;
    }
  });
  return BT_OK;
}

int bt_wav_probe(const char* path, bt_wav_info* info) {
  if (!path || !info) return BT_ERR_ARG;
  memset(info, 0, sizeof(*info));
  const int fd = open(path, O_RDONLY);
  if (fd < 0) return BT_ERR_IO;
  struct stat sb;
  if (fstat(fd, &sb) != 0) { close(fd); return BT_ERR_IO; }
  uint8_t hdr[12];
  if (pread(fd, hdr, 12, 0) != 12 || memcmp(hdr, "RIFF", 4) != 0 || memcmp(hdr + 8, "WAVE", 4) != 0) {
    close(fd);
    return BT_ERR_FORMAT;
  }
  int64_t pos = 12;
  bool have_fmt = false;
  int rc = BT_ERR_FORMAT;
  while (pos + 8 <= sb.st_size) {
    uint8_t ck[8];
    if (pread(fd, ck, 8, pos) != 8) break;
    const int64_t size = rd32(ck + 4);
    if (memcmp(ck, "fmt ", 4) == 0) {
      uint8_t f[40] = {0};
      const int64_t want = std::min<int64_t>(size, 40);
      if (want < 16 || pread(fd, f, want, pos + 8) != want) break;
      int32_t tag = rd16(f);
      info->channels = rd16(f + 2);
      info->sample_rate = static_cast<int32_t>(rd32(f + 4));
      const int32_t bits = rd16(f + 14);
      if (tag == 0xFFFE && want >= 26) tag = rd16(f + 24);  // WAVE_FORMAT_EXTENSIBLE: first two bytes of the sub-format GUID
      info->bytes_per_sample = bits / 8;
      info->is_float = tag == 3;
      const bool ok_int = tag == 1 && (bits == 8 || bits == 16 || bits == 24 || bits == 32);
      const bool ok_flt = tag == 3 && (bits == 32 || bits == 64);
      if (info->channels < 1 || !(ok_int || ok_flt)) break;
      have_fmt = true;
    } else if (memcmp(ck, "data", 4) == 0) {
      if (!have_fmt) break;
      int64_t bytes = size;
      if (pos + 8 + bytes > sb.st_size) bytes = sb.st_size - pos - 8;  // streamed files carry a bogus size
      info->data_offset = pos + 8;
      info->frames = bytes / (static_cast<int64_t>(info->bytes_per_sample) * info->channels);
      rc = BT_OK;
      break;
    }
    pos += 8 + size + (size & 1);
  }
  close(fd);
  return rc;
}

int bt_stage_wav_files(const char* const* paths, const bt_wav_info* infos, int32_t n_files, float* dst,
                       const int64_t* dst_offsets, int32_t n_threads, int32_t* status) {
  if (n_files <= 0) return BT_OK;
  if (!paths || !infos || !dst || !dst_offsets) return BT_ERR_ARG;
  std::vector<int64_t> frames(n_files);
  for (int32_t i = 0; i < n_files; ++i) frames[i] = infos[i].frames;
  const std::vector<Piece> pieces = split_pieces(frames.data(), n_files, 1 << 17);
  std::vector<int> fds(n_files, -1);
  std::atomic<int> failed{0};
  for (int32_t i = 0; i < n_files; ++i) {
    fds[i] = open(paths[i], O_RDONLY);
    if (status) status[i] = fds[i] < 0 ? BT_ERR_IO : BT_OK;
    if (fds[i] < 0) failed.fetch_add(1);
  }
  run_pool(pieces.size(), n_threads, [&](size_t k) {
    const Piece& p = pieces[k];
    const bt_wav_info& w = infos[p.clip];
    float* out = dst + dst_offsets[p.clip];
    if (fds[p.clip] < 0) {
      std::fill(out + p.lo, out + p.hi, 0.0f);
      return;
    }
    const int64_t stride = static_cast<int64_t>(w.bytes_per_sample) * w.channels;
    std::vector<uint8_t> buf(static_cast<size_t>((p.hi - p.lo) * stride));
    int64_t got = 0;
    while (got < static_cast<int64_t>(buf.size())) {
      const ssize_t r = pread(fds[p.clip], buf.data() + got, buf.size() - got, w.data_offset + p.lo * stride + got);
      if (r <= 0) break;
      got += r;
    }
    if (got < static_cast<int64_t>(buf.size())) {
      if (status) status[p.clip] = BT_ERR_IO;
      failed.fetch_add(1);
      std::fill(buf.begin() + got, buf.end(), 0);
    }
    // the piece was read to offset 0 of buf: shift the pointers so that frame t of the clip sits at index t
    if (w.is_float && w.bytes_per_sample == 4)
      mix_float<float, double>(reinterpret_cast<const float*>(buf.data()) - p.lo * w.channels, w.channels, p.lo, p.hi, out);
    else if (w.is_float)
      mix_float<double, double>(reinterpret_cast<const double*>(buf.data()) - p.lo * w.channels, w.channels, p.lo, p.hi, out);
    else
      mix_pcm(buf.data() - p.lo * stride, w.bytes_per_sample, w.channels, p.lo, p.hi, out);
  });
  for (int fd : fds)
    if (fd >= 0) close(fd);
  return failed.load() ? BT_ERR_IO : BT_OK;
}

}  // extern "C"
