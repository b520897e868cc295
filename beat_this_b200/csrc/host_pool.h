// The host thread pool of the staging entry points (host_stage.cpp, api_flac.cu, api_mp3.cu, api_vorbis.cu) and their
// whole-file reader.
#pragma once
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cstdint>
#include <algorithm>
#include <atomic>
#include <thread>
#include <vector>

namespace bt {

// fn(i) for i in [0, n_tasks) on n_threads threads (<= 0: one per hardware thread), the caller's thread among them
template <typename F>
void run_pool(size_t n_tasks, int n_threads, F&& fn) {
  if (n_threads <= 0) n_threads = static_cast<int>(std::thread::hardware_concurrency());
  n_threads = std::max(1, std::min<int>(n_threads, static_cast<int>(n_tasks)));
  std::atomic<size_t> next{0};
  auto worker = [&]() {
    for (;;) {
      const size_t i = next.fetch_add(1, std::memory_order_relaxed);
      if (i >= n_tasks) break;
      fn(i);
    }
  };
  if (n_threads == 1) { worker(); return; }
  std::vector<std::thread> th;
  th.reserve(n_threads - 1);
  for (int t = 1; t < n_threads; ++t) th.emplace_back(worker);
  worker();
  for (auto& t : th) t.join();
}

// The bytes of the file at path into *out; false when it cannot be opened or read.
inline bool read_whole_file(const char* path, std::vector<uint8_t>* out) {
  const int fd = open(path, O_RDONLY);
  if (fd < 0) return false;
  struct stat sb;
  bool ok = fstat(fd, &sb) == 0;
  if (ok) {
    out->resize(static_cast<size_t>(sb.st_size));
    int64_t got = 0;
    while (ok && got < sb.st_size) {
      const ssize_t r = pread(fd, out->data() + got, static_cast<size_t>(sb.st_size - got), got);
      ok = r > 0;
      got += r > 0 ? r : 0;
    }
  }
  close(fd);
  return ok;
}

}  // namespace bt
