// The host thread pool of the staging entry points (host_stage.cpp, api_flac.cu).
#pragma once
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

}  // namespace bt
