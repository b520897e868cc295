// Bar-pointer model of the DBN post-processor (beat_this_b200/dbn.py::_BarModel), shared by the host tracker
// (dbn_host.cpp) and the device tracker (bt_dbn_track_device in api_post.cu, kernels in kernels_dbn.cu): both decode
// exactly the tables built here.  Host code only.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

namespace bt {

struct BarModel {
  int32_t beats = 0, n_int = 0;
  int64_t per_beat = 0;
  std::vector<int32_t> intervals, pointers;  // pointers: 0 no beat, 1 beat, 2 downbeat
  std::vector<double> log_tempo;

  // beat_this_b200/dbn.py::_BarModel.__init__
  void build(int32_t beats_, double min_interval, double max_interval, int32_t num_tempi, double transition_lambda,
             double observation_lambda) {
    beats = beats_;
    std::vector<double> iv;
    for (double i = std::nearbyint(min_interval); i <= std::nearbyint(max_interval); i += 1.0) iv.push_back(i);
    if (num_tempi > 0 && num_tempi < static_cast<int32_t>(iv.size())) {  // log-spaced tempi, as few as requested
      int n_log = num_tempi;
      std::vector<double> u;
      while (static_cast<int32_t>(u.size()) < num_tempi) {
        u.clear();
        const double lo = std::log2(min_interval), hi = std::log2(max_interval);
        for (int i = 0; i < n_log; ++i) {
          const double e = n_log > 1 ? lo + (hi - lo) * i / (n_log - 1) : lo;
          u.push_back(std::nearbyint(std::exp2(e)));
        }
        std::sort(u.begin(), u.end());
        u.erase(std::unique(u.begin(), u.end()), u.end());
        ++n_log;
      }
      iv = u;
    }
    n_int = static_cast<int32_t>(iv.size());
    intervals.resize(n_int);
    per_beat = 0;
    for (int k = 0; k < n_int; ++k) { intervals[k] = static_cast<int32_t>(iv[k]); per_beat += intervals[k]; }
    log_tempo.assign(static_cast<size_t>(n_int) * n_int, 0.0);
    const double eps = std::nextafter(1.0, 2.0) - 1.0;  // np.spacing(1)
    for (int f = 0; f < n_int; ++f) {
      double sum = 0.0;
      for (int k = 0; k < n_int; ++k) {
        double p = std::exp(-transition_lambda * std::fabs(iv[k] / iv[f] - 1.0));
        if (p <= eps) p = 0.0;
        log_tempo[f * n_int + k] = p;
        sum += p;
      }
      for (int k = 0; k < n_int; ++k) log_tempo[f * n_int + k] = std::log(log_tempo[f * n_int + k] / sum);
    }
    const double border = 1.0 / observation_lambda;
    pointers.assign(per_beat * beats, 0);
    for (int b = 0; b < beats; ++b) {
      int64_t s = b * per_beat;
      for (int k = 0; k < n_int; ++k)
        for (int32_t j = 0; j < intervals[k]; ++j, ++s)
          if (static_cast<double>(j) / intervals[k] < border) pointers[s] = b == 0 ? 2 : 1;
    }
  }
};

}  // namespace bt
