// C ABI (include/beatthis.h): post-processing, evaluation and training on the device -- peak picking, the DBN
// tracker, beat metrics and the training losses -- and the DBN model and staging helpers the Viterbi hook shares.
#include "api_internal.h"
#include "dbn_model.h"

constexpr size_t kDbnStaticSmem = 512;  // dbn_viterbi_kernel's block reduction

int bt::dbn_host_model(bt_ctx* c, const char* fn, int32_t beats, int32_t n_int, const int32_t* intervals,
                   const double* log_tempo, const int32_t* pointers, DbnHostModel& m) {
  if (n_int < 1 || n_int > 255)
    return fail(c, BT_ERR_ARG, "%s: %d tempi; the device decoder stores back pointers as bytes and takes 1..255 tempi", fn, n_int);
  if (beats < 1 || beats > 127) return fail(c, BT_ERR_ARG, "%s: %d beats per bar; the device decoder takes 1..127", fn, beats);
  if (beats * n_int > 1024)
    return fail(c, BT_ERR_ARG, "%s: %d beats x %d tempi; the device decoder runs one thread per (beat, tempo), at most 1024",
                fn, beats, n_int);
  m.beats = beats;
  m.n_int = n_int;
  m.intervals.assign(intervals, intervals + n_int);
  m.first.resize(n_int);
  int64_t per_beat = 0;
  for (int k = 0; k < n_int; ++k) {
    if (intervals[k] <= 0) return fail(c, BT_ERR_ARG, "%s: beat intervals must be positive", fn);
    m.first[k] = static_cast<int32_t>(per_beat);
    per_beat += intervals[k];
  }
  const int64_t S = per_beat * beats;
  m.smem = dbn_viterbi_smem(beats, n_int, static_cast<int>(std::min<int64_t>(per_beat, INT32_MAX / 256)));
  int optin = 0;
  BT_CUDA(c, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
  if (per_beat > INT32_MAX / 256 || m.smem + kDbnStaticSmem > static_cast<size_t>(optin))
    return fail(c, BT_ERR_ARG, "%s: a %d-beat model with %d tempi has %lld states and needs %zu bytes of shared memory; the "
                "device allows %d per block", fn, beats, n_int, static_cast<long long>(S), m.smem + kDbnStaticSmem, optin);
  m.per_beat = static_cast<int32_t>(per_beat);
  // the ring form needs every (beat, tempo) to observe the (down)beat density on a leading run of positions and the
  // "no beat" density on the rest (what BarModel::build produces)
  m.nrun.resize(static_cast<size_t>(beats) * n_int);
  for (int b = 0; b < beats; ++b)
    for (int k = 0; k < n_int; ++k) {
      const int32_t* pt = pointers + static_cast<int64_t>(b) * per_beat + m.first[k];
      const int32_t lead = b == 0 ? 2 : 1;
      int32_t n = 0;
      while (n < intervals[k] && pt[n] == lead) ++n;
      bool ok = n > 0;
      for (int32_t p = n; p < intervals[k]; ++p) ok = ok && pt[p] == 0;
      if (!ok)
        return fail(c, BT_ERR_ARG, "%s: beat %d, tempo %d: the pointers are not a leading run of %d followed by 0 (the only "
                    "form the device decoder handles)", fn, b, k, lead);
      m.nrun[static_cast<size_t>(b) * n_int + k] = n;
    }
  m.log_tempo.assign(log_tempo, log_tempo + static_cast<size_t>(n_int) * n_int);
  m.init = -std::log(static_cast<double>(S));
  return BT_OK;
}

// Model tables, frame offsets and (optionally) the windows of the clips through one staging slot; device pointers
// into the slot come back.  bp_base of model i: the back pointers of the models before it, `total` frames each.
int bt::dbn_stage(bt_ctx* c, const std::vector<DbnHostModel>& ms, const int64_t* fo, int32_t n_clips, int64_t total,
              const int64_t* win_host, cudaStream_t st, const DbnModelDev** models_dev, const int64_t** fo_dev,
              const int64_t** win_dev) {
  const int nm = static_cast<int>(ms.size());
  size_t off = align16(sizeof(DbnModelDev) * nm);
  const size_t o_fo = off;
  off = align16(off + sizeof(int64_t) * (n_clips + 1));
  const size_t o_win = off;
  if (win_host) off = align16(off + sizeof(int64_t) * 2 * n_clips);
  std::vector<size_t> o_lt(nm), o_iv(nm), o_first(nm), o_nrun(nm);
  for (int i = 0; i < nm; ++i) {
    o_lt[i] = off; off = align16(off + sizeof(double) * ms[i].log_tempo.size());
    o_iv[i] = off; off = align16(off + sizeof(int32_t) * ms[i].n_int);
    o_first[i] = off; off = align16(off + sizeof(int32_t) * ms[i].n_int);
    o_nrun[i] = off; off = align16(off + sizeof(int32_t) * ms[i].nrun.size());
  }
  StageSlot* sl = nullptr;
  int r = acquire_stage(c, off, &sl);
  if (r != BT_OK) return r;
  char* h = sl->host.get();
  const char* d = sl->dev.get();
  int64_t bp_base = 0;
  for (int i = 0; i < nm; ++i) {
    const DbnHostModel& m = ms[i];
    DbnModelDev md{};
    md.intervals = reinterpret_cast<const int32_t*>(d + o_iv[i]);
    md.first = reinterpret_cast<const int32_t*>(d + o_first[i]);
    md.nrun = reinterpret_cast<const int32_t*>(d + o_nrun[i]);
    md.log_tempo = reinterpret_cast<const double*>(d + o_lt[i]);
    md.init = m.init;
    md.bp_base = bp_base;
    md.beats = m.beats; md.n_int = m.n_int; md.per_beat = m.per_beat;
    bp_base += static_cast<int64_t>(m.beats) * m.n_int * total;
    memcpy(h + sizeof(DbnModelDev) * i, &md, sizeof(md));
    memcpy(h + o_lt[i], m.log_tempo.data(), sizeof(double) * m.log_tempo.size());
    memcpy(h + o_iv[i], m.intervals.data(), sizeof(int32_t) * m.n_int);
    memcpy(h + o_first[i], m.first.data(), sizeof(int32_t) * m.n_int);
    memcpy(h + o_nrun[i], m.nrun.data(), sizeof(int32_t) * m.nrun.size());
  }
  memcpy(h + o_fo, fo, sizeof(int64_t) * (n_clips + 1));
  if (win_host) memcpy(h + o_win, win_host, sizeof(int64_t) * 2 * n_clips);
  if ((r = upload_stage(c, sl, off, st)) != BT_OK) return r;
  *models_dev = reinterpret_cast<const DbnModelDev*>(d);
  *fo_dev = reinterpret_cast<const int64_t*>(d + o_fo);
  if (win_dev) *win_dev = win_host ? reinterpret_cast<const int64_t*>(d + o_win) : nullptr;
  return BT_OK;
}

void bt::dbn_launch_shape(const std::vector<DbnHostModel>& ms, int* threads, size_t* smem, size_t* bp_per_frame) {
  int bn = 0;
  *smem = 0;
  *bp_per_frame = 0;
  for (const auto& m : ms) {
    bn = std::max(bn, m.beats * m.n_int);
    *smem = std::max(*smem, m.smem);
    *bp_per_frame += static_cast<size_t>(m.beats) * m.n_int;
  }
  *threads = (bn + 31) / 32 * 32;
}

static int peakpick(bt_ctx* c, const char* fn, const float* beat_dev, const float* downbeat_dev,
             const int64_t* frame_offsets_host, int32_t n_clips, double* beat_times_dev, int32_t* n_beats_dev,
             double* down_times_dev, int32_t* n_down_dev, int32_t max_peaks, double fps, void* stream) {
  if (!c) return BT_ERR_ARG;
  if (!std::isfinite(fps) || !(fps > 0)) return fail(c, BT_ERR_ARG, "%s: fps must be finite and > 0", fn);
  if (n_clips <= 0) return BT_OK;
  if (!beat_dev || !downbeat_dev || !frame_offsets_host || !beat_times_dev || !n_beats_dev || !down_times_dev ||
      !n_down_dev || max_peaks < 1)
    return fail(c, BT_ERR_ARG, "%s: bad argument", fn);
  int r = check_offsets(c, fn, "frame_offsets_host", frame_offsets_host, n_clips, kFromNonNegative);
  cudaStream_t st;
  if (r != BT_OK || (r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const int64_t* fo = nullptr;
  if ((r = stage(c, st, {{frame_offsets_host, static_cast<size_t>(n_clips + 1)}}, &fo)) != BT_OK) return r;
  launch_peakpick(beat_dev, downbeat_dev, fo, n_clips, beat_times_dev,
                  n_beats_dev, down_times_dev, n_down_dev, max_peaks, fps, st);
  BT_LAUNCHED(c, "peakpick", st);
  return BT_OK;
}

// The checks bt_beat_loss and its backward share, before anything is enqueued: params, pointers, offsets.  Fills the
// kernels' view of the params, the CTA prefix per row (forward or backward tiling) and the scored frames of all rows.
static int loss_prepare(bt_ctx* c, const char* fn, const float* preds, const float* targets, const float* mask,
                 const int64_t* off, int32_t n_rows, const bt_loss_params* params, bool backward, LossParams* p,
                 std::vector<int64_t>* tile_first, int64_t* n_scored) {
  if (!params || !off || !preds || !targets) return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  *p = LossParams{params->kind, params->tolerance, params->pos_weight};
  if (p->kind < BT_LOSS_MASKED_BCE || p->kind > BT_LOSS_SPLIT_SHIFT_TOLERANT)
    return fail(c, BT_ERR_ARG, "%s: unknown loss kind %d", fn, p->kind);
  if (p->tolerance < 0 || p->tolerance > BT_LOSS_MAX_TOLERANCE)
    return fail(c, BT_ERR_ARG, "%s: tolerance %d outside [0, %d]", fn, p->tolerance, BT_LOSS_MAX_TOLERANCE);
  if (!std::isfinite(p->pos_weight)) return fail(c, BT_ERR_ARG, "%s: pos_weight must be finite", fn);
  if (p->kind == BT_LOSS_SPLIT_SHIFT_TOLERANT && !mask) return fail(c, BT_ERR_ARG, "%s: the split kind needs a mask", fn);
  if (n_rows < 1) return fail(c, BT_ERR_ARG, "%s: need n_rows >= 1", fn);
  if (const int r = check_offsets(c, fn, "row_offsets_host", off, n_rows, kFromZero)) return r;
  const int64_t min_len = p->kind == BT_LOSS_MASKED_BCE ? 1 : 4 * static_cast<int64_t>(p->tolerance) + 1;
  tile_first->assign(1, 0);
  *n_scored = 0;
  for (int i = 0; i < n_rows; ++i) {
    const int64_t len = off[i + 1] - off[i];
    if (len < min_len) return fail(c, BT_ERR_ARG, "%s: row %d has %lld frames, fewer than %lld", fn, i,
                                   static_cast<long long>(len), static_cast<long long>(min_len));
    tile_first->push_back(tile_first->back() + loss_tiles(len, *p, backward));
    *n_scored += p->kind == BT_LOSS_MASKED_BCE ? len : len - 4 * static_cast<int64_t>(p->tolerance);
  }
  if (tile_first->back() > 0x7fffffff) return fail(c, BT_ERR_ARG, "%s: too many frames", fn);
  return BT_OK;
}

static_assert(BT_BEAT_METRIC_COLS == kBeatMetricCols, "bt_beat_metrics row width");
static_assert(BT_LOSS_MAX_TOLERANCE == kLossMaxTolerance, "bt_loss_params tolerance cap");

extern "C" {

int bt_peakpick(bt_ctx* c, const float* beat_dev, const float* downbeat_dev, const int64_t* frame_offsets_host,
                int32_t n_clips, double* beat_times_dev, int32_t* n_beats_dev, double* down_times_dev,
                int32_t* n_down_dev, int32_t max_peaks, void* stream) {
  return peakpick(c, "bt_peakpick", beat_dev, downbeat_dev, frame_offsets_host, n_clips, beat_times_dev, n_beats_dev,
                  down_times_dev, n_down_dev, max_peaks, 50.0, stream);
}

int bt_peakpick_fps(bt_ctx* c, const float* beat_dev, const float* downbeat_dev, const int64_t* frame_offsets_host,
                    int32_t n_clips, double fps, double* beat_times_dev, int32_t* n_beats_dev, double* down_times_dev,
                    int32_t* n_down_dev, int32_t max_peaks, void* stream) {
  return peakpick(c, "bt_peakpick_fps", beat_dev, downbeat_dev, frame_offsets_host, n_clips, beat_times_dev,
                  n_beats_dev, down_times_dev, n_down_dev, max_peaks, fps, stream);
}

int bt_dbn_track_device(bt_ctx* c, const float* beat_logits_dev, const float* downbeat_logits_dev,
                        const double* activations_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                        const int32_t* beats_per_bar, int32_t n_bar_lengths, double min_bpm, double max_bpm,
                        int32_t num_tempi, double transition_lambda, double observation_lambda, double threshold,
                        int32_t correct, double fps, double* times_dev, int32_t* numbers_dev, int64_t* counts_dev,
                        void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_dbn_track_device";
  const bool logits = beat_logits_dev || downbeat_logits_dev;
  if (logits == (activations_dev != nullptr) || (logits && !(beat_logits_dev && downbeat_logits_dev)))
    return fail(c, BT_ERR_ARG, "%s: pass either both logit arrays or the activations", fn);
  if (n_clips < 0 || !frame_offsets_host || !beats_per_bar || n_bar_lengths <= 0 || n_bar_lengths > 16 || !(min_bpm > 0) ||
      !(max_bpm > min_bpm) || !(fps > 0) || !(observation_lambda > 1))
    return fail(c, BT_ERR_ARG, "%s: bad model parameters (1..16 bar lengths, 0 < min_bpm < max_bpm, fps > 0, "
                "observation_lambda > 1)", fn);
  if (n_clips == 0) return BT_OK;
  if (!times_dev || !numbers_dev || !counts_dev) return fail(c, BT_ERR_ARG, "%s: null output", fn);
  std::vector<DbnHostModel> ms(n_bar_lengths);
  for (int i = 0; i < n_bar_lengths; ++i) {
    if (beats_per_bar[i] <= 0) return fail(c, BT_ERR_ARG, "%s: beats_per_bar must be positive", fn);
    BarModel bm;
    bm.build(beats_per_bar[i], 60.0 * fps / max_bpm, 60.0 * fps / min_bpm, num_tempi, transition_lambda, observation_lambda);
    int r = dbn_host_model(c, fn, bm.beats, bm.n_int, bm.intervals.data(), bm.log_tempo.data(), bm.pointers.data(), ms[i]);
    if (r != BT_OK) return r;
  }
  int threads;
  size_t smem, bp_per_frame;
  dbn_launch_shape(ms, &threads, &smem, &bp_per_frame);
  const int64_t total = frame_offsets_host[n_clips];
  const size_t nres = static_cast<size_t>(n_clips) * n_bar_lengths;
  const size_t o_dens = align16(sizeof(double) * 2 * total);
  const size_t o_win = align16(o_dens + sizeof(double) * 3 * total);
  const size_t o_logp = align16(o_win + sizeof(int64_t) * 2 * n_clips);
  const size_t o_state = align16(o_logp + sizeof(double) * nres);
  const size_t o_codes = align16(o_state + sizeof(int64_t) * nres);
  const size_t ws_bytes = o_codes + static_cast<size_t>(total);
  int r = check_offsets(c, fn, "frame_offsets_host", frame_offsets_host, n_clips, kFromNonNegative);
  cudaStream_t st;
  if (r != BT_OK || (r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const size_t bp_bytes = std::max<size_t>(bp_per_frame * total, 1);
  BT_CUDA(c, c->dbn_ws.reserve(ws_bytes, ws_bytes + ws_bytes / 4));
  BT_CUDA(c, c->dbn_bp.reserve(bp_bytes, bp_bytes + bp_bytes / 4));
  const DbnModelDev* md = nullptr;
  const int64_t* fo_dev = nullptr;
  if ((r = dbn_stage(c, ms, frame_offsets_host, n_clips, total, nullptr, st, &md, &fo_dev, nullptr)) != BT_OK) return r;
  char* ws = c->dbn_ws.get();
  double* act = reinterpret_cast<double*>(ws);
  double* dens = reinterpret_cast<double*>(ws + o_dens);
  int64_t* win = reinterpret_cast<int64_t*>(ws + o_win);
  double* res_logp = reinterpret_cast<double*>(ws + o_logp);
  int64_t* res_state = reinterpret_cast<int64_t*>(ws + o_state);
  uint8_t* codes = reinterpret_cast<uint8_t*>(ws + o_codes);
  uint8_t* bp = c->dbn_bp.get();
  launch_dbn_prep(beat_logits_dev, downbeat_logits_dev, activations_dev, fo_dev, n_clips, threshold, observation_lambda,
                  act, dens, win, st);
  BT_LAUNCHED(c, "dbn_prep", st);
  BT_LAUNCHED(c, "dbn_viterbi", st,
              launch_dbn_viterbi(md, n_bar_lengths, threads, smem, dens, fo_dev, win, n_clips, bp, res_logp, res_state, st));
  launch_dbn_backtrace(md, n_bar_lengths, fo_dev, win, n_clips, bp, res_logp, res_state, act, codes, correct != 0, fps,
                       times_dev, numbers_dev, counts_dev, nullptr, nullptr, st);
  BT_LAUNCHED(c, "dbn_backtrace", st);
  return BT_OK;
}

int bt_beat_metrics(bt_ctx* c, const double* est_dev, const int64_t* est_offsets_host, const double* ref_dev,
                    const int64_t* ref_offsets_host, int32_t n_sets, const bt_beat_metric_params* params, double* out_dev,
                    void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_beat_metrics";
  if (n_sets < 0 || !est_offsets_host || !ref_offsets_host || !params) return fail(c, BT_ERR_ARG, "%s: bad argument", fn);
  const BeatMetricParams p{params->min_beat_time, params->f_window, params->cemgil_sigma, params->phase_threshold,
                           params->period_threshold};
  if (!std::isfinite(p.min_beat_time) || !std::isfinite(p.f_window) || !std::isfinite(p.cemgil_sigma) ||
      !std::isfinite(p.phase_threshold) || !std::isfinite(p.period_threshold))
    return fail(c, BT_ERR_ARG, "%s: parameters must be finite", fn);
  int r = check_offsets(c, fn, "est_offsets_host", est_offsets_host, n_sets, kFromNonNegative);
  if (r == BT_OK) r = check_offsets(c, fn, "ref_offsets_host", ref_offsets_host, n_sets, kFromNonNegative);
  if (r != BT_OK) return r;
  if (n_sets == 0) return BT_OK;
  if (!out_dev || (!est_dev && est_offsets_host[n_sets] > 0) || (!ref_dev && ref_offsets_host[n_sets] > 0))
    return fail(c, BT_ERR_ARG, "%s: null device pointer", fn);
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const size_t n = n_sets + 1;
  const int64_t* off_dev[2];
  if ((r = stage(c, st, {{est_offsets_host, n}, {ref_offsets_host, n}}, off_dev)) != BT_OK) return r;
  launch_beat_metrics(est_dev, off_dev[0], ref_dev, off_dev[1], n_sets, p, out_dev, st);
  BT_LAUNCHED(c, "beat_metrics", st);
  return BT_OK;
}

int bt_beat_loss(bt_ctx* c, const float* preds_dev, const float* targets_dev, const float* mask_dev,
                 const int64_t* row_offsets_host, int32_t n_rows, const bt_loss_params* params, double* row_loss_dev,
                 float* mean_dev, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_beat_loss";
  if (!row_loss_dev || !mean_dev) return fail(c, BT_ERR_ARG, "%s: null output", fn);
  LossParams p;
  std::vector<int64_t> tiles;
  int64_t n_scored = 0;
  int r = loss_prepare(c, fn, preds_dev, targets_dev, mask_dev, row_offsets_host, n_rows, params, false, &p, &tiles,
                       &n_scored);
  cudaStream_t st;
  if (r != BT_OK || (r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const int64_t n_tiles = tiles.back();
  const size_t bytes = sizeof(double) * n_tiles;
  BT_CUDA(c, c->loss_partials.reserve(bytes, bytes + bytes / 4));
  const size_t n = static_cast<size_t>(n_rows) + 1;
  const int64_t* dev[2];
  if ((r = stage(c, st, {{row_offsets_host, n}, {tiles.data(), n}}, dev)) != BT_OK) return r;
  launch_beat_loss(preds_dev, targets_dev, mask_dev, dev[0], dev[1], n_rows, n_tiles, p, c->loss_partials.get(), st);
  BT_LAUNCHED(c, "beat_loss", st);
  launch_beat_loss_reduce(c->loss_partials.get(), dev[0], dev[1], n_rows, n_tiles, n_scored, p, row_loss_dev, mean_dev,
                          st);
  BT_LAUNCHED(c, "beat_loss_reduce", st);
  return BT_OK;
}

int bt_beat_loss_backward(bt_ctx* c, const float* preds_dev, const float* targets_dev, const float* mask_dev,
                          const int64_t* row_offsets_host, int32_t n_rows, const bt_loss_params* params,
                          const float* grad_mean_dev, float* grad_preds_dev, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_beat_loss_backward";
  if (!grad_mean_dev || !grad_preds_dev) return fail(c, BT_ERR_ARG, "%s: null gradient pointer", fn);
  LossParams p;
  std::vector<int64_t> tiles;
  int64_t n_scored = 0;
  int r = loss_prepare(c, fn, preds_dev, targets_dev, mask_dev, row_offsets_host, n_rows, params, true, &p, &tiles,
                       &n_scored);
  cudaStream_t st;
  if (r != BT_OK || (r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const size_t n = static_cast<size_t>(n_rows) + 1;
  const int64_t* dev[2];
  if ((r = stage(c, st, {{row_offsets_host, n}, {tiles.data(), n}}, dev)) != BT_OK) return r;
  launch_beat_loss_backward(preds_dev, targets_dev, mask_dev, dev[0], dev[1], n_rows, tiles.back(), n_scored, p,
                            grad_mean_dev, grad_preds_dev, st);
  BT_LAUNCHED(c, "beat_loss_backward", st);
  return BT_OK;
}

}  // extern "C"
