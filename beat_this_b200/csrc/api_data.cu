// C ABI: training batches (bt_train_batch).  The host checks every table entry before anything is enqueued, so the
// kernel may index without bounds checks.
#include "api_internal.h"

extern "C" {

int bt_train_batch(bt_ctx* c, const uint16_t* rows_dev, const int64_t* row_offsets_host, int32_t n_items,
                   int32_t length, const int32_t* row_map_host, const int32_t* beat_frames_host,
                   const int64_t* beat_offsets_host, const int32_t* downbeat_frames_host,
                   const int64_t* downbeat_offsets_host, uint16_t* out_spect_dev, uint8_t* truth_beat_dev,
                   uint8_t* truth_downbeat_dev, uint8_t* padding_mask_dev, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_train_batch";
  if (n_items < 0 || length < 1 || !row_offsets_host || !beat_offsets_host || !downbeat_offsets_host)
    return fail(c, BT_ERR_ARG, "%s: bad argument", fn);
  int r = check_offsets(c, fn, "row_offsets_host", row_offsets_host, n_items, kFromZero);
  if (r == BT_OK) r = check_offsets(c, fn, "beat_offsets_host", beat_offsets_host, n_items, kFromZero);
  if (r == BT_OK) r = check_offsets(c, fn, "downbeat_offsets_host", downbeat_offsets_host, n_items, kFromZero);
  if (r != BT_OK) return r;
  if (n_items == 0) return BT_OK;
  const int64_t n_rows = row_offsets_host[n_items], n_beats = beat_offsets_host[n_items],
                n_downs = downbeat_offsets_host[n_items];
  if (!out_spect_dev || !truth_beat_dev || !truth_downbeat_dev || !padding_mask_dev || (n_rows > 0 && !rows_dev) ||
      (n_beats > 0 && !beat_frames_host) || (n_downs > 0 && !downbeat_frames_host))
    return fail(c, BT_ERR_ARG, "%s: null pointer", fn);
  const struct { const char* name; const int32_t* v; const int64_t* off; } frames[2] = {
      {"beat_frames_host", beat_frames_host, beat_offsets_host},
      {"downbeat_frames_host", downbeat_frames_host, downbeat_offsets_host}};
  for (int32_t i = 0; i < n_items; ++i) {
    const int64_t n = row_offsets_host[i + 1] - row_offsets_host[i];
    if (n > length) return fail(c, BT_ERR_ARG, "%s: item %d has %lld rows, more than length %d", fn, i, (long long)n, length);
    if (row_map_host)
      for (int64_t k = row_offsets_host[i]; k < row_offsets_host[i + 1]; ++k)
        if (row_map_host[k] < -1 || row_map_host[k] >= n)
          return fail(c, BT_ERR_ARG, "%s: row_map_host[%lld] = %d outside [-1, %lld) of item %d", fn, (long long)k,
                      row_map_host[k], (long long)n, i);
    for (const auto& f : frames)
      for (int64_t k = f.off[i]; k < f.off[i + 1]; ++k) {
        if (f.v[k] < 0 || f.v[k] >= n)
          return fail(c, BT_ERR_ARG, "%s: %s[%lld] = %d outside [0, %lld) of item %d", fn, f.name, (long long)k, f.v[k],
                      (long long)n, i);
        if (k > f.off[i] && f.v[k] < f.v[k - 1])
          return fail(c, BT_ERR_ARG, "%s: %s of item %d must not decrease", fn, f.name, i);
      }
  }
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const size_t n = static_cast<size_t>(n_items) + 1;
  const int64_t* off_dev[3];
  if ((r = stage(c, st, {{row_offsets_host, n}, {beat_offsets_host, n}, {downbeat_offsets_host, n}}, off_dev)) != BT_OK)
    return r;
  static const int32_t kNone = 0;  // stands for an absent table of 0 entries
  const int32_t* tab_dev[3];
  if ((r = stage(c, st, {{row_map_host ? row_map_host : &kNone, row_map_host ? static_cast<size_t>(n_rows) : 0},
                         {n_beats ? beat_frames_host : &kNone, static_cast<size_t>(n_beats)},
                         {n_downs ? downbeat_frames_host : &kNone, static_cast<size_t>(n_downs)}}, tab_dev)) != BT_OK)
    return r;
  launch_train_batch(rows_dev, off_dev[0], n_items, length, row_map_host ? tab_dev[0] : nullptr, tab_dev[1], off_dev[1],
                     tab_dev[2], off_dev[2], out_spect_dev, truth_beat_dev, truth_downbeat_dev, padding_mask_dev, st);
  BT_LAUNCHED(c, "train_batch", st);
  return BT_OK;
}

}  // extern "C"
