// C ABI (include/beatthis.h): the signal entry points, which need no weights -- log-mel spectrograms, resampling, and
// the STFT, phase vocoder and inverse STFT of tempo and pitch augmentation.
#include "api_internal.h"

// n_fft of a bt_stft_config as log2, or 0 when it is not a power of two in [64, 8192]
static int fft_log2(int n_fft) {
  for (int l = 6; l <= 13; ++l)
    if ((1 << l) == n_fft) return l;
  return 0;
}

// Smallest window envelope sum w^2 over the samples [n_fft / 2, n_fft / 2 + len) that one of F frames covers, for the
// periodic Hann window in float64.  C[i] = w^2[i] + C[i - hop] sums a residue class of the window, so the envelope at
// p is a difference of two entries; the samples between the first and the last n_fft repeat with period hop.
static double istft_min_envelope(const std::vector<double>& C, int N, int hop, int64_t F, int64_t len) {
  const int64_t end = std::min<int64_t>(N / 2 + len, N + hop * (F - 1));
  double mn = INFINITY;
  auto env = [&](int64_t p) {
    const int64_t f_hi = std::min<int64_t>(F - 1, p / hop), f_lo = p < N ? 0 : (p - N) / hop + 1;
    const int64_t top = p - f_lo * hop, below = p - f_hi * hop - hop;  // window indices: top down to below + hop
    return C[top] - (below >= 0 ? C[below] : 0.0);
  };
  const int64_t head_end = std::min<int64_t>(end, static_cast<int64_t>(N) + hop);
  for (int64_t p = N / 2; p < head_end; ++p) mn = std::min(mn, env(p));
  for (int64_t p = std::max<int64_t>(head_end, end - N - hop); p < end; ++p) mn = std::min(mn, env(p));
  return mn;
}

extern "C" {

int bt_logmel(bt_ctx* c, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
              float* spect_dev, const int64_t* frame_offsets_host, void* stream) {
  if (!c) return BT_ERR_ARG;
  for (const char* n : {"mel.window", "mel.twiddle", "mel.fb_start", "mel.fb_ptr", "mel.fb_w"})
    if (!find_param(c, n)) return fail(c, BT_ERR_STATE, "bt_logmel: parameter '%s' not set", n);
  if (n_clips < 0) return fail(c, BT_ERR_ARG, "bt_logmel: negative clip count");
  if (n_clips == 0) return BT_OK;
  if (!audio_dev || !sample_offsets_host || !spect_dev || !frame_offsets_host)
    return fail(c, BT_ERR_ARG, "bt_logmel: null argument");
  int r = check_stft_frames(c, "bt_logmel", sample_offsets_host, frame_offsets_host, n_clips, BT_N_FFT, BT_HOP);
  cudaStream_t st;
  if (r != BT_OK || (r = enter(c, "bt_logmel", stream, &st)) != BT_OK) return r;
  const size_t n = n_clips + 1;
  const int64_t* d[2];
  if ((r = stage(c, st, {{sample_offsets_host, n}, {frame_offsets_host, n}}, d)) != BT_OK) return r;
  int64_t max_frames = 0;
  for (int i = 0; i < n_clips; ++i) max_frames = std::max(max_frames, frame_offsets_host[i + 1] - frame_offsets_host[i]);
  launch_logmel(audio_dev, d[0], d[1], n_clips, max_frames, find_param(c, "mel.window")->f32.get(),
                find_param(c, "mel.twiddle")->f32.get(), find_param(c, "mel.fb_start")->i32.get(),
                find_param(c, "mel.fb_ptr")->i32.get(), find_param(c, "mel.fb_w")->f32.get(), spect_dev, st);
  BT_LAUNCHED(c, "logmel", st);
  return BT_OK;
}

int bt_logmel_config(bt_ctx* c, const bt_mel_config* cfg, const float* window_dev, const float* twiddle_dev,
                     const int32_t* fb_start_dev, const int32_t* fb_ptr_dev, const float* fb_w_dev,
                     const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                     float* spect_dev, const int64_t* frame_offsets_host, void* stream) {
  static const char* fn = "bt_logmel_config";
  if (!c) return BT_ERR_ARG;
  if (!cfg) return fail(c, BT_ERR_ARG, "%s: null config", fn);
  const int log2n = fft_log2(cfg->n_fft);
  if (!log2n) return fail(c, BT_ERR_ARG, "%s: n_fft %d is not a power of two in [64, 8192]", fn, cfg->n_fft);
  if (cfg->hop_length < 1 || cfg->n_mels < 1 || cfg->n_mels > 1024)
    return fail(c, BT_ERR_ARG, "%s: need hop_length >= 1 and 1 <= n_mels <= 1024", fn);
  if (cfg->norm_mode < BT_MEL_NORM_NONE || cfg->norm_mode > BT_MEL_NORM_WINDOW)
    return fail(c, BT_ERR_ARG, "%s: unknown norm_mode %d", fn, cfg->norm_mode);
  if (!std::isfinite(cfg->power) || !(cfg->power > 0.f) || !std::isfinite(cfg->log_multiplier))
    return fail(c, BT_ERR_ARG, "%s: need a finite power > 0 and a finite log_multiplier", fn);
  if (n_clips < 0) return fail(c, BT_ERR_ARG, "%s: negative clip count", fn);
  if (n_clips == 0) return BT_OK;
  if (!window_dev || !twiddle_dev || !fb_start_dev || !fb_ptr_dev || !fb_w_dev || !audio_dev || !sample_offsets_host ||
      !spect_dev || !frame_offsets_host)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  int r = check_stft_frames(c, fn, sample_offsets_host, frame_offsets_host, n_clips, cfg->n_fft, cfg->hop_length);
  cudaStream_t st;
  if (r != BT_OK || (r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const size_t n = n_clips + 1;
  const int64_t* d[2];
  if ((r = stage(c, st, {{sample_offsets_host, n}, {frame_offsets_host, n}}, d)) != BT_OK) return r;
  const MelConfigArgs args{window_dev, twiddle_dev, fb_start_dev, fb_ptr_dev, fb_w_dev, spect_dev,
                           cfg->hop_length, cfg->n_mels, cfg->norm_mode, cfg->power, cfg->log_multiplier};
  BT_LAUNCHED(c, "logmel_config", st,
              launch_logmel_config(log2n, audio_dev, d[0], d[1], n_clips, frame_offsets_host[n_clips], args, st));
  return BT_OK;
}

int bt_resample(bt_ctx* c, const float* audio_in_dev, const int64_t* in_offsets_host, int32_t n_clips,
                const float* coef_dev, int32_t L, int32_t M, int32_t K, float* audio_out_dev,
                const int64_t* out_offsets_host, void* stream) {
  if (!c) return BT_ERR_ARG;
  if (n_clips < 0) return fail(c, BT_ERR_ARG, "bt_resample: negative clip count");
  if (n_clips == 0) return BT_OK;
  if (!audio_in_dev || !in_offsets_host || !coef_dev || !audio_out_dev || !out_offsets_host)
    return fail(c, BT_ERR_ARG, "bt_resample: null argument");
  if (L <= 0 || M <= 0 || K <= 0 || (K & 1)) return fail(c, BT_ERR_ARG, "bt_resample: need L, M > 0 and an even K > 0");
  int r = check_offsets(c, "bt_resample", "in_offsets_host", in_offsets_host, n_clips, kFromNonNegative);
  if (r == BT_OK) r = check_offsets(c, "bt_resample", "out_offsets_host", out_offsets_host, n_clips, kFromNonNegative);
  if (r != BT_OK) return r;
  int64_t max_out = 0;
  for (int i = 0; i < n_clips; ++i) max_out = std::max(max_out, out_offsets_host[i + 1] - out_offsets_host[i]);
  if (max_out > 0 && resample_smem(L, M, K) > kResampleMaxSmem)
    return fail(c, BT_ERR_ARG, "bt_resample: ratio %d/%d with %d taps needs too much shared memory", L, M, K);
  cudaStream_t st;
  if ((r = enter(c, "bt_resample", stream, &st)) != BT_OK) return r;
  const size_t n = n_clips + 1;
  const int64_t* d[2];
  if ((r = stage(c, st, {{in_offsets_host, n}, {out_offsets_host, n}}, d)) != BT_OK) return r;
  BT_LAUNCHED(c, "resample", st,
              launch_resample(audio_in_dev, d[0], audio_out_dev, d[1], n_clips, max_out, coef_dev, L, M, K, st));
  return BT_OK;
}

int bt_stft(bt_ctx* c, const bt_stft_config* cfg, const float* window_dev, const float* twiddle_dev,
            const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips, float* spec_dev,
            const int64_t* frame_offsets_host, void* stream) {
  static const char* fn = "bt_stft";
  if (!c) return BT_ERR_ARG;
  if (!cfg) return fail(c, BT_ERR_ARG, "%s: null config", fn);
  const int log2n = fft_log2(cfg->n_fft);
  if (!log2n) return fail(c, BT_ERR_ARG, "%s: n_fft %d is not a power of two in [64, 8192]", fn, cfg->n_fft);
  if (cfg->hop_length < 1) return fail(c, BT_ERR_ARG, "%s: need hop_length >= 1", fn);
  if (n_clips < 0) return fail(c, BT_ERR_ARG, "%s: negative clip count", fn);
  if (n_clips == 0) return BT_OK;
  if (!window_dev || !twiddle_dev || !audio_dev || !sample_offsets_host || !spec_dev || !frame_offsets_host)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  int r = check_stft_frames(c, fn, sample_offsets_host, frame_offsets_host, n_clips, cfg->n_fft, cfg->hop_length);
  cudaStream_t st;
  if (r != BT_OK || (r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const size_t n = n_clips + 1;
  const int64_t* d[2];
  if ((r = stage(c, st, {{sample_offsets_host, n}, {frame_offsets_host, n}}, d)) != BT_OK) return r;
  BT_LAUNCHED(c, "stft", st,
              launch_stft(log2n, audio_dev, d[0], d[1], n_clips, frame_offsets_host[n_clips], window_dev, twiddle_dev,
                          cfg->hop_length, spec_dev, st));
  return BT_OK;
}

int bt_phase_vocoder(bt_ctx* c, int32_t n_fft, const float* spec_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                     const int32_t* variant_clip_host, const double* variant_rate_host, int32_t n_variants,
                     float* out_dev, const int64_t* out_frame_offsets_host, void* stream) {
  static const char* fn = "bt_phase_vocoder";
  if (!c) return BT_ERR_ARG;
  if (!fft_log2(n_fft)) return fail(c, BT_ERR_ARG, "%s: n_fft %d is not a power of two in [64, 8192]", fn, n_fft);
  if (n_clips < 0 || n_variants < 0 || n_variants > 65535)
    return fail(c, BT_ERR_ARG, "%s: need n_clips >= 0 and 0 <= n_variants <= 65535", fn);
  if (n_variants == 0) return BT_OK;
  if (!spec_dev || !frame_offsets_host || !variant_clip_host || !variant_rate_host || !out_dev || !out_frame_offsets_host)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  int r = check_offsets(c, fn, "frame_offsets_host", frame_offsets_host, n_clips, kFromZero);
  if (r == BT_OK) r = check_offsets(c, fn, "out_frame_offsets_host", out_frame_offsets_host, n_variants, kFromZero);
  if (r != BT_OK) return r;
  std::vector<VocoderVariant> variants(n_variants);
  for (int v = 0; v < n_variants; ++v) {
    const int clip = variant_clip_host[v];
    const double rate = variant_rate_host[v];
    if (clip < 0 || clip >= n_clips) return fail(c, BT_ERR_ARG, "%s: variant %d names clip %d of %d", fn, v, clip, n_clips);
    if (!std::isfinite(rate) || rate < BT_VOCODER_MIN_RATE || rate > BT_VOCODER_MAX_RATE)
      return fail(c, BT_ERR_ARG, "%s: variant %d has rate %g outside [%g, %g]", fn, v, rate, BT_VOCODER_MIN_RATE,
                  BT_VOCODER_MAX_RATE);
    const int64_t T = frame_offsets_host[clip + 1] - frame_offsets_host[clip];
    if (T < 1) return fail(c, BT_ERR_ARG, "%s: clip %d has no frames", fn, clip);
    const int64_t T_out = static_cast<int64_t>(std::ceil(static_cast<double>(T) / rate));
    if (out_frame_offsets_host[v + 1] - out_frame_offsets_host[v] != T_out)
      return fail(c, BT_ERR_ARG, "%s: out_frame_offsets do not match ceil(%lld / %g) frames for variant %d", fn,
                  (long long)T, rate, v);
    variants[v] = VocoderVariant{frame_offsets_host[clip], out_frame_offsets_host[v], T, T_out, rate};
  }
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const VocoderVariant* d[1];
  if ((r = stage(c, st, {{variants.data(), variants.size()}}, d)) != BT_OK) return r;
  launch_phase_vocoder(spec_dev, d[0], n_variants, n_fft / 2 + 1, out_dev, st);
  BT_LAUNCHED(c, "phase_vocoder", st);
  return BT_OK;
}

int bt_istft(bt_ctx* c, const bt_stft_config* cfg, const float* window_dev, const float* twiddle_dev,
             const float* spec_dev, const int64_t* frame_offsets_host, int32_t n_seqs, float* audio_out_dev,
             const int64_t* out_sample_offsets_host, void* stream) {
  static const char* fn = "bt_istft";
  if (!c) return BT_ERR_ARG;
  if (!cfg) return fail(c, BT_ERR_ARG, "%s: null config", fn);
  const int log2n = fft_log2(cfg->n_fft);
  if (!log2n) return fail(c, BT_ERR_ARG, "%s: n_fft %d is not a power of two in [64, 8192]", fn, cfg->n_fft);
  if (cfg->hop_length < 1) return fail(c, BT_ERR_ARG, "%s: need hop_length >= 1", fn);
  if (n_seqs < 0 || n_seqs > 65535) return fail(c, BT_ERR_ARG, "%s: need 0 <= n_seqs <= 65535", fn);
  if (n_seqs == 0) return BT_OK;
  if (!window_dev || !twiddle_dev || !spec_dev || !frame_offsets_host || !audio_out_dev || !out_sample_offsets_host)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  int r = check_offsets(c, fn, "frame_offsets_host", frame_offsets_host, n_seqs, kFromZero);
  if (r == BT_OK) r = check_offsets(c, fn, "out_sample_offsets_host", out_sample_offsets_host, n_seqs, kFromNonNegative);
  if (r != BT_OK) return r;
  const int N = cfg->n_fft, hop = cfg->hop_length;
  if (hop >= N)
    return fail(c, BT_ERR_ARG, "%s: hop_length %d >= n_fft %d leaves samples with a zero window envelope", fn, hop, N);
  std::vector<double> C(N);
  for (int i = 0; i < N; ++i) {
    const double w = 0.5 - 0.5 * std::cos(2.0 * M_PI * i / N);
    C[i] = w * w + (i >= hop ? C[i - hop] : 0.0);
  }
  int64_t max_out = 0;
  for (int s = 0; s < n_seqs; ++s) {
    const int64_t F = frame_offsets_host[s + 1] - frame_offsets_host[s];
    const int64_t len = out_sample_offsets_host[s + 1] - out_sample_offsets_host[s];
    if (F < 1) return fail(c, BT_ERR_ARG, "%s: sequence %d has no frames", fn, s);
    if (len > 0 && istft_min_envelope(C, N, hop, F, len) < 1e-11)
      return fail(c, BT_ERR_ARG, "%s: sequence %d: window envelope below 1e-11 within its %lld samples (torch.istft "
                  "raises there as well)", fn, s, (long long)len);
    max_out = std::max(max_out, len);
  }
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const int64_t total_frames = frame_offsets_host[n_seqs];
  const size_t bytes = sizeof(float) * static_cast<size_t>(total_frames) * N;
  BT_CUDA(c, c->istft_frames.reserve(bytes, bytes));
  const size_t n = static_cast<size_t>(n_seqs) + 1;
  const int64_t* d[2];
  if ((r = stage(c, st, {{frame_offsets_host, n}, {out_sample_offsets_host, n}}, d)) != BT_OK) return r;
  BT_LAUNCHED(c, "istft", st,
              launch_istft_frames(log2n, spec_dev, total_frames, window_dev, twiddle_dev, c->istft_frames.get(), st));
  if (max_out > 0) {
    launch_istft_ola(c->istft_frames.get(), d[0], d[1], n_seqs, max_out, window_dev, N, hop, audio_out_dev, st);
    BT_LAUNCHED(c, "istft_overlap_add", st);
  }
  return BT_OK;
}
}  // extern "C"
