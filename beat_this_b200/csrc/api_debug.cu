// C ABI (include/beatthis.h): the kernel test hooks (bt_debug_*).  Each checks its own arguments, then runs the
// kernel under test once through run_hook (api_internal.h).
#include "api_internal.h"
#include "bt_train.h"

static bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

// The public chunk entries as the kernels' ChunkSrc, field by field (the internal layout stays private).
static std::vector<ChunkSrc> chunk_table(const bt_debug_chunk* chunks, int32_t n) {
  std::vector<ChunkSrc> v(n);
  for (int32_t i = 0; i < n; ++i) {
    ChunkSrc& s = v[i];
    s.frame_base = chunks[i].frame_base;
    s.T = chunks[i].T;
    s.start = chunks[i].start;
    s.out_base = chunks[i].out_base;
    s.write_lo = chunks[i].write_lo;
    s.write_hi = chunks[i].write_hi;
    s.len = chunks[i].len;
    s.pad_ = 0;
  }
  return v;
}

// A hook of a chunk-table kernel: uploads the checked table through the staging ring and launches the kernel
// (launch(table_dev, st)) under the profile name `what`.
template <class Launch>
static int run_chunk_hook(bt_ctx* c, const char* fn, const char* what, const bt_debug_chunk* chunks, int32_t n, void* stream,
                   Launch launch) {
  const std::vector<ChunkSrc> table = chunk_table(chunks, n);
  return run_hook(c, fn, stream, {}, [&](cudaStream_t st) {
    const ChunkSrc* dev = nullptr;
    const int r = stage(c, st, {{table.data(), table.size()}}, &dev);
    if (r != BT_OK) return r;
    launch(dev, st);
    return check_launch(c, what, st);
  });
}

extern "C" {

int bt_debug_dbn_viterbi(bt_ctx* c, const double* log_dens_dev, int64_t T, int32_t beats, int32_t n_int,
                         const int32_t* intervals, const double* log_tempo, const int32_t* pointers, int64_t* path_dev,
                         double* logp_dev, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_debug_dbn_viterbi";
  if (!log_dens_dev || !intervals || !log_tempo || !pointers || !path_dev || !logp_dev || T <= 0)
    return fail(c, BT_ERR_ARG, "%s: null argument or T <= 0", fn);
  std::vector<DbnHostModel> ms(1);
  int r = dbn_host_model(c, fn, beats, n_int, intervals, log_tempo, pointers, ms[0]);
  if (r != BT_OK) return r;
  int threads;
  size_t smem, bp_per_frame;
  dbn_launch_shape(ms, &threads, &smem, &bp_per_frame);
  return run_hook(c, fn, stream, {}, [&](cudaStream_t st) {
    const size_t ws_bytes = 2 * sizeof(double), bp_bytes = bp_per_frame * T;
    BT_CUDA(c, c->dbn_ws.reserve(ws_bytes, ws_bytes + ws_bytes / 4));
    BT_CUDA(c, c->dbn_bp.reserve(bp_bytes, bp_bytes + bp_bytes / 4));
    const int64_t fo[2] = {0, T}, win_h[2] = {0, T};
    const DbnModelDev* md = nullptr;
    const int64_t *fo_dev = nullptr, *win = nullptr;
    const int rs = dbn_stage(c, ms, fo, 1, T, win_h, st, &md, &fo_dev, &win);
    if (rs != BT_OK) return rs;
    double* res_logp = reinterpret_cast<double*>(c->dbn_ws.get());
    int64_t* res_state = reinterpret_cast<int64_t*>(res_logp + 1);
    uint8_t* bp = c->dbn_bp.get();
    BT_LAUNCHED(c, "dbn_viterbi", st,
                launch_dbn_viterbi(md, 1, threads, smem, log_dens_dev, fo_dev, win, 1, bp, res_logp, res_state, st));
    launch_dbn_backtrace(md, 1, fo_dev, win, 1, bp, res_logp, res_state, nullptr, nullptr, 0, 1.0, nullptr, nullptr,
                         nullptr, path_dev, logp_dev, st);
    return check_launch(c, "dbn_backtrace", st);
  });
}

int bt_debug_gemm(bt_ctx* c, const bt_debug_gemm_desc* d, const float* a_dev, const float* w_dev,
                  const float* bias_dev, const float* resid_dev, float* out_f32_dev, float* out_act_dev,
                  int64_t out_act_count, const float* rope_cos_dev, const float* rope_sin_dev, int32_t* tile_out,
                  void* stream) {
  const char* fn = "bt_debug_gemm";
  if (!c || !d || !a_dev || !w_dev) return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  if (d->nslab < 1 || d->nslab > kMaxSlabs || d->planes_out < 1 || d->L < 1 || d->N % 4 != 0 || d->Kslab % 16 != 0 ||
      d->lda % 4 != 0 || (out_act_dev && out_act_count < static_cast<int64_t>(d->planes_out) * d->L * d->N))
    return fail(c, BT_ERR_ARG, "%s: unsupported shape", fn);
  GemmShape g{};
  g.planes_out = d->planes_out; g.L = d->L; g.N = d->N; g.Kslab = d->Kslab; g.nslab = d->nslab;
  g.plane_mul = d->plane_mul; g.lda = d->lda;
  for (int s = 0; s < kMaxSlabs; ++s) { g.plane_add[s] = d->plane_add[s]; g.t_shift[s] = d->t_shift[s]; }
  EpiParams e{};
  e.kind = d->kind; e.bias = bias_dev; e.gelu = d->gelu;
  e.resid = resid_dev; e.ldr = d->N;
  e.out_f32 = out_f32_dev; e.ldo_f32 = d->N;
  e.out_act = out_act_dev; e.ldo_act = d->N;
  e.rope_cos = rope_cos_dev; e.rope_sin = rope_sin_dev;
  e.C = d->C; e.heads = d->heads; e.posmode = d->posmode; e.F = d->F; e.qscale = d->qscale;
  if (tile_out) tile_out[0] = tile_out[1] = 0;
  HookArray a(a_dev, static_cast<int64_t>(d->planes_in) * d->L * d->lda);
  HookArray w(w_dev, static_cast<int64_t>(d->N) * d->Kslab * d->nslab);
  HookArray out_act(out_act_dev, out_act_count, true);
  return run_hook(c, fn, stream, {&a, &w, &out_act}, [&](cudaStream_t st) {
    if (c->dtype != BT_DTYPE_H16) {
      launch_gemm_simt(a_dev, w_dev, g, e, st);
      return check_launch(c, "debug_gemm", st);
    }
    e.out_act = out_act.h16.get();
    GemmPlan p;
    const int r = make_plan(c, fn, p, [&](char* err, int n) {
      return tc_gemm_plan_create(a.h16.get(), w.h16.get(), g, d->planes_in, d->resid_epilogue != 0, e, err, n);
    });
    if (r != BT_OK) return r;
    if (tile_out) tc_gemm_plan_tile(p.get(), &tile_out[0], &tile_out[1]);
    launch_gemm_tc(p.get(), st);
    return check_launch(c, "debug_gemm", st);
  });
}

int bt_debug_attention(bt_ctx* c, const float* q_dev, const float* k_dev, const float* v_dev, const float* gates_dev,
                       float* o_dev, int64_t o_count, int32_t seqs, int32_t L, int32_t heads,
                       const int32_t* key_lens_host, int32_t seqs_per_chunk, void* stream) {
  const char* fn = "bt_debug_attention";
  if (!c || !q_dev || !k_dev || !v_dev || !gates_dev || !o_dev) return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  if (seqs < 1 || L < 1 || heads < 1 || (key_lens_host && (seqs_per_chunk < 1 || seqs % seqs_per_chunk != 0)))
    return fail(c, BT_ERR_ARG, "%s: bad geometry", fn);
  const int C = heads * 32;
  const int64_t M = static_cast<int64_t>(seqs) * L;
  if (o_count < M * C)
    return fail(c, BT_ERR_ARG, "%s: o holds %lld elements, fewer than M * C", fn, static_cast<long long>(o_count));
  // per-chunk key counts travel in the ChunkSrc table the forward pass hands the kernels (only .len is read)
  std::vector<ChunkSrc> chunks;
  if (key_lens_host) {
    chunks.assign(seqs / seqs_per_chunk, ChunkSrc{});
    for (size_t i = 0; i < chunks.size(); ++i) {
      if (key_lens_host[i] < 1 || key_lens_host[i] > L) return fail(c, BT_ERR_ARG, "%s: key length out of [1, L]", fn);
      chunks[i].len = key_lens_host[i];
    }
  }
  const bool tc = c->dtype == BT_DTYPE_H16;
  HookArray o(o_dev, o_count, true);
  DeviceBuffer<> qkv;
  return run_hook(c, fn, stream, {&o}, [&](cudaStream_t st) {
    BT_CUDA(c, qkv.alloc(M * 3 * C * (tc ? 2 : 4)));
    const ChunkSrc* chunks_dev = nullptr;
    int r = chunks.empty() ? BT_OK : stage(c, st, {{chunks.data(), chunks.size()}}, &chunks_dev);
    if (r != BT_OK) return r;
    if (tc) {
      launch_pack_qkv_test(q_dev, k_dev, v_dev, qkv.get(), seqs, L, heads, 0.17677669529663687f * 1.4426950408889634f, 1,
                           st);
      AttnPlan p;
      r = make_plan(c, fn, p, [&](char* err, int n) { return tc_attn_plan_create(qkv.get(), seqs, L, heads, err, n); });
      if (r != BT_OK) return r;
      launch_attn_time_tc(p.get(), gates_dev, o.h16.get(), st, chunks_dev, seqs_per_chunk);
    } else {
      launch_pack_qkv_test(q_dev, k_dev, v_dev, qkv.get(), seqs, L, heads, 1.0f, 0, st);
      launch_attn_time_simt(static_cast<const float*>(qkv.get()), gates_dev, o_dev, seqs, L, heads, st, chunks_dev,
                            seqs_per_chunk);
    }
    return check_launch(c, "debug_attention", st);
  });
}

int bt_debug_attention_freq(bt_ctx* c, const float* q_dev, const float* k_dev, const float* v_dev,
                            const float* gates_dev, float* o_dev, int64_t o_count, int32_t B, int32_t F, int32_t L,
                            int32_t heads, void* stream) {
  const char* fn = "bt_debug_attention_freq";
  if (!c || !q_dev || !k_dev || !v_dev || !gates_dev || !o_dev) return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  if (B < 1 || L < 1 || heads < 1 || (F != 8 && F != 16 && F != 32))
    return fail(c, BT_ERR_ARG, "%s: need B, L, heads >= 1 and F in {8, 16, 32}", fn);
  const int C = heads * 32;
  const int64_t M = static_cast<int64_t>(B) * F * L;
  if (o_count < M * C)
    return fail(c, BT_ERR_ARG, "%s: o holds %lld elements, fewer than M * C", fn, static_cast<long long>(o_count));
  const bool tc = c->dtype == BT_DTYPE_H16;
  const float inv_sqrt_d = 0.17677669529663687f;
  HookArray o(o_dev, o_count, true);
  DeviceBuffer<> qkv;
  return run_hook(c, fn, stream, {&o}, [&](cudaStream_t st) {
    BT_CUDA(c, qkv.alloc(M * 3 * C * (tc ? 2 : 4)));
    FreqPlan p;
    const int r = !tc ? BT_OK : make_plan(c, fn, p, [&](char* err, int n) {
      return tc_freq_plan_create(qkv.get(), o.h16.get(), B, F, L, heads, err, n);
    }, BT_ERR_ARG);
    if (r != BT_OK) return r;
    launch_pack_qkv_test(q_dev, k_dev, v_dev, qkv.get(), B * F, L, heads, 1.0f, tc ? 1 : 0, st);
    if (tc) launch_attn_freq_tc(p.get(), gates_dev, inv_sqrt_d, st);
    else launch_attn_freq_simt(static_cast<const float*>(qkv.get()), gates_dev, o_dev, B, F, L, heads, inv_sqrt_d, st);
    return check_launch(c, "debug_attention_freq", st);
  });
}

int bt_debug_norm(bt_ctx* c, const float* x_dev, float* xn_dev, int64_t M, int32_t C, const float* wg_dev,
                  const float* bg_dev, float* gates_dev, int32_t heads, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_debug_norm";
  const bool tc = c->dtype == BT_DTYPE_H16;
  if (!x_dev || !xn_dev || !aligned16(x_dev) || (!tc && !aligned16(xn_dev)))  // the fp32 context stores xn directly
    return fail(c, BT_ERR_ARG, "%s: need x and xn (16-byte aligned; xn only in the fp32 context)", fn);
  if (M < 1 || (C != 32 && C != 64 && C != 128 && C != 256 && C != 512 && C != 1024))
    return fail(c, BT_ERR_ARG, "%s: need M >= 1 and C in {32, 64, 128, 256, 512, 1024}", fn);
  if (gates_dev ? (!wg_dev || !bg_dev || !aligned16(wg_dev) || heads < 1 || 32 * heads > C) : heads != 0)
    return fail(c, BT_ERR_ARG, "%s: gates need wg (16-byte aligned), bg and 1 <= heads <= C / 32; no gates, heads 0", fn);
  HookArray xn(xn_dev, M * C, true);
  return run_hook(c, fn, stream, {&xn}, [&](cudaStream_t st) {
    launch_norm(x_dev, tc ? xn.h16.get() : static_cast<void*>(xn_dev), M, C, tc ? 1 : 0, st, gates_dev, wg_dev, bg_dev,
                heads);
    return check_launch(c, "debug_norm", st);
  });
}

int bt_debug_fused_qkv(bt_ctx* c, const float* x_dev, const float* wqkv_dev, const float* wg_dev, const float* bg_dev,
                       const float* rope_cos_dev, const float* rope_sin_dev, float* qkv_dev, float* gates_dev, int64_t M,
                       int32_t C, int32_t L, int32_t F, int32_t posmode, float qscale, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_debug_fused_qkv";
  if (c->dtype != BT_DTYPE_H16) return fail(c, BT_ERR_ARG, "%s: the fused kernel runs in the 16-bit context only", fn);
  if (!x_dev || !wqkv_dev || !wg_dev || !bg_dev || !rope_cos_dev || !rope_sin_dev || !qkv_dev || !gates_dev ||
      !aligned16(x_dev) || !aligned16(wg_dev))
    return fail(c, BT_ERR_ARG, "%s: null argument, or x / wg not 16-byte aligned", fn);
  if (M < 1 || (C != 32 && C != 64) || L < 1 || L > BT_CHUNK || (posmode != 0 && posmode != 1) ||
      (posmode == 1 && (F < 1 || F > BT_CHUNK)))
    return fail(c, BT_ERR_ARG, "%s: need M >= 1, C in {32, 64}, 1 <= L <= %d, posmode 0 or 1 (1: 1 <= F <= %d)", fn,
                BT_CHUNK, BT_CHUNK);
  HookArray wqkv(wqkv_dev, 3 * C * C), qkv(qkv_dev, M * 3 * C, true);
  return run_hook(c, fn, stream, {&wqkv, &qkv}, [&](cudaStream_t st) {
    QkvPlan p;
    const int r = make_plan(c, fn, p, [&](char* err, int n) { return tc_qkv_plan_create(wqkv.h16.get(), C, M, err, n); });
    if (r != BT_OK) return r;
    launch_fused_qkv(p.get(), x_dev, wg_dev, bg_dev, rope_cos_dev, rope_sin_dev, qkv.h16.get(), gates_dev, L, F, posmode,
                     qscale, st);
    return check_launch(c, "debug_fused_qkv", st);
  });
}

int bt_debug_fused_ff(bt_ctx* c, float* x_dev, const float* w1_dev, const float* b1_dev, const float* w2_dev,
                      const float* b2_dev, const float* o_dev, const float* wout_dev, float* xb_dev, int64_t M, int32_t C,
                      void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_debug_fused_ff";
  if (c->dtype != BT_DTYPE_H16) return fail(c, BT_ERR_ARG, "%s: the fused kernel runs in the 16-bit context only", fn);
  if (!x_dev || !w1_dev || !b1_dev || !w2_dev || !b2_dev || !aligned16(x_dev) || !aligned16(b1_dev) ||
      !aligned16(b2_dev) || !o_dev != !wout_dev)
    return fail(c, BT_ERR_ARG, "%s: null argument, x / b1 / b2 not 16-byte aligned, or only one of o and wout", fn);
  if (M < 1 || (C != 32 && C != 64)) return fail(c, BT_ERR_ARG, "%s: need M >= 1 and C in {32, 64}", fn);
  HookArray w1(w1_dev, 4 * C * C), w2(w2_dev, 4 * C * C), o(o_dev, M * C), wout(wout_dev, C * C), xb(xb_dev, M * C, true);
  return run_hook(c, fn, stream, {&w1, &w2, &o, &wout, &xb}, [&](cudaStream_t st) {
    FfPlan p;
    const int r = make_plan(c, fn, p, [&](char* err, int n) {
      return tc_ff_plan_create(w1.h16.get(), w2.h16.get(), C, M, o.h16.get(), wout.h16.get(), err, n);
    });
    if (r != BT_OK) return r;
    launch_fused_ff(p.get(), x_dev, b1_dev, b2_dev, xb.h16.get(), st);
    return check_launch(c, "debug_fused_ff", st);
  });
}

int bt_debug_stem(bt_ctx* c, const float* spect_dev, int64_t spect_frames, const bt_debug_chunk* chunks_host,
                  int32_t n_chunks, int32_t L, const float* bn1_scale_dev, const float* bn1_shift_dev, const float* w_dev,
                  const float* bias_dev, float* out_dev, int64_t out_count, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_debug_stem";
  if (!spect_dev || !chunks_host || !bn1_scale_dev || !bn1_shift_dev || !w_dev || !bias_dev || !out_dev ||
      !aligned16(spect_dev) || !aligned16(out_dev))
    return fail(c, BT_ERR_ARG, "%s: null argument, or spect / out not 16-byte aligned (float4 loads and stores)", fn);
  if (n_chunks < 1 || n_chunks > 65535 || L < 1 || L > kMaxChunkCap)
    return fail(c, BT_ERR_ARG, "%s: need 1 <= n_chunks <= 65535 and 1 <= L <= %lld", fn, (long long)kMaxChunkCap);
  for (int32_t i = 0; i < n_chunks; ++i) {
    const bt_debug_chunk& k = chunks_host[i];
    if (k.T < 1 || k.len < 1 || k.len > L || k.frame_base < 0 || k.frame_base > spect_frames - k.T)
      return fail(c, BT_ERR_ARG, "%s: chunk %d needs T >= 1, 1 <= len <= L and its clip inside the %lld spectrogram "
                  "frames", fn, i, (long long)spect_frames);
  }
  if (out_count < static_cast<int64_t>(n_chunks) * 32 * L * 32)
    return fail(c, BT_ERR_ARG, "%s: out holds %lld floats, fewer than n_chunks * 32 * L * 32", fn, (long long)out_count);
  return run_chunk_hook(c, fn, "stem", chunks_host, n_chunks, stream, [&](const ChunkSrc* t, cudaStream_t st) {
    launch_stem(spect_dev, t, n_chunks, L, bn1_scale_dev, bn1_shift_dev, w_dev, bias_dev, out_dev, st);
  });
}

int bt_debug_zero_tail(bt_ctx* c, void* buf_dev, int32_t elem_bytes, const bt_debug_chunk* chunks_host,
                       int32_t n_chunks, int32_t F, int32_t L, int32_t C, int64_t buf_bytes, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_debug_zero_tail";
  if (!buf_dev || !chunks_host || !aligned16(buf_dev))
    return fail(c, BT_ERR_ARG, "%s: null argument, or buf not 16-byte aligned", fn);
  if ((elem_bytes != 2 && elem_bytes != 4) || C < 1 || (static_cast<int64_t>(C) * elem_bytes) % 16 != 0 ||
      n_chunks < 1 || F < 1 || static_cast<int64_t>(n_chunks) * F > INT32_MAX || L < 1 || L > kMaxChunkCap)
    return fail(c, BT_ERR_ARG, "%s: need elem_bytes 2 or 4, C * elem_bytes a multiple of 16, n_chunks, F >= 1 with "
                "n_chunks * F < 2^31 and 1 <= L <= %lld", fn, (long long)kMaxChunkCap);
  for (int32_t i = 0; i < n_chunks; ++i)
    if (chunks_host[i].len < 1 || chunks_host[i].len > L)
      return fail(c, BT_ERR_ARG, "%s: chunk %d has len %d outside [1, L]", fn, i, chunks_host[i].len);
  if (buf_bytes / elem_bytes / C / L / F < n_chunks)
    return fail(c, BT_ERR_ARG, "%s: buf holds %lld bytes, fewer than n_chunks * F * L * C elements", fn,
                (long long)buf_bytes);
  return run_chunk_hook(c, fn, "zero_tail", chunks_host, n_chunks, stream, [&](const ChunkSrc* t, cudaStream_t st) {
    launch_zero_tail(buf_dev, elem_bytes, t, n_chunks, F, L, C, st);
  });
}

int bt_debug_head(bt_ctx* c, const float* x_dev, int32_t D, const float* w_dev, const float* b_dev,
                  const bt_debug_chunk* chunks_host, int32_t n_chunks, int32_t L, int32_t sum_head, float* beat_dev,
                  float* down_dev, int64_t out_count, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_debug_head";
  if (!x_dev || !w_dev || !b_dev || !chunks_host || !beat_dev || !down_dev)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  if (D < 64 || D > 1024 || D % 64 != 0 || n_chunks < 1 || L < 1 || static_cast<int64_t>(n_chunks) * L > INT32_MAX)
    return fail(c, BT_ERR_ARG, "%s: need D a multiple of 64 in [64, 1024], n_chunks, L >= 1 and n_chunks * L < 2^31", fn);
  for (int32_t i = 0; i < n_chunks; ++i) {
    const bt_debug_chunk& k = chunks_host[i];
    if (k.write_lo < 0 || k.write_lo > k.write_hi || k.write_hi > L)
      return fail(c, BT_ERR_ARG, "%s: chunk %d owns [%d, %d), not inside [0, L]", fn, i, k.write_lo, k.write_hi);
    const int64_t first = k.out_base + k.start + k.write_lo, last = k.out_base + k.start + k.write_hi - 1;
    if (k.write_lo < k.write_hi && (first < 0 || last >= out_count))
      return fail(c, BT_ERR_ARG, "%s: chunk %d writes frames [%lld, %lld], outside [0, %lld)", fn, i, (long long)first,
                  (long long)last, (long long)out_count);
  }
  return run_chunk_hook(c, fn, "head", chunks_host, n_chunks, stream, [&](const ChunkSrc* t, cudaStream_t st) {
    launch_head(x_dev, D, w_dev, b_dev, t, n_chunks, L, beat_dev, down_dev, sum_head ? 1 : 0, st);
  });
}

int bt_debug_attention_backward(bt_ctx* c, const float* qkv_dev, const float* gates_dev, const float* freqs_dev,
                                const float* dy_dev, int32_t seqs, int32_t n, int32_t heads, float* y_dev,
                                float* dqkv_dev, float* dgates_dev, void* stream) {
  const char* fn = "bt_debug_attention_backward";
  if (!c) return BT_ERR_ARG;
  if (c->dtype != BT_DTYPE_F32) return fail(c, BT_ERR_ARG, "%s: the training kernels run on a BT_DTYPE_F32 context", fn);
  if (!qkv_dev || !gates_dev || !freqs_dev || !dy_dev || !y_dev || !dqkv_dev || !dgates_dev)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  if (seqs < 1 || n < 1 || heads < 1 || heads > 32 || int64_t{seqs} * n > kMaxChunkCap)
    return fail(c, BT_ERR_ARG, "%s: bad geometry", fn);
  const int C = heads * 32;
  const int64_t M = int64_t{seqs} * n;
  const TrSeqs q{seqs, n, heads, 1, n, 0, 1};
  DeviceBuffer<float> qkv, o, dg, lse, delta;
  return run_hook(c, fn, stream, {}, [&](cudaStream_t st) {
    BT_CUDA(c, qkv.alloc(M * 3 * C * sizeof(float)));
    BT_CUDA(c, o.alloc(M * C * sizeof(float)));
    BT_CUDA(c, dg.alloc(M * C * sizeof(float)));
    BT_CUDA(c, lse.alloc(M * heads * sizeof(float)));
    BT_CUDA(c, delta.alloc(M * heads * sizeof(float)));
    BT_CUDA(c, cudaMemcpyAsync(qkv.get(), qkv_dev, M * 3 * C * sizeof(float), cudaMemcpyDeviceToDevice, st));
    BT_CUDA(c, cudaMemcpyAsync(dg.get(), dy_dev, M * C * sizeof(float), cudaMemcpyDeviceToDevice, st));
    launch_tr_rope(qkv.get(), freqs_dev, M, C, n, 1, 0, false, st);
    BT_LAUNCHED(c, "train_rope", st);
    launch_tr_attn_fwd(qkv.get(), q, o.get(), lse.get(), st);
    BT_LAUNCHED(c, "train_attention", st);
    launch_tr_gate_fwd(o.get(), gates_dev, M, C, y_dev, st);
    BT_LAUNCHED(c, "train_gate", st);
    launch_tr_gate_bwd(dg.get(), o.get(), gates_dev, M, C, dgates_dev, delta.get(), st);
    BT_LAUNCHED(c, "train_gate_bwd", st);
    launch_tr_attn_dq(qkv.get(), dg.get(), lse.get(), delta.get(), q, dqkv_dev, st);
    BT_LAUNCHED(c, "train_attention_dq", st);
    launch_tr_attn_dkv(qkv.get(), dg.get(), lse.get(), delta.get(), q, dqkv_dev, st);
    BT_LAUNCHED(c, "train_attention_dkv", st);
    launch_tr_rope(dqkv_dev, freqs_dev, M, C, n, 1, 0, true, st);
    BT_LAUNCHED(c, "train_rope", st);
    return BT_OK;
  });
}

}  // extern "C"

namespace {

// 1 + the largest offset sum_i (n_i - 1) stride_i of an array walked over dims n_i >= 1 with strides >= 0; -1 when it
// does not fit in int64 (no array is that long)
int64_t extent(std::initializer_list<std::pair<int64_t, int64_t>> dims) {
  int64_t e = 1;
  for (const auto& d : dims) {
    int64_t t;
    if (__builtin_mul_overflow(d.first - 1, d.second, &t) || __builtin_add_overflow(e, t, &e)) return -1;
  }
  return e;
}

// The slots of one bt_debug_train_kernel call.  need(i, n, ...) checks slot i against the n elements the op touches
// there and returns its pointer; the first failure is kept in `err` for the caller to report.
struct TrSlots {
  float* const* p;
  const int64_t* cnt;
  int32_t n;
  std::string err;
  float* need(int i, int64_t elems, bool required = true, bool align = false) {
    float* a = i < n ? p[i] : nullptr;
    if (!err.empty()) return a;
    if (!a) {
      if (required) err = "slot " + std::to_string(i) + " is NULL";
    } else if (elems < 0 || cnt[i] < elems) {
      err = "slot " + std::to_string(i) + " holds " + std::to_string(cnt[i]) + " elements, the op touches " +
            (elems < 0 ? std::string("more than 2^63") : std::to_string(elems));
    } else if (align && reinterpret_cast<uintptr_t>(a) % 16 != 0) {
      err = "slot " + std::to_string(i) + " is not 16-byte aligned (float4 access)";
    }
    return a;
  }
  bool present(int i) const { return i < n && p[i]; }
};

constexpr int64_t kMaxGrid1 = int64_t{INT32_MAX};  // gridDim.x
constexpr int64_t kMaxElems = kMaxGrid1 * 256;     // elementwise launches of 256 threads per element block

}  // namespace

extern "C" {

int bt_debug_train_kernel(bt_ctx* c, const bt_debug_train_desc* d, float* const* arrays_dev, const int64_t* counts,
                          int32_t n_arrays, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_debug_train_kernel";
  if (c->dtype != BT_DTYPE_F32) return fail(c, BT_ERR_ARG, "%s: the training kernels run on a BT_DTYPE_F32 context", fn);
  if (!d || n_arrays < 0 || (n_arrays > 0 && (!arrays_dev || !counts)))
    return fail(c, BT_ERR_ARG, "%s: null descriptor or array table", fn);
  TrSlots s{arrays_dev, counts, n_arrays, {}};
  const int64_t M = d->M;
  const int C = d->C;
  const auto bad = [&](const char* what) { return fail(c, BT_ERR_ARG, "%s: op %d: %s", fn, d->op, what); };
  const auto slots = [&]() { return s.err.empty() ? BT_OK : fail(c, BT_ERR_ARG, "%s: op %d: %s", fn, d->op, s.err.c_str()); };
  const auto elementwise = [&](int64_t n) { return n >= 1 && n <= kMaxElems; };
  // the BatchNorm of C channels in slots i .. i + 3
  const auto bn_at = [&](int i, int64_t ch, bool required = true) {
    return TrBn{s.need(i, ch, required), s.need(i + 1, ch, required), s.need(i + 2, ch, required),
                s.need(i + 3, ch, required)};
  };
  const auto hook = [&](auto launch) { return run_hook(c, fn, stream, {}, launch); };
  if (!(d->p >= 0.f && d->p < 1.f) || d->e0 < 0) return bad("need a dropout rate in [0, 1) and e0 >= 0");
  const TrDrop drop = tr_drop(d->seed, d->site, d->p, d->e0);

  switch (d->op) {
    case BT_TRAIN_GEMM: {
      const int Mi = static_cast<int>(M), N = d->N, K = d->K;
      if (M < 1 || M > INT32_MAX || N < 1 || K < 1 || d->a_rs < 0 || d->a_cs < 0 || d->b_rs < 0 || d->b_cs < 0 ||
          d->ldc < N || d->splits < 0 || (N + 63) / 64 > 65535)
        return bad("need 1 <= M < 2^31, N, K >= 1 (N <= 65535 * 64), strides >= 0, ldc >= N and splits >= 0");
      const int splits = d->splits ? d->splits : tr_dw_splits(K, Mi, N);
      const int parts = tr_gemm_parts(K, splits);
      const TrMat A{s.need(0, extent({{M, d->a_rs}, {K, d->a_cs}})), d->a_rs, d->a_cs};
      const TrMat Bm{s.need(1, extent({{N, d->b_rs}, {K, d->b_cs}})), d->b_rs, d->b_cs};
      float* Cp = s.need(2, extent({{M, d->ldc}, {N, 1}}));
      const float* bias = s.need(3, N, false);
      if (s.present(4) && d->ldr < N) return bad("resid needs ldr >= N");
      const float* resid = s.need(4, extent({{M, d->ldr}, {N, 1}}), false);
      float* gelu = s.need(5, extent({{M, d->ldc}, {N, 1}}), false);
      if (splits > 1 && (bias || resid || gelu || drop.thresh))
        return bad("a split GEMM takes no bias, resid, gelu_out or dropout");
      if (parts > 65535) return bad("more than 65535 K parts");
      if (parts > 1 && d->ldc != N) return bad("a GEMM of several K parts needs ldc = N (tr_reduce writes rows of N)");
      int64_t part_n = 0;
      if (parts > 1 && __builtin_mul_overflow(int64_t{parts} * N, M, &part_n)) part_n = -1;
      float* part = s.need(6, part_n, parts > 1);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        const TrGemmOut o{parts > 1 ? part : Cp, d->ldc, M * N, bias, resid, d->ldr, gelu, drop};
        launch_tr_gemm(A, Bm, o, Mi, N, K, splits, st);
        BT_LAUNCHED(c, "train_gemm", st);
        if (parts == 1) return BT_OK;
        launch_tr_reduce(part, parts, M * N, d->scale, Cp, st);
        return check_launch(c, "train_reduce", st);
      });
    }
    case BT_TRAIN_REDUCE: {
      if (!elementwise(M) || d->splits < 1 || d->splits > 65535)
        return bad("need 1 <= M <= 2^31 * 256 elements and 1 <= splits <= 65535 parts");
      const float* part = s.need(0, d->splits * M);
      float* out = s.need(1, M);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_reduce(part, d->splits, M, d->scale, out, st, d->beta, drop);
        return check_launch(c, "train_reduce", st);
      });
    }
    case BT_TRAIN_COLSUM: {
      const int N = d->N;
      if (M < 1 || N < 1 || d->splits < 0 || (N + 31) / 32 > kMaxGrid1)
        return bad("need M, N >= 1 and splits >= 0");
      const int splits = d->splits ? d->splits : tr_colsum_splits(M, N);
      const int64_t rps = (M + std::max(splits, 1) - 1) / std::max(splits, 1), parts = (M + rps - 1) / rps;
      if (splits < 1 || parts > 65535) return bad("the split gives no part or more than 65535 parts");
      const float* A = s.need(0, M * N);
      const float* Bm = s.need(1, M * N, false);
      const float* rs = s.need(2, M, false);
      float* part = s.need(3, parts * N);
      float* out = s.need(4, N);
      const float* shift = s.need(5, N, false);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        const int z = launch_tr_colsum(A, Bm, rs, M, N, splits, part, st, shift);
        BT_LAUNCHED(c, "train_colsum", st);
        launch_tr_reduce(part, z, N, d->scale, out, st);
        return check_launch(c, "train_reduce", st);
      });
    }
    case BT_TRAIN_RMS_FWD:
    case BT_TRAIN_RMS_BWD: {
      if (M < 1 || (M + 7) / 8 > kMaxGrid1 || C < 1) return bad("need M >= 1 rows (M / 8 < 2^31) and C >= 1");
      if (d->op == BT_TRAIN_RMS_FWD) {
        const float* x = s.need(0, M * C);
        const float* gamma = s.need(1, C);
        float* xn = s.need(2, M * C);
        float* inv = s.need(3, M);
        if (const int r = slots()) return r;
        return hook([&](cudaStream_t st) {
          launch_tr_rms_fwd(x, gamma, M, C, xn, inv, st);
          return check_launch(c, "train_rmsnorm", st);
        });
      }
      const float* dxn = s.need(0, M * C);
      const float* x = s.need(1, M * C);
      const float* inv = s.need(2, M);
      const float* gamma = s.need(3, C);
      float* dres = s.need(4, M * C);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_rms_bwd(dxn, x, inv, gamma, M, C, d->flag != 0, dres, st);
        return check_launch(c, "train_rmsnorm_bwd", st);
      });
    }
    case BT_TRAIN_BN_GELU_FWD:
    case BT_TRAIN_BN_GELU_BWD:
    case BT_TRAIN_BN_SCALE: {
      if (!elementwise(M) || C < 1) return bad("need 1 <= M <= 2^31 * 256 elements and C >= 1 channels");
      if (d->op == BT_TRAIN_BN_GELU_FWD) {
        const float* z = s.need(0, M);
        const TrBn b = bn_at(1, C);
        float* y = s.need(5, M);
        if (const int r = slots()) return r;
        return hook([&](cudaStream_t st) {
          launch_tr_bn_gelu_fwd(z, b, M, C, y, st);
          return check_launch(c, "train_bn_gelu", st);
        });
      }
      if (d->op == BT_TRAIN_BN_SCALE) {
        const float* g = s.need(0, M);
        const TrBn b = bn_at(1, C);
        float* dx = s.need(5, M);
        const bool batch = s.present(6);
        if (batch && d->bn_n < 1) return bad("batch statistics need bn_n >= 1 positions");
        const TrBnBatch bb{s.need(6, M, false), s.need(7, C, batch), s.need(8, C, batch),
                           static_cast<float>(1.0 / static_cast<double>(std::max<int64_t>(d->bn_n, 1)))};
        if (const int r = slots()) return r;
        return hook([&](cudaStream_t st) {
          launch_tr_bn_scale(g, b, M, C, dx, st, batch ? &bb : nullptr);
          return check_launch(c, "train_bn_scale", st);
        });
      }
      const float* dy = s.need(0, M);
      const float* z = s.need(1, M);
      const TrBn b = bn_at(2, C);
      float* dbn = s.need(6, M);
      float* dz = s.need(7, M);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_bn_gelu_bwd(dy, z, b, M, C, dbn, dz, st);
        return check_launch(c, "train_bn_gelu_bwd", st);
      });
    }
    case BT_TRAIN_BN_GRADS: {
      if (C < 1) return bad("need C >= 1");
      const float* sgz = s.need(0, C);
      const float* sg = s.need(1, C);
      const TrBn b = bn_at(2, C);
      float* dw = s.need(6, C, false);
      float* db = s.need(7, C, false);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_bn_grads(sgz, sg, b, C, dw, db, st);
        return check_launch(c, "train_bn_grads", st);
      });
    }
    case BT_TRAIN_GELU_BWD: {
      if (!elementwise(M)) return bad("need 1 <= M <= 2^31 * 256 elements");
      const float* da = s.need(0, M);
      const float* h = s.need(1, M);
      float* dh = s.need(2, M);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_gelu_bwd(da, h, M, dh, st, drop);
        return check_launch(c, "train_gelu_bwd", st);
      });
    }
    case BT_TRAIN_IM2COL:
    case BT_TRAIN_COL2IM: {
      if (d->B < 1 || d->F < 1 || d->S < 1 || d->L < 1 || C < 1 || d->sb < 0 || d->sf < 0 || d->st < 0 || d->sc < 0 ||
          int64_t{C} * d->S * 3 > INT32_MAX || int64_t{d->F} * d->S > INT32_MAX)
        return bad("need B, F, S, L, C >= 1, C S 3 and F S < 2^31, and strides >= 0");
      const TrImg g{d->B, d->F, d->S, d->L, C, d->sb, d->sf, d->st, d->sc};
      const int64_t in_n = extent({{d->B, d->sb}, {int64_t{d->F} * d->S, d->sf}, {d->L, d->st}, {C, d->sc}});
      const int64_t col_n = int64_t{d->B} * d->F * d->L * C * d->S * 3;
      if (!elementwise(col_n)) return bad("more than 2^31 * 256 im2col elements");
      if (d->op == BT_TRAIN_IM2COL) {
        const float* in = s.need(0, in_n);
        float* col = s.need(1, col_n);
        const TrBn b = bn_at(2, int64_t{d->F} * d->S, d->flag != 0);
        if (const int r = slots()) return r;
        return hook([&](cudaStream_t st) {
          launch_tr_im2col(in, g, d->flag ? &b : nullptr, col, st);
          return check_launch(c, "train_im2col", st);
        });
      }
      const float* dcol = s.need(0, col_n);
      float* din = s.need(1, in_n);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_col2im(dcol, g, din, st);
        return check_launch(c, "train_col2im", st);
      });
    }
    case BT_TRAIN_CONCAT: {
      const int64_t n = int64_t{d->B} * d->F * d->L * C;
      if (d->B < 1 || d->F < 1 || d->L < 1 || C < 1 || int64_t{C} * d->F > INT32_MAX || !elementwise(n))
        return bad("need B, F, L, C >= 1, C F < 2^31 and B F L C <= 2^31 * 256");
      const float* src = s.need(0, n);
      float* dst = s.need(1, n);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_concat(src, d->B, d->F, d->L, C, d->flag != 0, dst, st);
        return check_launch(c, "train_concat", st);
      });
    }
    case BT_TRAIN_ROPE: {
      if (M < 1 || C < 32 || C % 32 != 0 || !elementwise(M * C) || d->L < 1 || (d->posmode != 0 && d->posmode != 1) ||
          (d->posmode == 1 && d->F < 1))
        return bad("need M >= 1, C a multiple of 32, M C <= 2^31 * 256, L >= 1 and posmode 0 or 1 (1: F >= 1)");
      float* qkv = s.need(0, M * 3 * C);
      const float* freqs = s.need(1, 16);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_rope(qkv, freqs, M, C, d->L, d->F, d->posmode, d->flag != 0, st);
        return check_launch(c, "train_rope", st);
      });
    }
    case BT_TRAIN_GATE_FWD:
    case BT_TRAIN_GATE_BWD: {
      if (M < 1 || C < 32 || C % 32 != 0 || !elementwise(M * C))
        return bad("need M >= 1, C a multiple of 32 and M C <= 2^31 * 256");
      const int64_t heads = M * (C / 32);
      if (d->op == BT_TRAIN_GATE_FWD) {
        const float* O = s.need(0, M * C);
        const float* g = s.need(1, heads);
        float* G = s.need(2, M * C);
        if (const int r = slots()) return r;
        return hook([&](cudaStream_t st) {
          launch_tr_gate_fwd(O, g, M, C, G, st);
          return check_launch(c, "train_gate", st);
        });
      }
      float* dG = s.need(0, M * C);
      const float* O = s.need(1, M * C);
      const float* g = s.need(2, heads);
      float* dg = s.need(3, heads);
      float* delta = s.need(4, heads);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_gate_bwd(dG, O, g, M, C, dg, delta, st);
        return check_launch(c, "train_gate_bwd", st);
      });
    }
    case BT_TRAIN_HEAD_FWD:
    case BT_TRAIN_HEAD_BWD: {
      if (!elementwise(M)) return bad("need 1 <= M <= 2^31 * 256 rows");
      if (d->op == BT_TRAIN_HEAD_FWD) {
        const float* o = s.need(0, 2 * M);
        float* beat = s.need(1, M);
        float* down = s.need(2, M);
        if (const int r = slots()) return r;
        return hook([&](cudaStream_t st) {
          launch_tr_head_fwd(o, M, d->flag != 0, beat, down, st);
          return check_launch(c, "train_head", st);
        });
      }
      const float* dbeat = s.need(0, M);
      const float* ddown = s.need(1, M);
      float* dout = s.need(2, 2 * M);
      if (const int r = slots()) return r;
      return hook([&](cudaStream_t st) {
        launch_tr_head_bwd(dbeat, ddown, M, d->flag != 0, dout, st);
        return check_launch(c, "train_head", st);
      });
    }
    case BT_TRAIN_ATTN_FWD:
    case BT_TRAIN_ATTN_DQ:
    case BT_TRAIN_ATTN_DKV: {
      const TrSeqs q{d->seqs, d->n, d->heads, d->seq_in, d->s_out, d->s_in, d->s_pos};
      if (q.seqs < 1 || q.n < 1 || q.heads < 1 || q.heads > 65535 || q.seq_in < 1 || q.s_out < 0 || q.s_in < 0 ||
          q.s_pos < 0 || int64_t{q.seqs} * ((q.n + 63) / 64) > kMaxGrid1)
        return bad("need seqs, n, seq_in >= 1, 1 <= heads <= 65535, strides >= 0 and seqs ceil(n / 64) < 2^31");
      // the largest token row: the last sequence, or the last of the sequence block before it
      const int64_t ql = (q.seqs - 1) / q.seq_in, rl = (q.seqs - 1) % q.seq_in;
      int64_t r0 = extent({{ql + 1, q.s_out}, {rl + 1, q.s_in}});
      if (ql > 0) r0 = std::max(r0, extent({{ql, q.s_out}, {q.seq_in, q.s_in}}));
      const int64_t rows = r0 < 0 ? -1 : extent({{r0, 1}, {q.n, q.s_pos}});
      const int64_t Cq = int64_t{q.heads} * 32;
      const auto n_of = [&](int64_t per_row) {  // elements of an array of `rows` rows of per_row
        int64_t e;
        return rows < 0 || __builtin_mul_overflow(rows, per_row, &e) ? -1 : e;
      };
      const float* qkv = s.need(0, n_of(3 * Cq), true, true);
      if (d->op == BT_TRAIN_ATTN_FWD) {
        float* O = s.need(1, n_of(Cq), true, true);
        float* lse = s.need(2, n_of(q.heads));
        if (const int r = slots()) return r;
        return hook([&](cudaStream_t st) {
          launch_tr_attn_fwd(qkv, q, O, lse, st, drop);
          return check_launch(c, "train_attention", st);
        });
      }
      const float* dO = s.need(1, n_of(Cq), true, true);
      const float* lse = s.need(2, n_of(q.heads));
      const float* delta = s.need(3, n_of(q.heads));
      float* dqkv = s.need(4, n_of(3 * Cq), true, true);
      if (const int r = slots()) return r;
      const bool dq = d->op == BT_TRAIN_ATTN_DQ;
      return hook([&](cudaStream_t st) {
        if (dq) launch_tr_attn_dq(qkv, dO, lse, delta, q, dqkv, st, drop);
        else launch_tr_attn_dkv(qkv, dO, lse, delta, q, dqkv, st, drop);
        return check_launch(c, dq ? "train_attention_dq" : "train_attention_dkv", st);
      });
    }
    default:
      return bad("unknown op");
  }
}

}  // extern "C"
