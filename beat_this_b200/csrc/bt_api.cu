// C ABI (include/beatthis.h): context, packed-parameter registry, chunk planner, workspace and the per-wave schedule
// of the BeatThis forward pass (reference beat_this/model/beat_tracker.py:188-192), and the runtime all entry files
// share (api_internal.h): errors, launch checks, the entry prologue, offsets checks, staging ring and profiler.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "api_internal.h"

static char g_create_error[512] = "";

static int prof_event(bt_ctx* c, cudaStream_t st) {
  if (c->ev_used == c->ev_pool.size()) {
    cudaEvent_t ev;
    if (cudaEventCreate(&ev) != cudaSuccess) return -1;
    c->ev_pool.emplace_back(ev);
  }
  const int idx = static_cast<int>(c->ev_used++);
  cudaEventRecord(c->ev_pool[idx].get(), st);
  return idx;
}

static void prof_launch(bt_ctx* c, const char* what, cudaStream_t st) {
  int kind = -1;
  for (size_t i = 0; i < c->prof_names.size(); ++i)
    if (c->prof_names[i] == what) { kind = static_cast<int>(i); break; }
  if (kind < 0) {
    kind = static_cast<int>(c->prof_names.size());
    c->prof_names.push_back(what);
    c->prof_ms.push_back(0.0);
    c->prof_cnt.push_back(0);
  }
  const int ev = prof_event(c, st);
  if (ev >= 0 && c->prof_prev >= 0) c->prof_recs.push_back({kind, ev, c->prof_prev});
  c->prof_prev = ev;
}

int bt::fail(const bt_ctx* c, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  if (c) vsnprintf(c->err, sizeof(c->err), fmt, ap);
  else vsnprintf(g_create_error, sizeof(g_create_error), fmt, ap);
  va_end(ap);
  return code;
}

int bt::enter(bt_ctx* c, const char* fn, void* stream, cudaStream_t* st) {
  *st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  c->call = fn;
  if (c->prof) c->prof_prev = prof_event(c, *st);
  return BT_OK;
}

int bt::check_launch(bt_ctx* c, const char* what, cudaStream_t st, cudaError_t status) {
  if (status == cudaSuccess) {
    c->launches++;
    if (c->prof) prof_launch(c, what, st);
  }
  cudaError_t e = cudaGetLastError();  // also clears the error a failed host step leaves behind
  if (status != cudaSuccess) e = status;
  else if (e == cudaSuccess && c->sync_debug) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(c, BT_ERR_CUDA, "%s: kernel %s failed: %s", c->call, what, cudaGetErrorString(e));
  return BT_OK;
}

int bt::check_offsets(const bt_ctx* c, const char* fn, const char* name, const int64_t* off, int32_t n,
                      OffsetsStart start) {
  if (start == kFromZero ? off[0] != 0 : off[0] < 0)
    return fail(c, BT_ERR_ARG, "%s: %s must start at %s", fn, name, start == kFromZero ? "0" : ">= 0");
  for (int i = 0; i < n; ++i)
    if (off[i + 1] < off[i]) return fail(c, BT_ERR_ARG, "%s: %s must not decrease", fn, name);
  return BT_OK;
}

int bt::check_stft_frames(const bt_ctx* c, const char* fn, const int64_t* sample_off, const int64_t* frame_off,
                          int32_t n, int n_fft, int hop) {
  int r = check_offsets(c, fn, "sample_offsets_host", sample_off, n, kFromNonNegative);
  if (r != BT_OK || (r = check_offsets(c, fn, "frame_offsets_host", frame_off, n, kFromZero)) != BT_OK) return r;
  for (int i = 0; i < n; ++i) {
    const int64_t len = sample_off[i + 1] - sample_off[i];
    if (len <= n_fft / 2)
      return fail(c, BT_ERR_ARG, "%s: clip %d has %lld samples; reflect padding needs more than %d (torch.stft raises "
                  "for such input as well)", fn, i, (long long)len, n_fft / 2);
    if (frame_off[i + 1] - frame_off[i] != 1 + len / hop)
      return fail(c, BT_ERR_ARG, "%s: frame_offsets do not match 1 + len/%d for clip %d", fn, hop, i);
  }
  return BT_OK;
}

const Param* bt::find_param(const bt_ctx* c, const std::string& name) {
  auto it = c->params.find(name);
  return it == c->params.end() ? nullptr : &it->second;
}

int bt::acquire_stage(bt_ctx* c, size_t bytes, StageSlot** out) {
  StageSlot* sl = &c->stage[c->stage_next];
  c->stage_next = (c->stage_next + 1) % kStageSlots;
  if (sl->pending) {  // kStageSlots uploads ago: long finished unless the caller is that far ahead of the GPU
    BT_CUDA(c, cudaEventSynchronize(sl->ev.get()));
    sl->pending = false;
  }
  if (!sl->ev) {
    cudaEvent_t ev;
    BT_CUDA(c, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    sl->ev.reset(ev);
  }
  const size_t cap = std::max<size_t>(bytes * 2, 1 << 16);
  BT_CUDA(c, sl->host.reserve(bytes, cap));
  BT_CUDA(c, sl->dev.reserve(bytes, cap));
  *out = sl;
  return BT_OK;
}

int bt::upload_stage(bt_ctx* c, StageSlot* sl, size_t bytes, cudaStream_t st) {
  BT_CUDA(c, cudaMemcpyAsync(sl->dev.get(), sl->host.get(), bytes, cudaMemcpyHostToDevice, st));
  BT_CUDA(c, cudaEventRecord(sl->ev.get(), st));
  sl->pending = true;
  return BT_OK;
}

std::vector<Step> bt::model_steps(const bt_hparams& hp) {
  std::vector<Step> v;
  int C = hp.stem_dim, F = hp.spect_dim / 4;
  v.push_back({kStem, C, F, 0, "stem", "frontend.stem"});
  for (int i = 0; i < 3; ++i) {
    const std::string b = "b" + std::to_string(i), m = "frontend.blocks." + std::to_string(i);
    if (hp.partial_transformers) {
      v.push_back({kAttnFreq, C, F, 0, b + ".attnF", m + ".partial.attnF"});
      v.push_back({kFfn, C, F, 4, b + ".ffF", m + ".partial.ffF"});
      v.push_back({kAttnTime, C, F, 0, b + ".attnT", m + ".partial.attnT"});
      v.push_back({kFfn, C, F, 4, b + ".ffT", m + ".partial.ffT"});
    }
    v.push_back({kConv, C, F, 0, b + ".conv", m});
    C *= 2;
    F /= 2;
  }
  v.push_back({kLinear, C, F, 0, "lin", "frontend.linear"});
  const int D = hp.transformer_dim;
  for (int i = 0; i < hp.n_layers; ++i) {
    const std::string b = "l" + std::to_string(i), m = "transformer_blocks.layers." + std::to_string(i);
    v.push_back({kAttnTime, D, 1, 0, b + ".attn", m + ".0"});
    v.push_back({kFfn, D, 1, hp.ff_mult, b + ".ff", m + ".1"});
  }
  v.push_back({kHead, D, 1, 0, "head", ""});
  return v;
}

namespace {

constexpr bt_chunking kDefaultChunking{BT_CHUNK, BT_BORDER, BT_KEEP_FIRST};
bool chunking_valid(const bt_chunking* ck, int64_t max_chunk) {
  return ck && ck->chunk_size >= 1 && ck->chunk_size <= max_chunk && ck->border >= 0 &&
         2 * static_cast<int64_t>(ck->border) < ck->chunk_size &&
         (ck->overlap_mode == BT_KEEP_FIRST || ck->overlap_mode == BT_KEEP_LAST);
}

// The model entry points' state and chunking: a finalized ctx, and a valid ck up to its maximum chunk
int check_chunking(const bt_ctx* c, const char* fn, const bt_chunking* ck) {
  if (!c || !c->finalized) return fail(c, BT_ERR_STATE, "%s: context not finalized", fn);
  if (chunking_valid(ck, c->max_chunk)) return BT_OK;
  return fail(c, BT_ERR_ARG, "%s: need 1 <= chunk_size <= %d (bt_max_chunk), 0 <= 2 * border < chunk_size and "
              "overlap_mode BT_KEEP_FIRST or BT_KEEP_LAST", fn, c->max_chunk);
}

// The chunk plan of bt_plan_chunking (contract and coverage argument in include/beatthis.h) for a valid chunking:
// split_piece (reference inference.py:119-125) for the starts and lengths, aggregate_prediction (:174-184) for the
// owned piece frames [own_lo, own_hi).  Chunks are visited in order, so keep_first cuts a chunk's range where the
// previous one's ends and keep_last where the next one's begins.
int64_t plan_chunks(int64_t T, const bt_chunking& ck, int64_t* starts, int64_t* lens, int64_t* own_lo, int64_t* own_hi,
                    int64_t cap) {
  if (T <= 0) return 0;
  const int64_t c = ck.chunk_size, b = ck.border, step = c - 2 * b;
  const int64_t n = (T + step - 1) / step;  // the length of arange(-b, T - b, step)
  auto start = [&](int64_t i) { return i == n - 1 && T > step ? T - (c - b) : i * step - b; };
  auto len = [&](int64_t s) {
    const int64_t lo = std::max<int64_t>(s, 0), hi = std::min<int64_t>(s + c, T);
    const int64_t left = std::max<int64_t>(0, -s);
    const int64_t right = std::max<int64_t>(0, std::min<int64_t>(b, s + c - T));
    return (hi - lo) + left + right;
  };
  for (int64_t i = 0; i < std::min(n, cap); ++i) {
    const int64_t s = start(i), l = len(s);
    int64_t lo = s + b, hi = s + l - b;
    if (ck.overlap_mode == BT_KEEP_FIRST && i > 0) {
      const int64_t sp = start(i - 1);
      lo = std::max(lo, sp + len(sp) - b);
    } else if (ck.overlap_mode == BT_KEEP_LAST && i < n - 1) {
      hi = std::min(hi, start(i + 1) + b);
    }
    if (starts) starts[i] = s;
    if (lens) lens[i] = l;
    if (own_lo) own_lo[i] = lo;
    if (own_hi) own_hi[i] = std::max(lo, hi);
  }
  return n;
}

int64_t front_elems(const bt_ctx* c) {
  return static_cast<int64_t>(c->hp.spect_dim / 4) * c->hp.stem_dim;
}

// Padded frames a wave may hold: `wave` chunks of BT_CHUNK frames, or one chunk of the ctx's longest length
int64_t wave_frames(const bt_ctx* c) {
  return std::max<int64_t>(static_cast<int64_t>(c->wave) * BT_CHUNK, c->max_chunk);
}

int ensure_ws(bt_ctx* c) {
  // sized once for a full wave (bt_set_wave_chunks; ~46 MB per 1500 frames on the 16-bit path): growing later
  // would mean freeing and allocating device memory -- device-wide synchronisation -- amid a stream of batches
  const int want = c->wave;
  const int64_t frames = wave_frames(c);
  if (want <= c->ws.chunks && frames <= c->ws.frames) return BT_OK;
  c->ws = Workspace();  // the old blocks are freed before the new ones are allocated
  const int64_t fe = front_elems(c);                                     // 1024
  const int64_t D = c->hp.transformer_dim;
  const int64_t xe = frames * std::max(fe, D);                           // elements of the largest activation
  const size_t act = c->dtype == BT_DTYPE_H16 ? 2 : 4;
  Workspace& ws = c->ws;
  BT_CUDA(c, ws.X0.alloc(xe * 4));
  BT_CUDA(c, ws.X1.alloc(xe * 4));
  BT_CUDA(c, ws.GATES.alloc(frames * std::max(fe / 32, D / 32) * 4));
  BT_CUDA(c, ws.XN.alloc(xe * act));
  BT_CUDA(c, ws.QKV.alloc(3 * xe * act));
  BT_CUDA(c, ws.O.alloc(xe * act));
  BT_CUDA(c, ws.H.alloc(4 * xe * act));
  if (c->dtype == BT_DTYPE_H16) {
    BT_CUDA(c, ws.XB.alloc(xe * 2));
  }
  ws.chunks = want;
  ws.frames = frames;
  return BT_OK;
}

struct Wave {
  const ChunkSrc* chunks_dev;
  int nb;
  int L;         // padded length: the longest chunk of the wave
  bool varlen;   // some chunk is shorter than L
};

int do_tap(bt_ctx* c, const char* name, const void* buf, int64_t count, bool is_act, cudaStream_t st) {
  if (c->tap_name.empty() || !c->tap_out || c->tap_name != name) return BT_OK;
  if (count > c->tap_cap) return fail(c, BT_ERR_ARG, "tap %s needs %lld floats", name, (long long)count);
  if (is_act && c->dtype == BT_DTYPE_H16) {
    launch_h16_to_f32(buf, c->tap_out, count, st);
    BT_LAUNCHED(c, "tap_convert", st);
  } else {
    BT_CUDA(c, cudaMemcpyAsync(c->tap_out, buf, count * 4, cudaMemcpyDeviceToDevice, st));
  }
  c->tap_count = count;
  return BT_OK;
}

GemmShape plain_shape(int planes, int L, int N, int K, int lda) {
  GemmShape g{};
  g.planes_out = planes; g.L = L; g.N = N; g.Kslab = K; g.nslab = 1; g.plane_mul = 1; g.lda = lda;
  return g;
}

// A GEMM of layer l over a wave of nb chunks.  The GEMMs that add the residual (attention-out, FFN-down) are planned
// with the tile width of a residual epilogue.
int run_gemm(bt_ctx* c, const Layer& l, int nb, GemmPlan& plan, const void* A, const Param* W, const GemmShape& g,
             const EpiParams& e, const char* what, cudaStream_t st) {
  if (c->dtype == BT_DTYPE_H16) {
    const int r = make_plan(c, l.name.c_str(), plan, [&](char* err, int errlen) {
      return tc_gemm_plan_create(A, W->b16.get(), g, nb * l.F, e.resid != nullptr, e, err, errlen);
    });
    if (r != BT_OK) return r;
    launch_gemm_tc(plan.get(), st);
  } else {
    launch_gemm_simt(reinterpret_cast<const float*>(A), W->f32.get(), g, e, st);
  }
  BT_LAUNCHED(c, what, st);
  return BT_OK;
}

EpiParams epi_generic(const Param* bias, int gelu, const float* resid, int ldr, float* out_f32, int ldo32,
                      void* out_act, int ldoa) {
  EpiParams e{};
  e.kind = 0;
  e.bias = bias ? bias->f32.get() : nullptr;
  e.gelu = gelu;
  e.resid = resid; e.ldr = ldr;
  e.out_f32 = out_f32; e.ldo_f32 = ldo32;
  e.out_act = out_act; e.ldo_act = ldoa;
  return e;
}

bool is_attention(const Layer& l) { return l.kind == kAttnFreq || l.kind == kAttnTime; }

// sub-blocks of width C = 32 / 64 (the first two frontend blocks) run as one fused kernel each on the 16-bit path
bool fused(const Layer& l) { return (l.C == 32 || l.C == 64) && (l.kind != kFfn || l.mult == 4); }

// The out-projection + residual of attention layer i (before the head) run inside the fused FFN after it
// (fused_ff_kernel<C, true>) on the 16-bit path when the attention is a frontend one, unless a tap asks to see the
// residual stream between the two.
bool outproj_in_ff(const bt_ctx* c, size_t i) {
  const Layer& l = c->layers[i];
  return c->dtype == BT_DTYPE_H16 && is_attention(l) && l.F > 1 && c->layers[i + 1].kind == kFfn &&
         fused(c->layers[i + 1]) && c->tap_name != l.name;
}

// x += attention(x) over nb * F planes of L tokens with dim C (reference roformer.py:114-132).
// kAttnFreq: sequences run over the F planes of each chunk (PartialFTTransformer attnF).
int attention_block(bt_ctx* c, float* X, const Layer& l, LayerPlans& tp, int nb, int L, bool out_in_ff,
                    const ChunkSrc* vl_chunks, cudaStream_t st) {
  const Workspace& ws = c->ws;
  const bool tc = c->dtype == BT_DTYPE_H16;
  const bool freq = l.kind == kAttnFreq, front = l.F > 1;
  const int C = l.C, F = l.F, heads = C / kHeadDim, planes = nb * F;
  const Param *wqkv = l.w[0], *wg = l.w[1], *bg = l.w[2], *wout = l.w[3];
  const int64_t M = static_cast<int64_t>(planes) * L;
  const float inv_sqrt_d = 0.17677669529663687f;  // 1/sqrt(32): SDPA default scale (roformer.py:78-80)
  const float qscale = tc && !freq ? inv_sqrt_d * 1.4426950408889634f : 1.0f;
  int r = BT_OK;
  if (tc && fused(l)) {  // norm + gates + QKV + RoPE in one kernel
    r = make_plan(c, l.name.c_str(), tp.fqkv, [&](char* err, int n) {
      return tc_qkv_plan_create(wqkv->b16.get(), C, M, err, n);
    });
    if (r != BT_OK) return r;
    launch_fused_qkv(tp.fqkv.get(), X, wg->f32.get(), bg->f32.get(), c->rope_cos->f32.get(), c->rope_sin->f32.get(),
                     ws.QKV.get(), ws.GATES.get(), L, F, freq ? 1 : 0, qscale, st);
    BT_LAUNCHED(c, C == 32 ? "qkv_fused_c32" : "qkv_fused_c64", st);
  } else {
    // up to 2 heads (fp32 path only: the 16-bit path fuses those blocks): gates inside the norm kernel;
    // otherwise from a padded gates GEMM
    const bool gates_in_norm = heads <= 2;
    launch_norm(X, ws.XN.get(), M, C, tc, st, gates_in_norm ? ws.GATES.get() : nullptr, wg->f32.get(), bg->f32.get(),
                heads);
    BT_LAUNCHED(c, gates_in_norm ? "norm_gates" : (front ? "norm_front" : "norm"), st);
    if (!gates_in_norm) {  // gates = sigmoid(to_gates(x_normed)): a [heads -> 32 padded] x C GEMM on the same rows
      GemmShape gg = plain_shape(planes, L, 32, C, C);
      EpiParams eg{};
      eg.kind = 2;
      eg.bias = bg->f32.get();
      eg.heads = heads;
      eg.out_f32 = ws.GATES.get();
      int rg = run_gemm(c, l, nb, tp.gates, ws.XN.get(), wg, gg, eg, front ? "gemm_gates_front" : "gemm_gates", st);
      if (rg != BT_OK) return rg;
    }
    EpiParams e{};
    e.kind = 1;
    e.out_act = ws.QKV.get(); e.ldo_act = 3 * C;
    e.rope_cos = c->rope_cos->f32.get();
    e.rope_sin = c->rope_sin->f32.get();
    e.C = C; e.heads = heads; e.posmode = freq ? 1 : 0; e.F = F;
    e.qscale = qscale;
    GemmShape g = plain_shape(planes, L, 3 * C, C, C);
    r = run_gemm(c, l, nb, tp.qkv, ws.XN.get(), wqkv, g, e, front ? "gemm_qkv_front" : "gemm_qkv", st);
    if (r != BT_OK) return r;
  }
  if (freq) {
    if (tc) {
      r = make_plan(c, l.name.c_str(), tp.freq, [&](char* err, int n) {
        return tc_freq_plan_create(ws.QKV.get(), ws.O.get(), nb, F, L, heads, err, n);
      });
      if (r != BT_OK) return r;
      launch_attn_freq_tc(tp.freq.get(), ws.GATES.get(), inv_sqrt_d, st);
    } else {
      launch_attn_freq_simt(static_cast<const float*>(ws.QKV.get()), ws.GATES.get(), static_cast<float*>(ws.O.get()),
                            nb, F, L, heads, inv_sqrt_d, st);
    }
    BT_LAUNCHED(c, "attn_freq", st);
  } else if (tc) {
    r = make_plan(c, l.name.c_str(), tp.attn, [&](char* err, int n) {
      return tc_attn_plan_create(ws.QKV.get(), planes, L, heads, err, n);
    });
    if (r != BT_OK) return r;
    launch_attn_time_tc(tp.attn.get(), ws.GATES.get(), ws.O.get(), st, vl_chunks, F);
    BT_LAUNCHED(c, "attn_time_tc", st);
  } else {
    launch_attn_time_simt(static_cast<const float*>(ws.QKV.get()), ws.GATES.get(), static_cast<float*>(ws.O.get()),
                          planes, L, heads, st, vl_chunks, F);
    BT_LAUNCHED(c, "attn_time_simt", st);
  }
  if (out_in_ff) return BT_OK;
  GemmShape go = plain_shape(planes, L, C, C, C);
  EpiParams eo = epi_generic(nullptr, 0, X, C, X, C, nullptr, 0);
  return run_gemm(c, l, nb, tp.out, ws.O.get(), wout, go, eo, front ? "gemm_attn_out_front" : "gemm_attn_out", st);
}

// x += ff(x) (reference roformer.py:38-61); optionally also writes a 16-bit copy of the result.  wout: the
// out-projection weight of the attention in front, which the fused kernel first adds (outproj_in_ff), or null.
int ff_block(bt_ctx* c, float* X, const Layer& l, LayerPlans& tp, int nb, int L, const Param* wout, void* copy_act,
             cudaStream_t st) {
  const Workspace& ws = c->ws;
  const bool tc = c->dtype == BT_DTYPE_H16;
  const bool front = l.F > 1;
  const int C = l.C, mult = l.mult, planes = nb * l.F;
  const Param *w1 = l.w[0], *b1 = l.w[1], *w2 = l.w[2], *b2 = l.w[3];
  const int64_t M = static_cast<int64_t>(planes) * L;
  if (tc && fused(l)) {
    FfPlan& plan = wout ? tp.ff_op : tp.ff;
    const int r = make_plan(c, l.name.c_str(), plan, [&](char* err, int n) {
      return tc_ff_plan_create(w1->b16.get(), w2->b16.get(), C, M, wout ? ws.O.get() : nullptr,
                               wout ? wout->b16.get() : nullptr, err, n);
    });
    if (r != BT_OK) return r;
    launch_fused_ff(plan.get(), X, b1->f32.get(), b2->f32.get(), copy_act, st);
    BT_LAUNCHED(c, C == 32 ? "ff_fused_c32" : "ff_fused_c64", st);
    return BT_OK;
  }
  launch_norm(X, ws.XN.get(), M, C, tc, st);
  BT_LAUNCHED(c, front ? "norm_front" : "norm", st);
  GemmShape g1 = plain_shape(planes, L, mult * C, C, C);
  EpiParams e1 = epi_generic(b1, 1, nullptr, 0, nullptr, 0, ws.H.get(), mult * C);
  int r = run_gemm(c, l, nb, tp.ff1, ws.XN.get(), w1, g1, e1, front ? "gemm_ff1_front" : "gemm_ff1", st);
  if (r != BT_OK) return r;
  GemmShape g2 = plain_shape(planes, L, C, mult * C, mult * C);
  EpiParams e2 = epi_generic(b2, 0, X, C, X, C, copy_act, C);
  return run_gemm(c, l, nb, tp.ff2, ws.H.get(), w2, g2, e2, front ? "gemm_ff2_front" : "gemm_ff2", st);
}

GemmShape conv_shape(int nb, int F, int L, int C) {
  // Conv2d(C -> 2C, k(2 freq, 3 time), stride (2,1), padding (0,1)) over [nb, F, L, C] as an
  // implicit GEMM: slab s = df*3 + dt reads plane 2*p_out + df at time t + dt - 1.
  GemmShape g{};
  g.planes_out = nb * F / 2; g.L = L; g.N = 2 * C; g.Kslab = C; g.nslab = 6; g.plane_mul = 2; g.lda = C;
  for (int df = 0; df < 2; ++df)
    for (int dt = 0; dt < 3; ++dt) { g.plane_add[df * 3 + dt] = df; g.t_shift[df * 3 + dt] = dt - 1; }
  return g;
}
GemmShape lin_shape(int nb, int L, int D, int Fo, int Co) {
  // "b c f t -> b t (c f)" + Linear: slab f reads plane Fo*b + f; W columns permuted to (f, c) on the host
  GemmShape g{};
  g.planes_out = nb; g.L = L; g.N = D; g.Kslab = Co; g.nslab = Fo; g.plane_mul = Fo; g.lda = Co;
  for (int f = 0; f < Fo; ++f) { g.plane_add[f] = f; g.t_shift[f] = 0; }
  return g;
}

// The plans of the wave geometry (nb, L), one LayerPlans per layer, filled by the launches of its first wave (the fp32
// path fills none).  Bounded cache: tensor maps are copied into the kernel parameters at launch, so dropping the oldest
// geometry is safe while its kernels are still in flight.
std::vector<LayerPlans>& geometry_plans(bt_ctx* c, int nb, int L) {
  auto key = std::make_pair(nb, L);
  Workspace& ws = c->ws;
  auto it = ws.plans.find(key);
  if (it != ws.plans.end()) return it->second;
  constexpr size_t kMaxPlans = 48;
  while (ws.plans.size() >= kMaxPlans && !ws.plan_order.empty()) {
    auto old = ws.plans.find(ws.plan_order.front());
    if (old != ws.plans.end()) ws.plans.erase(old);
    ws.plan_order.erase(ws.plan_order.begin());
  }
  ws.plan_order.push_back(key);
  return ws.plans[key] = std::vector<LayerPlans>(c->layers.size());
}

// BeatThis.forward for one wave of nb equal-length chunks, scattering the head output.
int run_wave(bt_ctx* c, const float* spect, const Wave& wv, float* beat, float* down, cudaStream_t st) {
  const bool tc = c->dtype == BT_DTYPE_H16;
  const Workspace& ws = c->ws;
  const int nb = wv.nb, L = wv.L;
  std::vector<LayerPlans>& plans = geometry_plans(c, nb, L);
  int r;
  // chunks shorter than the wave's padded length: the time attentions mask their missing keys and the convolutions
  // see zeros beyond their last frame (everything else works row by row, padding rows are never read back)
  const ChunkSrc* vl = wv.varlen ? wv.chunks_dev : nullptr;
  // the fp32 residual stream: the stem writes X0, and every convolution but the last writes Xalt, which then carries it
  float *X = ws.X0.get(), *Xalt = ws.X1.get();
  const std::vector<Layer>& layers = c->layers;
  const Layer &stem = layers.front(), &head = layers.back();
  launch_stem(spect, wv.chunks_dev, nb, L, stem.w[0]->f32.get(), stem.w[1]->f32.get(), stem.w[2]->f32.get(),
              stem.w[3]->f32.get(), X, st);
  BT_LAUNCHED(c, "stem", st);
  if ((r = do_tap(c, "stem", X, static_cast<int64_t>(nb) * stem.F * L * stem.C, false, st)) != BT_OK) return r;
  for (size_t i = 1; i + 1 < layers.size(); ++i) {
    const Layer& l = layers[i];
    LayerPlans& tp = plans[i];
    const char* tap = l.name.c_str();
    const void* out = X;  // the layer's output (tap)
    bool out_act = false;
    int64_t elems = static_cast<int64_t>(nb) * l.F * L * l.C;
    if (is_attention(l)) {
      r = attention_block(c, X, l, tp, nb, L, outproj_in_ff(c, i), l.kind == kAttnFreq ? nullptr : vl, st);
    } else if (l.kind == kFfn) {
      // the FFN in front of a convolution also writes the 16-bit copy the convolution reads (16-bit path)
      void* copy_act = tc && layers[i + 1].kind == kConv ? ws.XB.get() : nullptr;
      r = ff_block(c, X, l, tp, nb, L, outproj_in_ff(c, i - 1) ? layers[i - 1].w[3] : nullptr, copy_act, st);
    } else if (l.kind == kConv) {
      if (tc && layers[i - 1].kind != kFfn) {  // no FFN in front (no partial transformers)
        launch_f32_to_h16(X, ws.XB.get(), elems, st);
        BT_LAUNCHED(c, "f32_to_h16", st);
      }
      if (vl) {
        launch_zero_tail(tc ? ws.XB.get() : static_cast<void*>(X), tc ? 2 : 4, vl, nb, l.F, L, l.C, st);
        BT_LAUNCHED(c, "zero_tail", st);
      }
      // conv C -> 2C (+ folded BN2d + GELU); the last one feeds frontend.linear in the activation dtype (XN) instead
      const bool last = layers[i + 1].kind == kLinear;
      void* act_out = last ? ws.XN.get() : nullptr;
      EpiParams e = epi_generic(l.w[1], 1, nullptr, 0, last ? nullptr : Xalt, 2 * l.C, act_out, 2 * l.C);
      r = run_gemm(c, l, nb, tp.gemm, tc ? ws.XB.get() : static_cast<const void*>(X), l.w[0],
                   conv_shape(nb, l.F, L, l.C), e, "gemm_conv", st);
      if (last) {
        out = ws.XN.get();
        out_act = true;
      } else {
        out = Xalt;
        std::swap(X, Xalt);
      }
    } else {  // kLinear
      const int D = c->hp.transformer_dim;
      EpiParams e = epi_generic(l.w[1], 0, nullptr, 0, X, D, nullptr, 0);
      r = run_gemm(c, l, nb, tp.gemm, ws.XN.get(), l.w[0], lin_shape(nb, L, D, l.F, l.C), e, "gemm_frontend_linear",
                   st);
      tap = "frontend";
      elems = static_cast<int64_t>(nb) * L * D;
    }
    if (r != BT_OK || (r = do_tap(c, tap, out, elems, out_act, st)) != BT_OK) return r;
  }
  launch_head(X, head.C, head.w[0]->f32.get(), head.w[1]->f32.get(), wv.chunks_dev, nb, L, beat, down,
              c->hp.sum_head ? 1 : 0, st);
  BT_LAUNCHED(c, "head", st);
  return BT_OK;
}

// upload the chunk table and run the forward pass in waves, longest first.  A wave is padded to its longest chunk and
// closes before it would hold more than ws.chunks chunks or more than ws.frames padded frames (chunks of up to
// BT_CHUNK frames never reach the frame budget).  A shorter chunk costs its padded share of one wave (a fraction of a
// millisecond) instead of ~90 launches of its own (~0.7 ms of fixed cost), so chunks of all lengths share waves
int run_chunks(bt_ctx* c, const float* spect_dev, std::vector<ChunkSrc>& all, float* beat_dev, float* downbeat_dev,
               cudaStream_t st) {
  int r = BT_OK;
  if (all.empty()) return BT_OK;
  if ((r = ensure_ws(c)) != BT_OK) return r;
  std::stable_sort(all.begin(), all.end(), [](const ChunkSrc& a, const ChunkSrc& b) { return a.len > b.len; });
  const ChunkSrc* ds = nullptr;
  if ((r = stage(c, st, {{all.data(), all.size()}}, &ds)) != BT_OK) return r;
  size_t i = 0;
  while (i < all.size()) {
    const int64_t L = all[i].len;
    size_t j = i + 1;  // a chunk alone fits: its length is at most max_chunk <= ws.frames
    while (j < all.size() && j - i < static_cast<size_t>(c->ws.chunks) &&
           static_cast<int64_t>(j - i + 1) * L <= c->ws.frames)
      ++j;
    Wave wv{ds + i, static_cast<int>(j - i), all[i].len, all[j - 1].len != all[i].len};
    if ((r = run_wave(c, spect_dev, wv, beat_dev, downbeat_dev, st)) != BT_OK) return r;
    i = j;
  }
  return BT_OK;
}

// the parameters of a layer in the order of Layer::w: name suffix, element count, and whether a GEMM reads it as
// a 16-bit operand
struct ParamSpec { const char* suffix; int64_t count; bool gemm; };
std::vector<ParamSpec> layer_params(const Layer& l, const bt_hparams& hp) {
  const int64_t C = l.C, m = l.mult, D = hp.transformer_dim;
  switch (l.kind) {
    case kStem:
      return {{".bn1_scale", hp.spect_dim, false}, {".bn1_shift", hp.spect_dim, false}, {".w", C * 12, false},
              {".bias", C, false}};
    case kFfn: return {{".w1", m * C * C, true}, {".b1", m * C, false}, {".w2", m * C * C, true}, {".b2", C, false}};
    case kConv: return {{".w", 2 * C * 6 * C, true}, {".bias", 2 * C, false}};
    case kLinear: return {{".w", D * C * l.F, true}, {".b", D, false}};
    case kHead: return {{".w", 2 * C, false}, {".b", 2, false}};
    default: return {{".wqkv", 3 * C * C, true}, {".wg", 32 * C, true}, {".bg", 32, false}, {".wout", C * C, true}};
  }
}

}  // namespace

// ================================================================================== C ABI
extern "C" {

int bt_version(void) { return 219; }

const char* bt_act_dtype(void) {
#if defined(BT_ACT_BF16)
  return "bf16";
#else
  return "f16";
#endif
}

const char* bt_last_error(const bt_ctx* ctx) { return ctx ? ctx->err : g_create_error; }

int64_t bt_num_frames(int64_t n_samples) { return n_samples < 0 ? 0 : 1 + n_samples / BT_HOP; }

int64_t bt_plan_chunks(int64_t T, int64_t* starts, int64_t* lens, int64_t cap) {
  return plan_chunks(T, kDefaultChunking, starts, lens, nullptr, nullptr, cap);
}

int64_t bt_plan_chunking_max(int64_t T, const bt_chunking* ck, int32_t max_chunk, int64_t* starts, int64_t* lens,
                             int64_t* own_lo, int64_t* own_hi, int64_t cap) {
  if (!chunking_valid(ck, max_chunk)) return BT_ERR_ARG;
  return plan_chunks(T, *ck, starts, lens, own_lo, own_hi, cap);
}

int64_t bt_plan_chunking(int64_t T, const bt_chunking* ck, int64_t* starts, int64_t* lens, int64_t* own_lo,
                         int64_t* own_hi, int64_t cap) {
  return bt_plan_chunking_max(T, ck, BT_CHUNK, starts, lens, own_lo, own_hi, cap);
}

int bt_create(bt_ctx** out, int device_ordinal, const bt_hparams* hp, int compute_dtype) {
  if (!out || !hp) return fail(nullptr, BT_ERR_ARG, "bt_create: null argument");
  *out = nullptr;
  if (compute_dtype != BT_DTYPE_F32 && compute_dtype != BT_DTYPE_H16)
    return fail(nullptr, BT_ERR_ARG, "bt_create: compute_dtype must be BT_DTYPE_F32 or BT_DTYPE_H16");
  if (hp->spect_dim != 128 || hp->head_dim != 32 || hp->stem_dim != 32 || hp->transformer_dim % 64 != 0 ||
      hp->transformer_dim < 64 || hp->transformer_dim > 1024 || hp->n_layers < 1 || hp->ff_mult < 1 ||
      hp->ff_mult > 4)
    return fail(nullptr, BT_ERR_ARG,
                "bt_create: unsupported hyper-parameters (need spect_dim 128, head_dim 32, stem_dim 32, "
                "transformer_dim multiple of 64 in [64,1024], ff_mult <= 4)");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(nullptr, BT_ERR_CUDA, "bt_create: no CUDA device (%s); this library has no CPU fallback",
                cudaGetErrorString(e));
  if (device_ordinal < 0 || device_ordinal >= ndev)
    return fail(nullptr, BT_ERR_ARG, "bt_create: device %d out of range (%d devices)", device_ordinal, ndev);
  if ((e = cudaSetDevice(device_ordinal)) != cudaSuccess)
    return fail(nullptr, BT_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device_ordinal);
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, BT_ERR_CUDA, "bt_create: device is sm_%d%d; this library is built for sm_90a only",
                prop.major, prop.minor);
  bt_ctx* c = new bt_ctx();
  c->device = device_ordinal;
  c->hp = *hp;
  c->dtype = compute_dtype;
  const char* dbg = getenv("BT_SYNC_DEBUG");
  c->sync_debug = dbg && dbg[0] == '1';

  if (compute_dtype == BT_DTYPE_H16) {
    char err[512];
    if (tc_init(err, sizeof(err)) != 0) {
      delete c;
      return fail(nullptr, BT_ERR_CUDA, "%s", err);
    }
  }
  *out = c;
  return BT_OK;
}

int bt_set_param(bt_ctx* c, const char* name, const float* data_host, int64_t count) {
  if (!c || !name || !data_host || count <= 0) return fail(c, BT_ERR_ARG, "bt_set_param: bad argument");
  if (c->finalized) return fail(c, BT_ERR_STATE, "bt_set_param after bt_finalize");
  BT_CUDA(c, cudaSetDevice(c->device));
  Param& p = c->params[name];
  p = Param();
  p.n = count;
  const std::string n(name);
  if (n == "mel.fb_start" || n == "mel.fb_ptr") {
    std::vector<int32_t> tmp(count);
    for (int64_t i = 0; i < count; ++i) tmp[i] = static_cast<int32_t>(lrintf(data_host[i]));
    BT_CUDA(c, p.i32.alloc(count * 4));
    BT_CUDA(c, cudaMemcpy(p.i32.get(), tmp.data(), count * 4, cudaMemcpyHostToDevice));
  }
  BT_CUDA(c, p.f32.alloc(count * 4));
  BT_CUDA(c, cudaMemcpy(p.f32.get(), data_host, count * 4, cudaMemcpyHostToDevice));
  return BT_OK;
}

int bt_finalize(bt_ctx* c) {
  if (!c) return BT_ERR_ARG;
  if (c->finalized) return BT_OK;
  BT_CUDA(c, cudaSetDevice(c->device));
  // every parameter the forward pass reads, with its element count (-1: not checked), resolved once here (no name
  // lookups per launch)
  struct Need { std::string name; int64_t count; const Param** dst; bool gemm; };
  std::vector<Need> need = {
      {"mel.window", 1024, nullptr, false}, {"mel.twiddle", 1024, nullptr, false}, {"mel.fb_start", 128, nullptr, false},
      {"mel.fb_ptr", 129, nullptr, false}, {"mel.fb_w", -1, nullptr, false},
      {"rope.cos", -1, &c->rope_cos, false}, {"rope.sin", -1, &c->rope_sin, false}};  // checked below
  c->layers.clear();
  for (const Step& s : model_steps(c->hp)) c->layers.push_back({s});
  for (Layer& l : c->layers) {
    const std::vector<ParamSpec> specs = layer_params(l, c->hp);
    for (size_t k = 0; k < specs.size(); ++k) need.push_back({l.name + specs[k].suffix, specs[k].count, &l.w[k], specs[k].gemm});
  }
  for (const Need& n : need)
    if (!find_param(c, n.name)) return fail(c, BT_ERR_PARAM, "bt_finalize: missing parameter '%s'", n.name.c_str());
  for (const Need& n : need) {
    const Param* p = find_param(c, n.name);
    if (n.count >= 0 && p->n != n.count)
      return fail(c, BT_ERR_PARAM, "parameter '%s' has %lld elements, expected %lld", n.name.c_str(), (long long)p->n,
                  (long long)n.count);
    if (n.dst) *n.dst = p;
  }
  // the RoPE tables hold positions 0 .. P - 1, and P is the longest chunk this ctx takes
  const int64_t rows = c->rope_cos->n / 16;
  if (c->rope_cos->n % 16 != 0 || rows < BT_CHUNK || rows > kMaxChunkCap || c->rope_sin->n != c->rope_cos->n)
    return fail(c, BT_ERR_PARAM, "parameters 'rope.cos' / 'rope.sin' have %lld / %lld elements; both need P x 16 with "
                "%d <= P <= %lld", (long long)c->rope_cos->n, (long long)c->rope_sin->n, BT_CHUNK, (long long)kMaxChunkCap);
  c->max_chunk = static_cast<int>(rows);
  if (c->dtype == BT_DTYPE_H16) {
    for (const Need& n : need) {
      if (!n.gemm) continue;
      Param& p = c->params[n.name];
      BT_CUDA(c, p.b16.alloc(p.n * 2));
      launch_f32_to_h16(p.f32.get(), p.b16.get(), p.n, nullptr);
    }
    BT_CUDA(c, cudaDeviceSynchronize());
  }
  c->finalized = true;
  return BT_OK;
}

void bt_destroy(bt_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  delete c;
}

int bt_set_wave_chunks(bt_ctx* c, int32_t chunks) {
  if (!c || chunks < 1 || chunks > kMaxWaveChunks) return fail(c, BT_ERR_ARG, "bt_set_wave_chunks: 1..%d", kMaxWaveChunks);
  c->wave = chunks;
  if (c->ws.chunks > chunks) {  // shrink: drop the workspace, it is re-created on the next call
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    c->ws = Workspace();
  }
  return BT_OK;
}

int32_t bt_max_chunk(const bt_ctx* c) { return c ? c->max_chunk : BT_ERR_ARG; }

int64_t bt_launch_count(const bt_ctx* c) { return c ? c->launches : 0; }

int bt_profile_enable(bt_ctx* c, int enable) {
  if (!c) return BT_ERR_ARG;
  c->prof = enable != 0;
  c->prof_prev = -1;
  return BT_OK;
}

int bt_profile_collect(bt_ctx* c) {
  if (!c) return BT_ERR_ARG;
  BT_CUDA(c, cudaSetDevice(c->device));
  BT_CUDA(c, cudaDeviceSynchronize());
  for (const auto& r : c->prof_recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev_pool[r.prev].get(), c->ev_pool[r.ev].get()) == cudaSuccess) {
      c->prof_ms[r.kind] += ms;
      c->prof_cnt[r.kind] += 1;
    }
  }
  c->prof_recs.clear();
  c->ev_used = 0;
  c->prof_prev = -1;
  return BT_OK;
}

int bt_profile_reset(bt_ctx* c) {
  if (!c) return BT_ERR_ARG;
  int r = bt_profile_collect(c);
  for (auto& v : c->prof_ms) v = 0.0;
  for (auto& v : c->prof_cnt) v = 0;
  return r;
}

int bt_profile_count(const bt_ctx* c) { return c ? static_cast<int>(c->prof_names.size()) : 0; }

int bt_profile_get(const bt_ctx* c, int index, char* name, int name_cap, double* total_ms, int64_t* launches) {
  if (!c || index < 0 || index >= static_cast<int>(c->prof_names.size())) return BT_ERR_ARG;
  if (name && name_cap > 0) snprintf(name, name_cap, "%s", c->prof_names[index].c_str());
  if (total_ms) *total_ms = c->prof_ms[index];
  if (launches) *launches = c->prof_cnt[index];
  return BT_OK;
}

int bt_debug_request_tap(bt_ctx* c, const char* tap, float* out_dev, int64_t cap) {
  if (!c) return BT_ERR_ARG;
  c->tap_name = tap ? tap : "";
  c->tap_out = out_dev;
  c->tap_cap = cap;
  c->tap_count = 0;
  return BT_OK;
}
int64_t bt_debug_tap_count(const bt_ctx* c) { return c ? c->tap_count : 0; }

// bt_spect2frames(_chunked); `fn` names the entry point in errors
static int spect2frames(bt_ctx* c, const float* spect_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                        float* beat_dev, float* downbeat_dev, const bt_chunking* ck, void* stream, const char* fn) {
  if (const int r = check_chunking(c, fn, ck)) return r;
  if (n_clips <= 0) return BT_OK;
  if (!spect_dev || !frame_offsets_host || !beat_dev || !downbeat_dev) return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  int r = check_offsets(c, fn, "frame_offsets_host", frame_offsets_host, n_clips, kFromNonNegative);
  cudaStream_t st;
  if (r != BT_OK || (r = enter(c, fn, stream, &st)) != BT_OK) return r;
  // plan: all chunks of all clips; run_chunks groups them by chunk length
  std::vector<ChunkSrc> all;
  std::vector<int64_t> starts, lens, own_lo, own_hi;
  for (int i = 0; i < n_clips; ++i) {
    const int64_t T = frame_offsets_host[i + 1] - frame_offsets_host[i];
    if (T == 0) continue;
    const int64_t n = plan_chunks(T, *ck, nullptr, nullptr, nullptr, nullptr, 0);
    starts.resize(n); lens.resize(n); own_lo.resize(n); own_hi.resize(n);
    plan_chunks(T, *ck, starts.data(), lens.data(), own_lo.data(), own_hi.data(), n);
    for (int64_t j = 0; j < n; ++j) {
      ChunkSrc s{};
      s.frame_base = frame_offsets_host[i];
      s.out_base = frame_offsets_host[i];
      s.T = static_cast<int32_t>(T);
      s.start = static_cast<int32_t>(starts[j]);
      s.write_lo = static_cast<int32_t>(own_lo[j] - starts[j]);
      s.write_hi = static_cast<int32_t>(own_hi[j] - starts[j]);
      s.len = static_cast<int32_t>(lens[j]);
      all.push_back(s);
    }
  }
  return run_chunks(c, spect_dev, all, beat_dev, downbeat_dev, st);
}

int bt_spect2frames(bt_ctx* c, const float* spect_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                    float* beat_dev, float* downbeat_dev, void* stream) {
  return spect2frames(c, spect_dev, frame_offsets_host, n_clips, beat_dev, downbeat_dev, &kDefaultChunking, stream,
                      "bt_spect2frames");
}

int bt_spect2frames_chunked(bt_ctx* c, const float* spect_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                            float* beat_dev, float* downbeat_dev, const bt_chunking* ck, void* stream) {
  return spect2frames(c, spect_dev, frame_offsets_host, n_clips, beat_dev, downbeat_dev, ck, stream,
                      "bt_spect2frames_chunked");
}

int bt_forward_chunks(bt_ctx* c, const float* chunks_dev, int32_t n_chunks, int32_t chunk_frames, float* beat_dev,
                      float* downbeat_dev, void* stream) {
  if (!c || !c->finalized) return fail(c, BT_ERR_STATE, "bt_forward_chunks: context not finalized");
  if (n_chunks <= 0) return BT_OK;
  if (!chunks_dev || !beat_dev || !downbeat_dev) return fail(c, BT_ERR_ARG, "bt_forward_chunks: null argument");
  if (chunk_frames < 1 || chunk_frames > c->max_chunk)
    return fail(c, BT_ERR_ARG, "bt_forward_chunks: chunk_frames must be in [1, %d] (bt_max_chunk)", c->max_chunk);
  cudaStream_t st;
  if (const int r = enter(c, "bt_forward_chunks", stream, &st)) return r;
  std::vector<ChunkSrc> all(n_chunks);
  for (int i = 0; i < n_chunks; ++i) {
    ChunkSrc& s = all[i];
    s.frame_base = static_cast<int64_t>(i) * chunk_frames;
    s.out_base = s.frame_base;
    s.T = chunk_frames;
    s.start = 0;
    s.write_lo = 0;
    s.write_hi = chunk_frames;
    s.len = chunk_frames;
    s.pad_ = 0;
  }
  return run_chunks(c, chunks_dev, all, beat_dev, downbeat_dev, st);
}

// bt_audio2frames(_chunked): the offsets are checked (as bt_logmel does) before the spectrogram scratch may grow
static int audio2frames(bt_ctx* c, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                        float* beat_dev, float* downbeat_dev, const int64_t* frame_offsets_host, const bt_chunking* ck,
                        void* stream, const char* fn) {
  if (const int r = check_chunking(c, fn, ck)) return r;
  if (n_clips <= 0) return BT_OK;
  if (!audio_dev || !sample_offsets_host || !frame_offsets_host || !beat_dev || !downbeat_dev)
    return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  int r = check_stft_frames(c, fn, sample_offsets_host, frame_offsets_host, n_clips, BT_N_FFT, BT_HOP);
  if (r != BT_OK) return r;
  BT_CUDA(c, cudaSetDevice(c->device));
  const size_t need = frame_offsets_host[n_clips] * 128 * 4;
  BT_CUDA(c, c->spect_ws.reserve(need, need + need / 4));
  if ((r = bt_logmel(c, audio_dev, sample_offsets_host, n_clips, c->spect_ws.get(), frame_offsets_host, stream)) != BT_OK)
    return r;
  return spect2frames(c, c->spect_ws.get(), frame_offsets_host, n_clips, beat_dev, downbeat_dev, ck, stream, fn);
}

int bt_audio2frames(bt_ctx* c, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                    float* beat_dev, float* downbeat_dev, const int64_t* frame_offsets_host, void* stream) {
  return audio2frames(c, audio_dev, sample_offsets_host, n_clips, beat_dev, downbeat_dev, frame_offsets_host,
                      &kDefaultChunking, stream, "bt_audio2frames");
}

int bt_audio2frames_chunked(bt_ctx* c, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                            float* beat_dev, float* downbeat_dev, const int64_t* frame_offsets_host,
                            const bt_chunking* ck, void* stream) {
  return audio2frames(c, audio_dev, sample_offsets_host, n_clips, beat_dev, downbeat_dev, frame_offsets_host, ck, stream,
                      "bt_audio2frames_chunked");
}

}  // extern "C"
