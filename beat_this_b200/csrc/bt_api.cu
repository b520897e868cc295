// C ABI (include/beatthis.h): context, packed-parameter registry, chunk planner, workspace
// and the per-wave schedule of the BeatThis forward pass (reference
// beat_this/model/beat_tracker.py:188-192).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/beatthis.h"
#include "bt_kernels.h"
#include "cuda_owned.h"
#include "dbn_model.h"

using namespace bt;

namespace {

struct Param {
  DeviceBuffer<float> f32;
  DeviceBuffer<> b16;
  DeviceBuffer<int32_t> i32;
  int64_t n = 0;
};

// One layer of the forward pass between the stem and the head.  bt_finalize builds the list from bt_hparams, in schedule
// order: b{i}.attnF, b{i}.ffF, b{i}.attnT, b{i}.ffT (with partial transformers), b{i}.conv for i < 3, lin, then
// l{l}.attn, l{l}.ff for every main layer.
enum LayerKind { kAttnF, kAttnT, kAttn, kFf, kConv, kLin };  // kAttnF / kAttnT: frequency / time attention of a frontend block
struct Layer {
  LayerKind kind;
  std::string name;  // parameter prefix, and the tap name of the layer's output (frontend.linear: "frontend")
  int C, F;          // channels; frequency planes per chunk (1 in the main layers)
  int mult;          // FFN hidden width multiplier
  const Param* w[4]; // resolved weights, in the order of layer_params
};

// small host -> device tables (offsets, chunk descriptors) travel through a ring of pinned slots: a slot is only
// waited for when it comes round again, kStageSlots uploads later, so no API call blocks on earlier GPU work
constexpr int kStageSlots = 16;
struct StageSlot {
  PinnedBuffer<char> host;
  DeviceBuffer<char> dev;
  Event ev;
  bool pending = false;
};

// Tensor-core plans of one layer for one (wave size, chunk length) geometry.  Each launch of the 16-bit path makes its
// plan from its operands when the geometry first runs; later waves of the geometry reuse it.
struct LayerPlans {
  QkvPlan fqkv;              // attention, fused (C = 32 / 64)
  GemmPlan gates, qkv, out;  // attention: gates and QKV unless fused; out-projection
  AttnPlan attn;             // time attention
  FreqPlan freq;             // frequency attention
  FfPlan ff, ff_op;          // FFN, fused; ff_op: with the attention's out-projection in front (outproj_in_ff)
  GemmPlan ff1, ff2;         // FFN, unfused
  GemmPlan gemm;             // convolution, frontend.linear
};

// The activations of a wave of up to `chunks` chunks and `frames` padded frames (XB only on the 16-bit path), and the
// tensor-core plans made for them: their tensor maps hold workspace addresses, so the two are dropped together.
struct Workspace {
  int chunks = 0;
  int64_t frames = 0;
  DeviceBuffer<float> X0, X1, GATES;
  DeviceBuffer<> XB, XN, QKV, O, H;
  std::map<std::pair<int, int>, std::vector<LayerPlans>> plans;  // per (nb, L) geometry, parallel to bt_ctx::layers
  std::vector<std::pair<int, int>> plan_order;                   // insertion order: oldest geometry is evicted first
};

char g_create_error[512] = "";

}  // namespace

struct bt_ctx {
  int device = 0;
  bt_hparams hp{};
  int dtype = BT_DTYPE_F32;
  bool finalized = false;
  std::map<std::string, Param> params;
  mutable char err[1024] = "";
  const char* call = "";  // the entry point that is launching (begin_call)
  int64_t launches = 0;
  bool sync_debug = false;

  int wave = 128;  // the workspace grows on demand up to `wave` chunks
  int max_chunk = BT_CHUNK;  // longest chunk the forward pass takes: the rows of the RoPE tables (bt_finalize)
  Workspace ws;
  // spectrogram scratch for bt_audio2frames
  DeviceBuffer<float> spect_ws;
  // DBN scratch for bt_dbn_track_device / bt_debug_dbn_viterbi (grows on demand): activations, densities, windows,
  // per-model results and path codes; back pointers
  DeviceBuffer<char> dbn_ws;
  DeviceBuffer<uint8_t> dbn_bp;
  // per-CTA partial sums of bt_beat_loss (grows on demand)
  DeviceBuffer<double> loss_partials;
  // windowed inverse transforms of bt_istft's frames, n_fft floats each (grows on demand)
  DeviceBuffer<float> istft_frames;
  // pinned staging + device tables
  StageSlot stage[kStageSlots];
  int stage_next = 0;
  std::vector<Layer> layers;  // built by bt_finalize
  // parameters outside the layer list, resolved in bt_finalize
  const Param *rope_cos = nullptr, *rope_sin = nullptr, *bn1_scale = nullptr, *bn1_shift = nullptr, *stem_w = nullptr,
              *stem_b = nullptr, *head_w = nullptr, *head_b = nullptr;

  // per-kernel-class device timing (bt_profile_*): one event after every launch; the
  // duration of a launch is the gap to the previous event on the same stream
  bool prof = false;
  std::vector<Event> ev_pool;
  size_t ev_used = 0;
  struct ProfRec { int kind; int ev; int prev; };
  std::vector<ProfRec> prof_recs;
  int prof_prev = -1;
  std::vector<std::string> prof_names;
  std::vector<double> prof_ms;
  std::vector<int64_t> prof_cnt;

  // debug tap
  std::string tap_name;
  float* tap_out = nullptr;
  int64_t tap_cap = 0;
  int64_t tap_count = 0;
};

namespace {

int fail(const bt_ctx* c, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  if (c) vsnprintf(c->err, sizeof(c->err), fmt, ap);
  else vsnprintf(g_create_error, sizeof(g_create_error), fmt, ap);
  va_end(ap);
  return code;
}

#define BT_CUDA(ctx, call)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (call);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return fail(ctx, BT_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), \
                  __FILE__, __LINE__);                                                       \
  } while (0)

int prof_event(bt_ctx* c, cudaStream_t st) {
  if (c->ev_used == c->ev_pool.size()) {
    cudaEvent_t ev;
    if (cudaEventCreate(&ev) != cudaSuccess) return -1;
    c->ev_pool.emplace_back(ev);
  }
  const int idx = static_cast<int>(c->ev_used++);
  cudaEventRecord(c->ev_pool[idx].get(), st);
  return idx;
}

// Start of an API call that launches: fn is the entry point its launch errors name, and the profile gets the reference
// point of its first kernel.
void begin_call(bt_ctx* c, const char* fn, cudaStream_t st) {
  c->call = fn;
  if (c->prof) c->prof_prev = prof_event(c, st);
}

void prof_launch(bt_ctx* c, const char* what, cudaStream_t st) {
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

// Follows every launcher call.  status: what the launcher returned; a failed host step launched nothing.  Otherwise the
// launch is counted (bt_launch_count), profiled as `what`, checked, and under BT_SYNC_DEBUG waited for.
int check_launch(bt_ctx* c, const char* what, cudaStream_t st, cudaError_t status = cudaSuccess) {
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
// check_launch(c, what, st[, status]), returning from the caller on failure
#define BT_LAUNCHED(c, what, st, ...)                       \
  do {                                                      \
    int _r = check_launch(c, what, st, ##__VA_ARGS__);      \
    if (_r != BT_OK) return _r;                             \
  } while (0)

const Param* find_param(const bt_ctx* c, const std::string& name) {
  auto it = c->params.find(name);
  return it == c->params.end() ? nullptr : &it->second;
}

constexpr bt_chunking kDefaultChunking{BT_CHUNK, BT_BORDER, BT_KEEP_FIRST};
constexpr int kMaxWaveChunks = 256;  // bt_set_wave_chunks
// Longest chunk a ctx takes: the largest frame budget bt_set_wave_chunks allows, so that no wave holds more frames
// than one of kMaxWaveChunks chunks of BT_CHUNK frames (the 32-bit element counts of the kernels stay within that)
constexpr int64_t kMaxChunkCap = static_cast<int64_t>(kMaxWaveChunks) * BT_CHUNK;

bool chunking_valid(const bt_chunking* ck, int64_t max_chunk) {
  return ck && ck->chunk_size >= 1 && ck->chunk_size <= max_chunk && ck->border >= 0 &&
         2 * static_cast<int64_t>(ck->border) < ck->chunk_size &&
         (ck->overlap_mode == BT_KEEP_FIRST || ck->overlap_mode == BT_KEEP_LAST);
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

int acquire_stage(bt_ctx* c, size_t bytes, StageSlot** out) {
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

int upload_stage(bt_ctx* c, StageSlot* sl, size_t bytes, cudaStream_t st) {
  BT_CUDA(c, cudaMemcpyAsync(sl->dev.get(), sl->host.get(), bytes, cudaMemcpyHostToDevice, st));
  BT_CUDA(c, cudaEventRecord(sl->ev.get(), st));
  sl->pending = true;
  return BT_OK;
}

inline size_t align16(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }

// Copies a few host arrays of n[k] elements into the next ring slot, each at a 16-byte aligned offset, and uploads the
// slot: dev[k] is array k on the device.
template <class T>
int stage(bt_ctx* c, cudaStream_t st, std::initializer_list<std::pair<const T*, size_t>> arrays, const T** dev) {
  size_t bytes = 0;
  for (const auto& a : arrays) bytes = align16(bytes) + sizeof(T) * a.second;
  StageSlot* sl = nullptr;
  const int r = acquire_stage(c, bytes, &sl);
  if (r != BT_OK) return r;
  size_t off = 0;
  for (const auto& a : arrays) {
    off = align16(off);
    memcpy(sl->host.get() + off, a.first, sizeof(T) * a.second);
    *dev++ = reinterpret_cast<const T*>(sl->dev.get() + off);
    off += sizeof(T) * a.second;
  }
  return upload_stage(c, sl, bytes, st);
}

// elements per frame of the largest frontend activation: F*C is the same for all blocks
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

// Fills an empty plan slot: create(err, errlen) makes the plan from the operands of the launch that uses it.  label
// (the layer, or the test hook) names it in the error; a refused plan returns `code`.
template <class Plan, class Create>
int make_plan(bt_ctx* c, const char* label, std::unique_ptr<Plan, CudaDestroy>& slot, Create create,
              int code = BT_ERR_CUDA) {
  if (slot) return BT_OK;
  char err[512] = "";
  slot.reset(create(err, static_cast<int>(sizeof(err))));
  if (!slot) return fail(c, code, "tensor-core plan creation failed (%s): %s", label, err);
  return BT_OK;
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

bool is_attention(const Layer& l) { return l.kind == kAttnF || l.kind == kAttnT || l.kind == kAttn; }

// sub-blocks of width C = 32 / 64 (the first two frontend blocks) run as one fused kernel each on the 16-bit path
bool fused(const Layer& l) { return (l.C == 32 || l.C == 64) && (l.kind != kFf || l.mult == 4); }

// The out-projection + residual of attention layer i run inside the fused FFN after it (fused_ff_kernel<C, true>) on
// the 16-bit path when the attention is a frontend one, unless a tap asks to see the residual stream between the two.
bool outproj_in_ff(const bt_ctx* c, size_t i) {
  const Layer& l = c->layers[i];
  return c->dtype == BT_DTYPE_H16 && (l.kind == kAttnF || l.kind == kAttnT) && i + 1 < c->layers.size() &&
         c->layers[i + 1].kind == kFf && fused(c->layers[i + 1]) && c->tap_name != l.name;
}

// x += attention(x) over nb * F planes of L tokens with dim C (reference roformer.py:114-132).
// kAttnF: sequences run over the F planes of each chunk (PartialFTTransformer attnF).
int attention_block(bt_ctx* c, float* X, const Layer& l, LayerPlans& tp, int nb, int L, bool out_in_ff,
                    const ChunkSrc* vl_chunks, cudaStream_t st) {
  const Workspace& ws = c->ws;
  const bool tc = c->dtype == BT_DTYPE_H16;
  const bool freq = l.kind == kAttnF, front = l.F > 1;
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
  launch_stem(spect, wv.chunks_dev, nb, L, c->bn1_scale->f32.get(), c->bn1_shift->f32.get(), c->stem_w->f32.get(),
              c->stem_b->f32.get(), X, st);
  BT_LAUNCHED(c, "stem", st);
  if ((r = do_tap(c, "stem", X, static_cast<int64_t>(nb) * (c->hp.spect_dim / 4) * L * c->hp.stem_dim, false, st)) != BT_OK)
    return r;
  const std::vector<Layer>& layers = c->layers;
  for (size_t i = 0; i < layers.size(); ++i) {
    const Layer& l = layers[i];
    LayerPlans& tp = plans[i];
    const char* tap = l.name.c_str();
    const void* out = X;  // the layer's output (tap)
    bool out_act = false;
    int64_t elems = static_cast<int64_t>(nb) * l.F * L * l.C;
    if (is_attention(l)) {
      r = attention_block(c, X, l, tp, nb, L, outproj_in_ff(c, i), l.kind == kAttnF ? nullptr : vl, st);
    } else if (l.kind == kFf) {
      // the FFN in front of a convolution also writes the 16-bit copy the convolution reads (16-bit path)
      void* copy_act = tc && i + 1 < layers.size() && layers[i + 1].kind == kConv ? ws.XB.get() : nullptr;
      r = ff_block(c, X, l, tp, nb, L, i > 0 && outproj_in_ff(c, i - 1) ? layers[i - 1].w[3] : nullptr, copy_act, st);
    } else if (l.kind == kConv) {
      if (tc && (i == 0 || layers[i - 1].kind != kFf)) {  // no FFN in front (no partial transformers)
        launch_f32_to_h16(X, ws.XB.get(), elems, st);
        BT_LAUNCHED(c, "f32_to_h16", st);
      }
      if (vl) {
        launch_zero_tail(tc ? ws.XB.get() : static_cast<void*>(X), tc ? 2 : 4, vl, nb, l.F, L, l.C, st);
        BT_LAUNCHED(c, "zero_tail", st);
      }
      // conv C -> 2C (+ folded BN2d + GELU); the last one feeds frontend.linear in the activation dtype (XN) instead
      const bool last = i + 1 < layers.size() && layers[i + 1].kind == kLin;
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
    } else {  // kLin
      const int D = c->hp.transformer_dim;
      EpiParams e = epi_generic(l.w[1], 0, nullptr, 0, X, D, nullptr, 0);
      r = run_gemm(c, l, nb, tp.gemm, ws.XN.get(), l.w[0], lin_shape(nb, L, D, l.F, l.C), e, "gemm_frontend_linear",
                   st);
      tap = "frontend";
      elems = static_cast<int64_t>(nb) * L * D;
    }
    if (r != BT_OK || (r = do_tap(c, tap, out, elems, out_act, st)) != BT_OK) return r;
  }
  launch_head(X, c->hp.transformer_dim, c->head_w->f32.get(), c->head_b->f32.get(), wv.chunks_dev, nb, L, beat, down,
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

std::vector<Layer> layer_list(const bt_hparams& hp) {
  std::vector<Layer> v;
  int C = hp.stem_dim, F = hp.spect_dim / 4;
  for (int i = 0; i < 3; ++i) {
    const std::string b = "b" + std::to_string(i);
    if (hp.partial_transformers) {
      v.push_back({kAttnF, b + ".attnF", C, F, 0, {}});
      v.push_back({kFf, b + ".ffF", C, F, 4, {}});
      v.push_back({kAttnT, b + ".attnT", C, F, 0, {}});
      v.push_back({kFf, b + ".ffT", C, F, 4, {}});
    }
    v.push_back({kConv, b + ".conv", C, F, 0, {}});
    C *= 2; F /= 2;
  }
  v.push_back({kLin, "lin", C, F, 0, {}});
  for (int l = 0; l < hp.n_layers; ++l) {
    v.push_back({kAttn, "l" + std::to_string(l) + ".attn", hp.transformer_dim, 1, 0, {}});
    v.push_back({kFf, "l" + std::to_string(l) + ".ff", hp.transformer_dim, 1, hp.ff_mult, {}});
  }
  return v;
}

// the parameters of a layer in the order of Layer::w: name suffix, element count, and whether a GEMM reads it as
// a 16-bit operand
struct ParamSpec { const char* suffix; int64_t count; bool gemm; };
std::vector<ParamSpec> layer_params(const Layer& l, int64_t D) {
  const int64_t C = l.C, m = l.mult;
  switch (l.kind) {
    case kFf: return {{".w1", m * C * C, true}, {".b1", m * C, false}, {".w2", m * C * C, true}, {".b2", C, false}};
    case kConv: return {{".w", 2 * C * 6 * C, true}, {".bias", 2 * C, false}};
    case kLin: return {{".w", D * C * l.F, true}, {".b", D, false}};
    default: return {{".wqkv", 3 * C * C, true}, {".wg", 32 * C, true}, {".bg", 32, false}, {".wout", C * C, true}};
  }
}

bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

// A test hook's fp32 device array of n elements that its kernel reads in the activation type: the 16-bit context hands
// the kernel h16, a rounded copy, and rounds an `out` array (an output the caller pre-filled, so that elements the
// kernel does not store survive) back after the launch.  A null array stays null.
struct HookArray {
  float* f32;
  int64_t n;
  bool out;
  DeviceBuffer<> h16;
  HookArray(const float* p, int64_t n, bool out = false) : f32(const_cast<float*>(p)), n(n), out(out) {}
};

// Runs a test hook after its own argument checks: sets the device, takes the stream and begins the call; in the 16-bit
// context rounds `arrays`; launch(st) makes its plans (make_plan) and launches the kernel(s) under test (check_launch:
// only they are counted and profiled); then rounds the out arrays back and synchronises the stream.  Scratch that
// launch uses must outlive the call.
template <class Launch>
int run_hook(bt_ctx* c, const char* fn, void* stream, std::initializer_list<HookArray*> arrays, Launch launch) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool tc = c->dtype == BT_DTYPE_H16;
  cudaError_t e = cudaSetDevice(c->device);
  if (e == cudaSuccess) begin_call(c, fn, st);
  for (HookArray* a : arrays)
    if (tc && a->f32 && e == cudaSuccess && (e = a->h16.alloc(a->n * 2)) == cudaSuccess)
      launch_f32_to_h16(a->f32, a->h16.get(), a->n, st);
  if (e != cudaSuccess) return fail(c, BT_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(e));
  int rc = launch(st);
  for (HookArray* a : arrays)
    if (tc && a->f32 && a->out && rc == BT_OK) launch_h16_to_f32(a->h16.get(), a->f32, a->n, st);
  e = cudaStreamSynchronize(st);
  if (rc == BT_OK && e != cudaSuccess) rc = fail(c, BT_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(e));
  return rc;
}

}  // namespace

// ================================================================================== C ABI
extern "C" {

int bt_version(void) { return 210; }

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
  const int64_t D = c->hp.transformer_dim;
  // every parameter the forward pass reads, with its element count (-1: not checked), resolved once here (no name
  // lookups per launch)
  struct Need { std::string name; int64_t count; const Param** dst; bool gemm; };
  std::vector<Need> need = {
      {"mel.window", 1024, nullptr, false}, {"mel.twiddle", 1024, nullptr, false}, {"mel.fb_start", 128, nullptr, false},
      {"mel.fb_ptr", 129, nullptr, false}, {"mel.fb_w", -1, nullptr, false},
      {"rope.cos", -1, &c->rope_cos, false}, {"rope.sin", -1, &c->rope_sin, false},  // checked below
      {"stem.bn1_scale", -1, &c->bn1_scale, false}, {"stem.bn1_shift", -1, &c->bn1_shift, false},
      {"stem.w", 32 * 12, &c->stem_w, false}, {"stem.bias", -1, &c->stem_b, false},
      {"head.w", 2 * D, &c->head_w, false}, {"head.b", 2, &c->head_b, false}};
  c->layers = layer_list(c->hp);
  for (Layer& l : c->layers) {
    const std::vector<ParamSpec> specs = layer_params(l, D);
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

int bt_logmel(bt_ctx* c, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
              float* spect_dev, const int64_t* frame_offsets_host, void* stream) {
  if (!c) return BT_ERR_ARG;
  for (const char* n : {"mel.window", "mel.twiddle", "mel.fb_start", "mel.fb_ptr", "mel.fb_w"})
    if (!find_param(c, n)) return fail(c, BT_ERR_STATE, "bt_logmel: parameter '%s' not set", n);
  if (n_clips <= 0) return BT_OK;
  if (!audio_dev || !sample_offsets_host || !spect_dev || !frame_offsets_host)
    return fail(c, BT_ERR_ARG, "bt_logmel: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, "bt_logmel", st);
  for (int i = 0; i < n_clips; ++i) {
    const int64_t len = sample_offsets_host[i + 1] - sample_offsets_host[i];
    if (len <= BT_N_FFT / 2)
      return fail(c, BT_ERR_ARG, "bt_logmel: clip %d has %lld samples; reflect padding needs more than %d "
                  "(torch.stft raises for such input as well)", i, (long long)len, BT_N_FFT / 2);
    if (frame_offsets_host[i + 1] - frame_offsets_host[i] != bt_num_frames(len))
      return fail(c, BT_ERR_ARG, "bt_logmel: frame_offsets do not match 1 + len/441 for clip %d", i);
  }
  const size_t n = n_clips + 1;
  const int64_t* d[2];
  const int r = stage(c, st, {{sample_offsets_host, n}, {frame_offsets_host, n}}, d);
  if (r != BT_OK) return r;
  if (frame_offsets_host[0] != 0) return fail(c, BT_ERR_ARG, "bt_logmel: frame_offsets_host[0] must be 0");
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
  int log2n = 6;
  while (log2n < 13 && (1 << log2n) != cfg->n_fft) ++log2n;
  if ((1 << log2n) != cfg->n_fft)
    return fail(c, BT_ERR_ARG, "%s: n_fft %d is not a power of two in [64, 8192]", fn, cfg->n_fft);
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
  if (sample_offsets_host[0] < 0 || frame_offsets_host[0] != 0)
    return fail(c, BT_ERR_ARG, "%s: sample offsets must start at >= 0 and frame offsets at 0", fn);
  for (int i = 0; i < n_clips; ++i) {
    const int64_t len = sample_offsets_host[i + 1] - sample_offsets_host[i];
    if (len <= cfg->n_fft / 2)
      return fail(c, BT_ERR_ARG, "%s: clip %d has %lld samples; reflect padding needs more than %d (torch.stft raises "
                  "for such input as well)", fn, i, (long long)len, cfg->n_fft / 2);
    if (frame_offsets_host[i + 1] - frame_offsets_host[i] != 1 + len / cfg->hop_length)
      return fail(c, BT_ERR_ARG, "%s: frame_offsets do not match 1 + len/%d for clip %d", fn, cfg->hop_length, i);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
  const size_t n = n_clips + 1;
  const int64_t* d[2];
  const int r = stage(c, st, {{sample_offsets_host, n}, {frame_offsets_host, n}}, d);
  if (r != BT_OK) return r;
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
  if (n_clips <= 0) return BT_OK;
  if (!audio_in_dev || !in_offsets_host || !coef_dev || !audio_out_dev || !out_offsets_host)
    return fail(c, BT_ERR_ARG, "bt_resample: null argument");
  if (L <= 0 || M <= 0 || K <= 0 || (K & 1)) return fail(c, BT_ERR_ARG, "bt_resample: need L, M > 0 and an even K > 0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, "bt_resample", st);
  int64_t max_out = 0;
  for (int i = 0; i < n_clips; ++i) {
    if (in_offsets_host[i + 1] < in_offsets_host[i] || out_offsets_host[i + 1] < out_offsets_host[i])
      return fail(c, BT_ERR_ARG, "bt_resample: offsets must be non-decreasing");
    max_out = std::max(max_out, out_offsets_host[i + 1] - out_offsets_host[i]);
  }
  if (max_out > 0 && resample_smem(L, M, K) > kResampleMaxSmem)
    return fail(c, BT_ERR_ARG, "bt_resample: ratio %d/%d with %d taps needs too much shared memory", L, M, K);
  const size_t n = n_clips + 1;
  const int64_t* d[2];
  const int r = stage(c, st, {{in_offsets_host, n}, {out_offsets_host, n}}, d);
  if (r != BT_OK) return r;
  BT_LAUNCHED(c, "resample", st,
              launch_resample(audio_in_dev, d[0], audio_out_dev, d[1], n_clips, max_out, coef_dev, L, M, K, st));
  return BT_OK;
}

// bt_spect2frames(_chunked) under a chunking already checked by chunking_valid; `fn` names the entry point in errors
static int spect2frames(bt_ctx* c, const float* spect_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                        float* beat_dev, float* downbeat_dev, const bt_chunking& ck, void* stream, const char* fn) {
  if (n_clips <= 0) return BT_OK;
  if (!spect_dev || !frame_offsets_host || !beat_dev || !downbeat_dev) return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
  // plan: all chunks of all clips; run_chunks groups them by chunk length
  std::vector<ChunkSrc> all;
  std::vector<int64_t> starts, lens, own_lo, own_hi;
  for (int i = 0; i < n_clips; ++i) {
    const int64_t T = frame_offsets_host[i + 1] - frame_offsets_host[i];
    if (T < 0) return fail(c, BT_ERR_ARG, "%s: negative clip length", fn);
    if (T == 0) continue;
    const int64_t n = plan_chunks(T, ck, nullptr, nullptr, nullptr, nullptr, 0);
    starts.resize(n); lens.resize(n); own_lo.resize(n); own_hi.resize(n);
    plan_chunks(T, ck, starts.data(), lens.data(), own_lo.data(), own_hi.data(), n);
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
  if (!c || !c->finalized) return fail(c, BT_ERR_STATE, "bt_spect2frames: context not finalized");
  return spect2frames(c, spect_dev, frame_offsets_host, n_clips, beat_dev, downbeat_dev, kDefaultChunking, stream,
                      "bt_spect2frames");
}

int bt_spect2frames_chunked(bt_ctx* c, const float* spect_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                            float* beat_dev, float* downbeat_dev, const bt_chunking* ck, void* stream) {
  if (!c || !c->finalized) return fail(c, BT_ERR_STATE, "bt_spect2frames_chunked: context not finalized");
  if (!chunking_valid(ck, c->max_chunk))
    return fail(c, BT_ERR_ARG, "bt_spect2frames_chunked: need 1 <= chunk_size <= %d (bt_max_chunk), 0 <= 2 * border < "
                "chunk_size and overlap_mode BT_KEEP_FIRST or BT_KEEP_LAST", c->max_chunk);
  return spect2frames(c, spect_dev, frame_offsets_host, n_clips, beat_dev, downbeat_dev, *ck, stream,
                      "bt_spect2frames_chunked");
}

int bt_forward_chunks(bt_ctx* c, const float* chunks_dev, int32_t n_chunks, int32_t chunk_frames, float* beat_dev,
                      float* downbeat_dev, void* stream) {
  if (!c || !c->finalized) return fail(c, BT_ERR_STATE, "bt_forward_chunks: context not finalized");
  if (n_chunks <= 0) return BT_OK;
  if (!chunks_dev || !beat_dev || !downbeat_dev) return fail(c, BT_ERR_ARG, "bt_forward_chunks: null argument");
  if (chunk_frames < 1 || chunk_frames > c->max_chunk)
    return fail(c, BT_ERR_ARG, "bt_forward_chunks: chunk_frames must be in [1, %d] (bt_max_chunk)", c->max_chunk);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, "bt_forward_chunks", st);
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

// bt_audio2frames(_chunked) under a chunking already checked by chunking_valid
static int audio2frames(bt_ctx* c, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                        float* beat_dev, float* downbeat_dev, const int64_t* frame_offsets_host, const bt_chunking& ck,
                        void* stream, const char* fn) {
  if (n_clips <= 0) return BT_OK;
  if (!frame_offsets_host) return fail(c, BT_ERR_ARG, "%s: null argument", fn);
  BT_CUDA(c, cudaSetDevice(c->device));
  const int64_t total = frame_offsets_host[n_clips];
  const size_t need = total * 128 * 4;
  BT_CUDA(c, c->spect_ws.reserve(need, need + need / 4));
  int r = bt_logmel(c, audio_dev, sample_offsets_host, n_clips, c->spect_ws.get(), frame_offsets_host, stream);
  if (r != BT_OK) return r;
  return spect2frames(c, c->spect_ws.get(), frame_offsets_host, n_clips, beat_dev, downbeat_dev, ck, stream, fn);
}

int bt_audio2frames(bt_ctx* c, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                    float* beat_dev, float* downbeat_dev, const int64_t* frame_offsets_host, void* stream) {
  if (!c || !c->finalized) return fail(c, BT_ERR_STATE, "bt_audio2frames: context not finalized");
  return audio2frames(c, audio_dev, sample_offsets_host, n_clips, beat_dev, downbeat_dev, frame_offsets_host,
                      kDefaultChunking, stream, "bt_audio2frames");
}

int bt_audio2frames_chunked(bt_ctx* c, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                            float* beat_dev, float* downbeat_dev, const int64_t* frame_offsets_host,
                            const bt_chunking* ck, void* stream) {
  if (!c || !c->finalized) return fail(c, BT_ERR_STATE, "bt_audio2frames_chunked: context not finalized");
  if (!chunking_valid(ck, c->max_chunk))
    return fail(c, BT_ERR_ARG, "bt_audio2frames_chunked: need 1 <= chunk_size <= %d (bt_max_chunk), 0 <= 2 * border < "
                "chunk_size and overlap_mode BT_KEEP_FIRST or BT_KEEP_LAST", c->max_chunk);
  return audio2frames(c, audio_dev, sample_offsets_host, n_clips, beat_dev, downbeat_dev, frame_offsets_host, *ck,
                      stream, "bt_audio2frames_chunked");
}

namespace {

int peakpick(bt_ctx* c, const char* fn, const float* beat_dev, const float* downbeat_dev,
             const int64_t* frame_offsets_host, int32_t n_clips, double* beat_times_dev, int32_t* n_beats_dev,
             double* down_times_dev, int32_t* n_down_dev, int32_t max_peaks, double fps, void* stream) {
  if (!c) return BT_ERR_ARG;
  if (!std::isfinite(fps) || !(fps > 0)) return fail(c, BT_ERR_ARG, "%s: fps must be finite and > 0", fn);
  if (n_clips <= 0) return BT_OK;
  if (!beat_dev || !downbeat_dev || !frame_offsets_host || !beat_times_dev || !n_beats_dev || !down_times_dev ||
      !n_down_dev || max_peaks < 1)
    return fail(c, BT_ERR_ARG, "%s: bad argument", fn);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
  const int64_t* fo = nullptr;
  const int r = stage(c, st, {{frame_offsets_host, static_cast<size_t>(n_clips + 1)}}, &fo);
  if (r != BT_OK) return r;
  launch_peakpick(beat_dev, downbeat_dev, fo, n_clips, beat_times_dev,
                  n_beats_dev, down_times_dev, n_down_dev, max_peaks, fps, st);
  BT_LAUNCHED(c, "peakpick", st);
  return BT_OK;
}

}  // namespace

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

namespace {

// One bar model as the device decodes it: the tables of DbnModelDev, checked, with the kernel's shared-memory need.
struct DbnHostModel {
  int32_t beats = 0, n_int = 0, per_beat = 0;
  std::vector<int32_t> intervals, first, nrun;
  std::vector<double> log_tempo;
  double init = 0.0;
  size_t smem = 0;
};

constexpr size_t kDbnStaticSmem = 512;  // dbn_viterbi_kernel's block reduction

int dbn_host_model(bt_ctx* c, const char* fn, int32_t beats, int32_t n_int, const int32_t* intervals,
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
int dbn_stage(bt_ctx* c, const std::vector<DbnHostModel>& ms, const int64_t* fo, int32_t n_clips, int64_t total,
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

void dbn_launch_shape(const std::vector<DbnHostModel>& ms, int* threads, size_t* smem, size_t* bp_per_frame) {
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

}  // namespace

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
  if (frame_offsets_host[0] < 0) return fail(c, BT_ERR_ARG, "%s: negative frame offset", fn);
  for (int i = 0; i < n_clips; ++i)
    if (frame_offsets_host[i + 1] < frame_offsets_host[i]) return fail(c, BT_ERR_ARG, "%s: frame offsets must not decrease", fn);
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
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  const size_t bp_bytes = std::max<size_t>(bp_per_frame * total, 1);
  BT_CUDA(c, c->dbn_ws.reserve(ws_bytes, ws_bytes + ws_bytes / 4));
  BT_CUDA(c, c->dbn_bp.reserve(bp_bytes, bp_bytes + bp_bytes / 4));
  begin_call(c, fn, st);
  const DbnModelDev* md = nullptr;
  const int64_t* fo_dev = nullptr;
  const int r = dbn_stage(c, ms, frame_offsets_host, n_clips, total, nullptr, st, &md, &fo_dev, nullptr);
  if (r != BT_OK) return r;
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

static_assert(BT_BEAT_METRIC_COLS == kBeatMetricCols, "bt_beat_metrics row width");

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
  for (const int64_t* off : {est_offsets_host, ref_offsets_host}) {
    if (off[0] < 0) return fail(c, BT_ERR_ARG, "%s: negative offset", fn);
    for (int i = 0; i < n_sets; ++i)
      if (off[i + 1] < off[i]) return fail(c, BT_ERR_ARG, "%s: offsets must not decrease", fn);
  }
  if (n_sets == 0) return BT_OK;
  if (!out_dev || (!est_dev && est_offsets_host[n_sets] > 0) || (!ref_dev && ref_offsets_host[n_sets] > 0))
    return fail(c, BT_ERR_ARG, "%s: null device pointer", fn);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
  const size_t n = n_sets + 1;
  const int64_t* off_dev[2];
  const int r = stage(c, st, {{est_offsets_host, n}, {ref_offsets_host, n}}, off_dev);
  if (r != BT_OK) return r;
  launch_beat_metrics(est_dev, off_dev[0], ref_dev, off_dev[1], n_sets, p, out_dev, st);
  BT_LAUNCHED(c, "beat_metrics", st);
  return BT_OK;
}

static_assert(BT_LOSS_MAX_TOLERANCE == kLossMaxTolerance, "bt_loss_params tolerance cap");

namespace {

// The checks bt_beat_loss and its backward share, before anything is enqueued: params, pointers, offsets.  Fills the
// kernels' view of the params, the CTA prefix per row (forward or backward tiling) and the scored frames of all rows.
int loss_prepare(bt_ctx* c, const char* fn, const float* preds, const float* targets, const float* mask,
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
  if (n_rows < 1 || off[0] != 0) return fail(c, BT_ERR_ARG, "%s: need n_rows >= 1 and offsets from 0", fn);
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

}  // namespace

int bt_beat_loss(bt_ctx* c, const float* preds_dev, const float* targets_dev, const float* mask_dev,
                 const int64_t* row_offsets_host, int32_t n_rows, const bt_loss_params* params, double* row_loss_dev,
                 float* mean_dev, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_beat_loss";
  LossParams p;
  std::vector<int64_t> tiles;
  int64_t n_scored = 0;
  int r = loss_prepare(c, fn, preds_dev, targets_dev, mask_dev, row_offsets_host, n_rows, params, false, &p, &tiles,
                       &n_scored);
  if (r != BT_OK) return r;
  if (!row_loss_dev || !mean_dev) return fail(c, BT_ERR_ARG, "%s: null output", fn);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
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
  LossParams p;
  std::vector<int64_t> tiles;
  int64_t n_scored = 0;
  int r = loss_prepare(c, fn, preds_dev, targets_dev, mask_dev, row_offsets_host, n_rows, params, true, &p, &tiles,
                       &n_scored);
  if (r != BT_OK) return r;
  if (!grad_mean_dev || !grad_preds_dev) return fail(c, BT_ERR_ARG, "%s: null gradient pointer", fn);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
  const size_t n = static_cast<size_t>(n_rows) + 1;
  const int64_t* dev[2];
  if ((r = stage(c, st, {{row_offsets_host, n}, {tiles.data(), n}}, dev)) != BT_OK) return r;
  launch_beat_loss_backward(preds_dev, targets_dev, mask_dev, dev[0], dev[1], n_rows, tiles.back(), n_scored, p,
                            grad_mean_dev, grad_preds_dev, st);
  BT_LAUNCHED(c, "beat_loss_backward", st);
  return BT_OK;
}

namespace {

// n_fft of a bt_stft_config as log2, or 0 when it is not a power of two in [64, 8192]
int fft_log2(int n_fft) {
  for (int l = 6; l <= 13; ++l)
    if ((1 << l) == n_fft) return l;
  return 0;
}

// Smallest window envelope sum w^2 over the samples [n_fft / 2, n_fft / 2 + len) that one of F frames covers, for the
// periodic Hann window in float64.  C[i] = w^2[i] + C[i - hop] sums a residue class of the window, so the envelope at
// p is a difference of two entries; the samples between the first and the last n_fft repeat with period hop.
double istft_min_envelope(const std::vector<double>& C, int N, int hop, int64_t F, int64_t len) {
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

}  // namespace

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
  if (sample_offsets_host[0] < 0 || frame_offsets_host[0] != 0)
    return fail(c, BT_ERR_ARG, "%s: sample offsets must start at >= 0 and frame offsets at 0", fn);
  for (int i = 0; i < n_clips; ++i) {
    const int64_t len = sample_offsets_host[i + 1] - sample_offsets_host[i];
    if (len <= cfg->n_fft / 2)
      return fail(c, BT_ERR_ARG, "%s: clip %d has %lld samples; reflect padding needs more than %d", fn, i, (long long)len,
                  cfg->n_fft / 2);
    if (frame_offsets_host[i + 1] - frame_offsets_host[i] != 1 + len / cfg->hop_length)
      return fail(c, BT_ERR_ARG, "%s: frame_offsets do not match 1 + len/%d for clip %d", fn, cfg->hop_length, i);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
  const size_t n = n_clips + 1;
  const int64_t* d[2];
  const int r = stage(c, st, {{sample_offsets_host, n}, {frame_offsets_host, n}}, d);
  if (r != BT_OK) return r;
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
  if (frame_offsets_host[0] != 0 || out_frame_offsets_host[0] != 0)
    return fail(c, BT_ERR_ARG, "%s: frame offsets must start at 0", fn);
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
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
  const VocoderVariant* d[1];
  const int r = stage(c, st, {{variants.data(), variants.size()}}, d);
  if (r != BT_OK) return r;
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
  if (frame_offsets_host[0] != 0 || out_sample_offsets_host[0] < 0)
    return fail(c, BT_ERR_ARG, "%s: frame offsets must start at 0 and sample offsets at >= 0", fn);
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
    if (F < 1 || len < 0) return fail(c, BT_ERR_ARG, "%s: sequence %d needs at least one frame and a length >= 0", fn, s);
    if (len > 0 && istft_min_envelope(C, N, hop, F, len) < 1e-11)
      return fail(c, BT_ERR_ARG, "%s: sequence %d: window envelope below 1e-11 within its %lld samples (torch.istft "
                  "raises there as well)", fn, s, (long long)len);
    max_out = std::max(max_out, len);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BT_CUDA(c, cudaSetDevice(c->device));
  begin_call(c, fn, st);
  const int64_t total_frames = frame_offsets_host[n_seqs];
  const size_t bytes = sizeof(float) * static_cast<size_t>(total_frames) * N;
  BT_CUDA(c, c->istft_frames.reserve(bytes, bytes));
  const size_t n = static_cast<size_t>(n_seqs) + 1;
  const int64_t* d[2];
  const int r = stage(c, st, {{frame_offsets_host, n}, {out_sample_offsets_host, n}}, d);
  if (r != BT_OK) return r;
  BT_LAUNCHED(c, "istft", st,
              launch_istft_frames(log2n, spec_dev, total_frames, window_dev, twiddle_dev, c->istft_frames.get(), st));
  if (max_out > 0) {
    launch_istft_ola(c->istft_frames.get(), d[0], d[1], n_seqs, max_out, window_dev, N, hop, audio_out_dev, st);
    BT_LAUNCHED(c, "istft_overlap_add", st);
  }
  return BT_OK;
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

}  // extern "C"

namespace {

// The public chunk entries as the kernels' ChunkSrc, field by field (the internal layout stays private).
std::vector<ChunkSrc> chunk_table(const bt_debug_chunk* chunks, int32_t n) {
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
int run_chunk_hook(bt_ctx* c, const char* fn, const char* what, const bt_debug_chunk* chunks, int32_t n, void* stream,
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

}  // namespace

extern "C" {

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

}  // extern "C"
