// Private to the C ABI's host files (bt_api.cu, api_signal.cu, api_post.cu, api_data.cu, api_train.cu, api_debug.cu): bt_ctx, the entry prologue
// and argument checks, errors and launch checks, the staging ring, plan slots and the test-hook harness.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/beatthis.h"
#include "bt_kernels.h"
#include "cuda_owned.h"

namespace bt {

struct Param {
  DeviceBuffer<float> f32;
  DeviceBuffer<> b16;
  DeviceBuffer<int32_t> i32;
  int64_t n = 0;
};

// One step of the model.  model_steps lists them in the order BeatThis.forward runs them: the stem; per frontend block
// i < 3 attnF, ffF, attnT, ffT (with partial transformers) and the convolution; frontend.linear; per main layer its
// attention and FFN; the head.  The inference pass (bt_ctx::layers) and the training passes (api_train.cu) both walk
// this one list, and a step's index in it numbers its dropout sites (include/beatthis.h).
enum StepKind { kStem, kAttnFreq, kAttnTime, kFfn, kConv, kLinear, kHead };
struct Step {
  StepKind kind;
  int C, F;            // channels; frequency planes per chunk (F > 1: a frontend step)
  int mult;            // FFN hidden width multiplier
  std::string name;    // packed-parameter prefix, and the tap name of the step's output (frontend.linear's: "frontend")
  std::string module;  // state_dict prefix (the head has none: its entries sit under two modules)
};
std::vector<Step> model_steps(const bt_hparams& hp);

// A step of the inference pass with its packed weights, resolved by bt_finalize in the order of layer_params.
struct Layer : Step {
  const Param* w[4] = {};
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

}  // namespace bt

using namespace bt;

struct bt_ctx {
  int device = 0;
  bt_hparams hp{};
  int dtype = BT_DTYPE_F32;
  bool finalized = false;
  std::map<std::string, Param> params;
  mutable char err[1024] = "";
  const char* call = "";  // the entry point that is launching (enter)
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
  // scratch of bt_train_forward / bt_train_backward (grows on demand)
  DeviceBuffer<float> train_ws;
  // windowed inverse transforms of bt_istft's frames, n_fft floats each (grows on demand)
  DeviceBuffer<float> istft_frames;
  // decoded samples of bt_flac_decode, [channels][n_samples] int64 per stream (grows on demand)
  DeviceBuffer<int64_t> flac_ws;
  // granule records and IMDCT blocks of bt_mp3_decode (grows on demand)
  DeviceBuffer<char> mp3_ws;
  // packet spectra and blocks, floor posts and residue classifications of bt_vorbis_decode (grows on demand)
  DeviceBuffer<char> vorbis_ws;
  // pinned staging + device tables
  StageSlot stage[kStageSlots];
  int stage_next = 0;
  std::vector<Layer> layers;  // model_steps, built by bt_finalize: the stem first, the head last
  // the RoPE tables, resolved in bt_finalize
  const Param *rope_cos = nullptr, *rope_sin = nullptr;

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

namespace bt {

// Longest chunk a ctx takes: the largest frame budget bt_set_wave_chunks allows, so that no wave holds more frames
// than one of kMaxWaveChunks chunks of BT_CHUNK frames (the 32-bit element counts of the kernels stay within that)
constexpr int kMaxWaveChunks = 256;  // bt_set_wave_chunks
constexpr int64_t kMaxChunkCap = static_cast<int64_t>(kMaxWaveChunks) * BT_CHUNK;

int fail(const bt_ctx* c, int code, const char* fmt, ...);
#define BT_CUDA(ctx, call)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (call);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return fail(ctx, BT_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), \
                  __FILE__, __LINE__);                                                       \
  } while (0)

// The prologue of every entry point that launches, once its arguments have passed their checks: sets the ctx's device,
// takes the caller's stream as *st and begins the call: fn is the entry point its launch errors name, and the profile
// gets the reference point of its first kernel.  BT_OK, or BT_ERR_CUDA when the device cannot be set.
int enter(bt_ctx* c, const char* fn, void* stream, cudaStream_t* st);
// Follows every launcher call.  status: what the launcher returned; a failed host step launched nothing.  Otherwise the
// launch is counted (bt_launch_count), profiled as `what`, checked, and under BT_SYNC_DEBUG waited for.
int check_launch(bt_ctx* c, const char* what, cudaStream_t st, cudaError_t status = cudaSuccess);
// check_launch(c, what, st[, status]), returning from the caller on failure
#define BT_LAUNCHED(c, what, st, ...)                       \
  do {                                                      \
    int _r = check_launch(c, what, st, ##__VA_ARGS__);      \
    if (_r != BT_OK) return _r;                             \
  } while (0)
// The host offsets rule (include/beatthis.h, Conventions): off[0 .. n] starts at 0 or at >= 0, as `start` says, and
// does not decrease; BT_ERR_ARG "<fn>: <name> ..." otherwise.
enum OffsetsStart { kFromZero, kFromNonNegative };
int check_offsets(const bt_ctx* c, const char* fn, const char* name, const int64_t* off, int32_t n, OffsetsStart start);
// STFT offsets (bt_logmel, bt_logmel_config, bt_stft): samples from >= 0, frames from 0, 1 + len / hop frames per clip
// of more than n_fft / 2 samples (reflect padding).
int check_stft_frames(const bt_ctx* c, const char* fn, const int64_t* sample_off, const int64_t* frame_off, int32_t n,
                      int n_fft, int hop);

const Param* find_param(const bt_ctx* c, const std::string& name);
int acquire_stage(bt_ctx* c, size_t bytes, StageSlot** out);
int upload_stage(bt_ctx* c, StageSlot* sl, size_t bytes, cudaStream_t st);
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

// Runs a test hook after its own argument checks: enters the call; in the 16-bit context rounds `arrays`; launch(st)
// makes its plans (make_plan) and launches the kernel(s) under test (check_launch: only they are counted and
// profiled); then rounds the out arrays back and synchronises the stream.  Scratch that launch uses must outlive the
// call.
template <class Launch>
int run_hook(bt_ctx* c, const char* fn, void* stream, std::initializer_list<HookArray*> arrays, Launch launch) {
  cudaStream_t st;
  if (const int r = enter(c, fn, stream, &st)) return r;
  const bool tc = c->dtype == BT_DTYPE_H16;
  cudaError_t e = cudaSuccess;
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

// One bar model as the device decodes it: the tables of DbnModelDev, checked, with the kernel's shared-memory need.
struct DbnHostModel {
  int32_t beats = 0, n_int = 0, per_beat = 0;
  std::vector<int32_t> intervals, first, nrun;
  std::vector<double> log_tempo;
  double init = 0.0;
  size_t smem = 0;
};

// The DBN helpers of api_post.cu, which bt_debug_dbn_viterbi shares.
int dbn_host_model(bt_ctx* c, const char* fn, int32_t beats, int32_t n_int, const int32_t* intervals,
                   const double* log_tempo, const int32_t* pointers, DbnHostModel& m);
int dbn_stage(bt_ctx* c, const std::vector<DbnHostModel>& ms, const int64_t* fo, int32_t n_clips, int64_t total,
              const int64_t* win_host, cudaStream_t st, const DbnModelDev** models_dev, const int64_t** fo_dev,
              const int64_t** win_dev);
void dbn_launch_shape(const std::vector<DbnHostModel>& ms, int* threads, size_t* smem, size_t* bp_per_frame);

}  // namespace bt
