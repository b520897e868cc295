// The training entry points: bt_train_param_count / _info (the reference's state_dict as a table),
// bt_train_activation_bytes(_ex), bt_train_forward(_ex) and bt_train_backward(_ex).  Parameters are the caller's
// unfolded fp32 device tensors; the forward pass saves what the backward pass reads in the caller's activation store.
// A bt_train_mode selects the reference's training-mode function: dropout and batch-statistics BatchNorm.
// bt_adamw_step: the AdamW update of a parameter table in one launch (csrc/kernels_optim.cu).
// Data-parallel training: bt_grad_pack and bt_grad_ordered_sum (csrc/kernels_dp.cu) move a gradient table into and out
// of packed rows, and bt_train_running_replay applies captured batch statistics to the running statistics.
#include "api_internal.h"
#include "bt_train.h"
#include "common.cuh"

namespace {

struct TrParam {
  std::string name;
  int ndim;
  int64_t shape[4];
  bool trainable;
};

// A step of model_steps as the training passes run it.  p: table index of the step's first parameter.  Offsets (in
// floats) into the activation store; -1 where the step saves nothing there.  bn1 / bn2 (training mode): the batch mean
// and, 4-float aligned after it, the biased variance of the step's BatchNorms (the stem: bn1d, bn2d; a convolution: bn2
// of its block's norm).
struct TrLayer : Step {
  int p;
  int64_t in = -1, xn = -1, inv = -1, qkv = -1, gate = -1, lse = -1, o = -1, h = -1, a = -1, z = -1, xl = -1;
  int64_t bn1 = -1, bn2 = -1;
};

// The dropout site numbering of include/beatthis.h: site k (0 or 1) of step `step` of model_steps.  An attention
// step's site 0 is its probabilities and site 1 the output of to_out; a feed-forward step's site 0 is the GELU output
// (net.3) and site 1 the output of net.4 (net.5).
uint32_t dropout_site(size_t step, int k) { return static_cast<uint32_t>(2 * step + k); }

struct TrModel {
  std::vector<TrParam> table;
  std::vector<TrLayer> layers;
  int64_t floats = 0;  // activation store
};

void add(std::vector<TrParam>& t, const std::string& name, std::initializer_list<int64_t> shape, bool trainable = true) {
  TrParam p{name, static_cast<int>(shape.size()), {1, 1, 1, 1}, trainable};
  int i = 0;
  for (int64_t s : shape) p.shape[i++] = s;
  t.push_back(p);
}
void add_bn(std::vector<TrParam>& t, const std::string& p, int n) {
  add(t, p + ".weight", {n});
  add(t, p + ".bias", {n});
  add(t, p + ".running_mean", {n}, false);
  add(t, p + ".running_var", {n}, false);
  add(t, p + ".num_batches_tracked", {}, false);
}
// table order of an attention: rotary_embed.freqs, norm.gamma, to_qkv.weight, to_gates.weight, to_gates.bias,
// to_out.0.weight; of a feed-forward: net.0.gamma, net.1.weight, net.1.bias, net.4.weight, net.4.bias
void add_attn(std::vector<TrParam>& t, const std::string& p, int C) {
  add(t, p + ".rotary_embed.freqs", {16}, false);
  add(t, p + ".norm.gamma", {C});
  add(t, p + ".to_qkv.weight", {3 * C, C});
  add(t, p + ".to_gates.weight", {C / 32, C});
  add(t, p + ".to_gates.bias", {C / 32});
  add(t, p + ".to_out.0.weight", {C, C});
}
void add_ffn(std::vector<TrParam>& t, const std::string& p, int C, int mult) {
  add(t, p + ".net.0.gamma", {C});
  add(t, p + ".net.1.weight", {mult * C, C});
  add(t, p + ".net.1.bias", {mult * C});
  add(t, p + ".net.4.weight", {C, mult * C});
  add(t, p + ".net.4.bias", {C});
}

// The parameter table in BeatThis.state_dict() order and, for a batch of B x L frames (B = 0: table only), the steps
// and their activation store (training mode: the BatchNorms' batch statistics appended).  Token rows of the frontend:
// ((b F + f) L + t), C channels.
TrModel train_model(const bt_hparams& hp, int64_t B, int64_t L, bool train = false) {
  TrModel m;
  auto& t = m.table;
  const int64_t BL = B * L;
  auto alloc = [&](int64_t n) {
    const int64_t off = m.floats;
    m.floats += (n + 3) & ~int64_t{3};
    return off;
  };
  for (const Step& s : model_steps(hp)) {
    TrLayer l{s, static_cast<int>(t.size())};
    const int C = s.C, H = s.mult * C;
    const int64_t M = BL * s.F;
    switch (s.kind) {
      case kStem:
        add_bn(t, s.module + ".bn1d", hp.spect_dim);
        add(t, s.module + ".conv2d.weight", {C, 1, 4, 3});
        add_bn(t, s.module + ".bn2d", C);
        l.in = alloc(BL * hp.spect_dim), l.z = alloc(M * C);
        break;
      case kAttnFreq:
      case kAttnTime:
        add_attn(t, s.module, C);
        l.in = alloc(M * C), l.xn = alloc(M * C), l.inv = alloc(M), l.qkv = alloc(3 * M * C), l.gate = alloc(M * C / 32);
        l.lse = alloc(M * C / 32), l.o = alloc(M * C);
        break;
      case kFfn:
        add_ffn(t, s.module, C, s.mult);
        l.in = alloc(M * C), l.xn = alloc(M * C), l.inv = alloc(M), l.h = alloc(M * H), l.a = alloc(M * H);
        break;
      case kConv:
        add(t, s.module + ".conv2d.weight", {2 * C, C, 2, 3});
        add_bn(t, s.module + ".norm", 2 * C);
        l.in = alloc(M * C), l.z = alloc(M / 2 * 2 * C);
        break;
      case kLinear:
        add(t, s.module + ".weight", {hp.transformer_dim, C * s.F});
        add(t, s.module + ".bias", {hp.transformer_dim});
        l.in = alloc(M * C), l.xl = alloc(M * C);
        break;
      case kHead:
        add(t, "transformer_blocks.norm.gamma", {C});
        add(t, "task_heads.beat_downbeat_lin.weight", {2, C});
        add(t, "task_heads.beat_downbeat_lin.bias", {2});
        l.in = alloc(M * C), l.xn = alloc(M * C), l.inv = alloc(M);
        break;
    }
    m.layers.push_back(l);
  }
  if (train)
    for (TrLayer& l : m.layers) {
      const auto stats = [&](int ch) { return alloc(2 * ((ch + 3) & ~3)); };
      if (l.kind == kStem) l.bn1 = stats(hp.spect_dim), l.bn2 = stats(l.C);
      if (l.kind == kConv) l.bn2 = stats(2 * l.C);
    }
  return m;
}

// Scratch of one call, in floats: the stream gradient, the im2col / FFN-hidden buffer, two [tokens, channels] buffers,
// q/k/v gradients, per-head rows, and split-K / column-sum partials.
struct TrScratch {
  float *dcur, *big, *s1, *s2, *dqkv, *hd1, *hd2, *part;
};
int64_t scratch_floats(int64_t BL) {
  // widest per frame: 1024 channels of tokens (every frontend stage: F C <= 32 * 32 ... 4 * 256; the main layers:
  // D <= 1024), 4096 for the FFN hidden (4 * 32 * 32, or ff_mult D) and the convolutions' im2col (3 * 2 * C * F), 32
  // per-head values (F heads <= 32 in the frontend, D / 32 in the main layers); and one value per channel, at least, for
  // the column sums of the BatchNorm gradients
  return BL * (3 * 1024 + 4096 + 3 * 1024 + 2 * 32) + 2 * 1024 + kTrPartFloats;
}

struct TrRun {
  bt_ctx* c;
  cudaStream_t st;
  const float* const* P;  // parameters, table order
  float* const* G;        // gradients, table order (backward)
  float* act;
  TrScratch s;
  int B, L;
  const float *dbeat, *ddown;  // backward: the gradient at the logits
  const bt_train_mode* mode;   // null: eval mode
  float* const* running;       // training-mode forward: the running statistics to update, table order
  const float* w(int i) const { return P[i]; }
  float* at(int64_t off) const { return act + off; }
  // the BatchNorm at table index p over ch channels: on its running statistics (eval mode) or on the batch statistics
  // the forward pass keeps at store offset off
  TrBn bn(int p, int64_t off, int ch) const {
    if (!mode) return TrBn{P[p], P[p + 1], P[p + 2], P[p + 3]};
    return TrBn{P[p], P[p + 1], at(off), at(off + ((ch + 3) & ~3))};
  }
  // dropout site k of step `step` (none in eval mode), at the frontend rate in a frontend step (F > 1)
  TrDrop drop(const TrLayer& l, size_t step, int k) const {
    if (!mode) return TrDrop{};
    return tr_drop(mode->seed, dropout_site(step, k), l.F > 1 ? mode->dropout_frontend : mode->dropout_transformer);
  }

  // out[M, N] = X[M, K] W[N, K]^T (+ bias) (+ resid) (gelu_out: GELU of it as well), dropout as TrGemmOut states
  int linear(const float* X, int64_t M, int K, const float* W, int N, const float* bias, float* out,
             const float* resid = nullptr, float* gelu_out = nullptr, const TrDrop& drop = {}) {
    launch_tr_gemm({X, K, 1}, {W, K, 1}, {out, N, 0, bias, resid, N, gelu_out, drop}, static_cast<int>(M), N, K, 1, st);
    return check_launch(c, "train_gemm", st);
  }
  // dX[M, K] = dY[M, N] W[N, K] (+ resid)
  int grad_input(const float* dY, int64_t M, int N, const float* W, int K, float* dX, const float* resid = nullptr) {
    launch_tr_gemm({dY, N, 1}, {W, 1, K}, {dX, K, 0, nullptr, resid, K, nullptr}, static_cast<int>(M), K, N, 1, st);
    return check_launch(c, "train_gemm_dx", st);
  }
  // dW[N, K] = dY[M, N]^T X[M, K], split over M with a fixed-order reduction; dW null: not wanted
  int grad_weight(const float* dY, int64_t M, int N, const float* X, int K, float* dW) {
    if (!dW) return BT_OK;
    const int splits = tr_dw_splits(M, N, K);
    const int parts = tr_gemm_parts(static_cast<int>(M), splits);
    launch_tr_gemm({dY, 1, N}, {X, 1, K}, {parts > 1 ? s.part : dW, K, int64_t{N} * K, nullptr, nullptr, 0, nullptr}, N,
                   K, static_cast<int>(M), splits, st);
    if (const int r = check_launch(c, "train_gemm_dw", st)) return r;
    if (parts == 1) return BT_OK;
    launch_tr_reduce(s.part, parts, int64_t{N} * K, 1.f, dW, st);
    return check_launch(c, "train_reduce", st);
  }
  // out[n] = scale sum_m A[m, n] (B[m, n]) (rs[m]); with shift, A centred by shift[n] (squared without B)
  int colsum(const float* A, const float* Bm, const float* rs, int64_t M, int N, float scale, float* out,
             const float* shift = nullptr) {
    if (!out) return BT_OK;
    const int parts = launch_tr_colsum(A, Bm, rs, M, N, tr_colsum_splits(M, N), s.part, st, shift);
    if (const int r = check_launch(c, "train_colsum", st)) return r;
    launch_tr_reduce(s.part, parts, N, scale, out, st);
    return check_launch(c, "train_reduce", st);
  }
  TrSeqs seqs(const TrLayer& l) const {
    const int heads = l.C / 32;
    if (l.kind == kAttnFreq) return {B * L, l.F, heads, L, int64_t{l.F} * L, 1, L};  // sequences (b, t) over f
    return {B * l.F, L, heads, 1, L, 0, 1};                                       // sequences (b, f) over t
  }
  // mask and scale of a [M, N] gradient at a dropout site (the copy reads from, and writes to, other buffers)
  int masked(const float* g, int64_t n, const TrDrop& d, float* out) {
    launch_tr_reduce(g, 1, n, 1.f, out, st, 0.f, d);
    return check_launch(c, "train_reduce", st);
  }
  TrImg img(const TrLayer& l) const {
    if (l.kind == kStem) return {B, l.F, 4, L, 1, int64_t{L} * 4 * l.F, 1, 4 * l.F, 0};  // the [B, L, 128] input
    return {B, l.F / 2, 2, L, l.C, int64_t{l.F} * L * l.C, int64_t{L} * l.C, l.C, 1};
  }
};

#define TR_OK(x)                 \
  do {                           \
    const int _r = (x);          \
    if (_r != BT_OK) return _r;  \
  } while (0)

// The running statistics rm, rv of a BatchNorm of ch channels moved towards a batch mean and biased variance over N
// positions (momentum 0.1, the unbiased variance N / (N - 1)).  The training-mode forward pass and
// bt_train_running_replay make the same launches.
int running_update(bt_ctx* c, cudaStream_t st, const float* mean, const float* var, int64_t N, int ch, float* rm,
                   float* rv) {
  launch_tr_reduce(mean, 1, ch, 0.1f, rm, st, 0.9f);
  TR_OK(check_launch(c, "train_reduce", st));
  launch_tr_reduce(var, 1, ch, static_cast<float>(0.1 * static_cast<double>(N) / static_cast<double>(N - 1)), rv, st,
                   0.9f);
  return check_launch(c, "train_reduce", st);
}

// Training mode: the batch mean and biased variance (two passes: the mean, then centred squares) of x [N, ch] into the
// store at off, and the running statistics of the BatchNorm at table index p moved towards them.
int bn_stats(TrRun& R, const float* x, int64_t N, int ch, int p, int64_t off) {
  float* mean = R.at(off);
  float* var = R.at(off + ((ch + 3) & ~3));
  const float inv_n = static_cast<float>(1.0 / static_cast<double>(N));
  TR_OK(R.colsum(x, nullptr, nullptr, N, ch, inv_n, mean));
  TR_OK(R.colsum(x, nullptr, nullptr, N, ch, inv_n, var, mean));
  return running_update(R.c, R.st, mean, var, N, ch, R.running[p + 2], R.running[p + 3]);
}

// The BatchNorms of a training-mode pass over B x L frames in the order the forward pass updates them: table index p of
// the BatchNorm's weight, offset of its batch mean in the store (its variance follows, 4-float aligned), channels and
// positions N.
struct TrBnStat {
  int p;
  int64_t off;
  int ch;
  int64_t N;
};
std::vector<TrBnStat> bn_stat_list(const TrModel& m, const bt_hparams& hp, int64_t B, int64_t L) {
  std::vector<TrBnStat> out;
  for (const TrLayer& l : m.layers) {
    const int64_t M = B * L * l.F;
    if (l.kind == kStem) out.push_back({l.p, l.bn1, hp.spect_dim, B * L}), out.push_back({l.p + 6, l.bn2, l.C, M});
    if (l.kind == kConv) out.push_back({l.p + 1, l.bn2, 2 * l.C, M / 2});
  }
  return out;
}

// Each step reads l.in and writes the next step's in (the head: the logits).  step: its index in the layer list.
int forward_layer(TrRun& R, const TrLayer& l, size_t step, float* next, float* beat, float* down) {
  const cudaStream_t st = R.st;
  bt_ctx* c = R.c;
  const int64_t M = int64_t{R.B} * R.L * l.F;
  const int C = l.C, p = l.p;
  switch (l.kind) {
    case kStem: {
      const TrImg g = R.img(l);
      const int Fs = c->hp.spect_dim;
      if (R.mode) TR_OK(bn_stats(R, R.at(l.in), int64_t{R.B} * R.L, Fs, p, l.bn1));
      const TrBn bn1 = R.bn(p, l.bn1, Fs);
      launch_tr_im2col(R.at(l.in), g, &bn1, R.s.big, st);
      BT_LAUNCHED(c, "train_im2col", st);
      TR_OK(R.linear(R.s.big, M, 12, R.w(p + 5), C, nullptr, R.at(l.z)));
      if (R.mode) TR_OK(bn_stats(R, R.at(l.z), M, C, p + 6, l.bn2));
      launch_tr_bn_gelu_fwd(R.at(l.z), R.bn(p + 6, l.bn2, C), M * C, C, next, st);
      BT_LAUNCHED(c, "train_bn_gelu", st);
      return BT_OK;
    }
    case kAttnFreq:
    case kAttnTime: {
      const int heads = C / 32;
      launch_tr_rms_fwd(R.at(l.in), R.w(p + 1), M, C, R.at(l.xn), R.at(l.inv), st);
      BT_LAUNCHED(c, "train_rmsnorm", st);
      TR_OK(R.linear(R.at(l.xn), M, C, R.w(p + 2), 3 * C, nullptr, R.at(l.qkv)));
      TR_OK(R.linear(R.at(l.xn), M, C, R.w(p + 3), heads, R.w(p + 4), R.at(l.gate)));
      launch_tr_rope(R.at(l.qkv), R.w(p), M, C, R.L, l.F, l.kind == kAttnFreq, false, st);
      BT_LAUNCHED(c, "train_rope", st);
      launch_tr_attn_fwd(R.at(l.qkv), R.seqs(l), R.at(l.o), R.at(l.lse), st, R.drop(l, step, 0));
      BT_LAUNCHED(c, "train_attention", st);
      launch_tr_gate_fwd(R.at(l.o), R.at(l.gate), M, C, R.s.s1, st);
      BT_LAUNCHED(c, "train_gate", st);
      return R.linear(R.s.s1, M, C, R.w(p + 5), C, nullptr, next, R.at(l.in), nullptr, R.drop(l, step, 1));
    }
    case kFfn: {
      launch_tr_rms_fwd(R.at(l.in), R.w(p), M, C, R.at(l.xn), R.at(l.inv), st);
      BT_LAUNCHED(c, "train_rmsnorm", st);
      TR_OK(R.linear(R.at(l.xn), M, C, R.w(p + 1), l.mult * C, R.w(p + 2), R.at(l.h), nullptr, R.at(l.a),
                     R.drop(l, step, 0)));
      return R.linear(R.at(l.a), M, l.mult * C, R.w(p + 3), C, R.w(p + 4), next, R.at(l.in), nullptr,
                      R.drop(l, step, 1));
    }
    case kConv: {
      const TrImg g = R.img(l);
      const int64_t Mo = M / 2;
      launch_tr_im2col(R.at(l.in), g, nullptr, R.s.big, st);
      BT_LAUNCHED(c, "train_im2col", st);
      TR_OK(R.linear(R.s.big, Mo, 6 * C, R.w(p), 2 * C, nullptr, R.at(l.z)));
      if (R.mode) TR_OK(bn_stats(R, R.at(l.z), Mo, 2 * C, p + 1, l.bn2));
      launch_tr_bn_gelu_fwd(R.at(l.z), R.bn(p + 1, l.bn2, 2 * C), Mo * 2 * C, 2 * C, next, st);
      BT_LAUNCHED(c, "train_bn_gelu", st);
      return BT_OK;
    }
    case kLinear: {
      launch_tr_concat(R.at(l.in), R.B, l.F, R.L, C, false, R.at(l.xl), st);
      BT_LAUNCHED(c, "train_concat", st);
      return R.linear(R.at(l.xl), int64_t{R.B} * R.L, C * l.F, R.w(p), c->hp.transformer_dim, R.w(p + 1), next);
    }
    case kHead: {
      launch_tr_rms_fwd(R.at(l.in), R.w(p), M, C, R.at(l.xn), R.at(l.inv), st);
      BT_LAUNCHED(c, "train_rmsnorm", st);
      TR_OK(R.linear(R.at(l.xn), M, C, R.w(p + 1), 2, R.w(p + 2), R.s.s1));
      launch_tr_head_fwd(R.s.s1, M, c->hp.sum_head, beat, down, st);
      BT_LAUNCHED(c, "train_head", st);
      return BT_OK;
    }
  }
  return BT_OK;
}

// RMSNorm backward of a residual branch: dcur += d(branch)/d(input) from dxn; gamma's gradient.
int rms_backward(TrRun& R, const TrLayer& l, int gamma, const float* dxn, int64_t M, bool add) {
  launch_tr_rms_bwd(dxn, R.at(l.in), R.at(l.inv), R.w(gamma), M, l.C, add, R.s.dcur, R.st);
  BT_LAUNCHED(R.c, "train_rmsnorm_bwd", R.st);
  return R.colsum(dxn, R.at(l.in), R.at(l.inv), M, l.C, sqrtf(static_cast<float>(l.C)), R.G[gamma]);
}

// s.dcur holds the gradient at the step's output; on return, at its input.  Dropout masks are regenerated from the
// forward's sites; BatchNorms use the forward's batch statistics from the store.
int backward_layer(TrRun& R, const TrLayer& l, size_t step, float* dspect) {
  const cudaStream_t st = R.st;
  bt_ctx* c = R.c;
  const int64_t M = int64_t{R.B} * R.L * l.F;
  const int C = l.C, p = l.p;
  float* const* G = R.G;
  const TrScratch& s = R.s;
  switch (l.kind) {
    case kHead: {
      launch_tr_head_bwd(R.dbeat, R.ddown, M, c->hp.sum_head, s.s1, st);
      BT_LAUNCHED(c, "train_head", st);
      TR_OK(R.grad_weight(s.s1, M, 2, R.at(l.xn), C, G[p + 1]));
      TR_OK(R.colsum(s.s1, nullptr, nullptr, M, 2, 1.f, G[p + 2]));
      TR_OK(R.grad_input(s.s1, M, 2, R.w(p + 1), C, s.s2));
      return rms_backward(R, l, p, s.s2, M, false);
    }
    case kAttnFreq:
    case kAttnTime: {
      const int heads = C / 32;
      launch_tr_gate_fwd(R.at(l.o), R.at(l.gate), M, C, s.s1, st);
      BT_LAUNCHED(c, "train_gate", st);
      // to_out's dropout: its GEMMs see the masked gradient (in dqkv, free until the attention passes), the residual
      // path the plain one
      const TrDrop d1 = R.drop(l, step, 1), d0 = R.drop(l, step, 0);
      const float* dy = s.dcur;
      if (d1.thresh) {
        TR_OK(R.masked(s.dcur, M * C, d1, s.dqkv));
        dy = s.dqkv;
      }
      TR_OK(R.grad_weight(dy, M, C, s.s1, C, G[p + 5]));
      TR_OK(R.grad_input(dy, M, C, R.w(p + 5), C, s.s2));
      launch_tr_gate_bwd(s.s2, R.at(l.o), R.at(l.gate), M, C, s.hd1, s.hd2, st);
      BT_LAUNCHED(c, "train_gate_bwd", st);
      const TrSeqs q = R.seqs(l);
      launch_tr_attn_dq(R.at(l.qkv), s.s2, R.at(l.lse), s.hd2, q, s.dqkv, st, d0);
      BT_LAUNCHED(c, "train_attention_dq", st);
      launch_tr_attn_dkv(R.at(l.qkv), s.s2, R.at(l.lse), s.hd2, q, s.dqkv, st, d0);
      BT_LAUNCHED(c, "train_attention_dkv", st);
      launch_tr_rope(s.dqkv, R.w(p), M, C, R.L, l.F, l.kind == kAttnFreq, true, st);
      BT_LAUNCHED(c, "train_rope", st);
      TR_OK(R.grad_weight(s.dqkv, M, 3 * C, R.at(l.xn), C, G[p + 2]));
      TR_OK(R.grad_weight(s.hd1, M, heads, R.at(l.xn), C, G[p + 3]));
      TR_OK(R.colsum(s.hd1, nullptr, nullptr, M, heads, 1.f, G[p + 4]));
      TR_OK(R.grad_input(s.dqkv, M, 3 * C, R.w(p + 2), C, s.s1));
      TR_OK(R.grad_input(s.hd1, M, heads, R.w(p + 3), C, s.s1, s.s1));
      return rms_backward(R, l, p + 1, s.s1, M, true);
    }
    case kFfn: {
      const int H = l.mult * C;
      const TrDrop d1 = R.drop(l, step, 1);
      const float* dy = s.dcur;  // net.5's dropout: the masked gradient to net.4, the plain one to the residual path
      if (d1.thresh) {
        TR_OK(R.masked(s.dcur, M * C, d1, s.s2));
        dy = s.s2;
      }
      TR_OK(R.grad_weight(dy, M, C, R.at(l.a), H, G[p + 3]));
      TR_OK(R.colsum(dy, nullptr, nullptr, M, C, 1.f, G[p + 4]));
      TR_OK(R.grad_input(dy, M, C, R.w(p + 3), H, s.big));
      launch_tr_gelu_bwd(s.big, R.at(l.h), M * H, s.big, st, R.drop(l, step, 0));
      BT_LAUNCHED(c, "train_gelu_bwd", st);
      TR_OK(R.grad_weight(s.big, M, H, R.at(l.xn), C, G[p + 1]));
      TR_OK(R.colsum(s.big, nullptr, nullptr, M, H, 1.f, G[p + 2]));
      TR_OK(R.grad_input(s.big, M, H, R.w(p + 1), C, s.s1));
      return rms_backward(R, l, p, s.s1, M, true);
    }
    case kLinear: {
      const int64_t BL = int64_t{R.B} * R.L;
      const int D = c->hp.transformer_dim, K = C * l.F;
      TR_OK(R.grad_weight(s.dcur, BL, D, R.at(l.xl), K, G[p]));
      TR_OK(R.colsum(s.dcur, nullptr, nullptr, BL, D, 1.f, G[p + 1]));
      TR_OK(R.grad_input(s.dcur, BL, D, R.w(p), K, s.s1));
      launch_tr_concat(s.s1, R.B, l.F, R.L, C, true, s.dcur, st);
      BT_LAUNCHED(c, "train_concat", st);
      return BT_OK;
    }
    case kConv:
    case kStem: {
      // the convolution's output: Mo rows of Co channels, K = Ci S 3 columns of im2col
      const bool stem = l.kind == kStem;
      const TrImg g = R.img(l);
      const int Co = stem ? C : 2 * C, K = g.C * g.S * 3, bn2 = stem ? p + 6 : p + 1, wc = stem ? p + 5 : p;
      const int64_t Mo = int64_t{g.B} * g.Fo * g.L;
      const int64_t BL = int64_t{R.B} * R.L;
      const int Fs = c->hp.spect_dim;
      const TrBn b2 = R.bn(bn2, l.bn2, Co), b1 = stem ? R.bn(p, l.bn1, Fs) : TrBn{};
      launch_tr_bn_gelu_bwd(s.dcur, R.at(l.z), b2, Mo * Co, Co, s.s1, s.s2, st);  // s1: at the BatchNorm, s2: at z
      BT_LAUNCHED(c, "train_bn_gelu_bwd", st);
      TR_OK(R.colsum(s.s1, R.at(l.z), nullptr, Mo, Co, 1.f, s.hd1));
      TR_OK(R.colsum(s.s1, nullptr, nullptr, Mo, Co, 1.f, s.hd2));
      launch_tr_bn_grads(s.hd1, s.hd2, b2, Co, G[bn2], G[bn2 + 1], st);
      BT_LAUNCHED(c, "train_bn_grads", st);
      if (R.mode) {  // batch statistics: the gradient at z gains the terms through the mean and variance
        const TrBnBatch bb{R.at(l.z), s.hd1, s.hd2, static_cast<float>(1.0 / static_cast<double>(Mo))};
        launch_tr_bn_scale(s.s1, b2, Mo * Co, Co, s.s2, st, &bb);
        BT_LAUNCHED(c, "train_bn_scale", st);
      }
      launch_tr_im2col(R.at(l.in), g, stem ? &b1 : nullptr, s.big, st);
      BT_LAUNCHED(c, "train_im2col", st);
      TR_OK(R.grad_weight(s.s2, Mo, Co, s.big, K, G[wc]));
      if (stem && !dspect && !G[p] && !G[p + 1]) return BT_OK;
      TR_OK(R.grad_input(s.s2, Mo, Co, R.w(wc), K, s.big));
      launch_tr_col2im(s.big, g, stem ? s.s1 : s.dcur, st);  // the stem: the gradient at the 1-d BatchNorm's output
      BT_LAUNCHED(c, "train_col2im", st);
      if (!stem) return BT_OK;
      TR_OK(R.colsum(s.s1, R.at(l.in), nullptr, BL, Fs, 1.f, s.hd1));
      TR_OK(R.colsum(s.s1, nullptr, nullptr, BL, Fs, 1.f, s.hd2));
      launch_tr_bn_grads(s.hd1, s.hd2, b1, Fs, G[p], G[p + 1], st);
      BT_LAUNCHED(c, "train_bn_grads", st);
      if (!dspect) return BT_OK;
      const TrBnBatch bb{R.at(l.in), s.hd1, s.hd2, static_cast<float>(1.0 / static_cast<double>(BL))};
      launch_tr_bn_scale(s.s1, b1, BL * Fs, Fs, dspect, st, R.mode ? &bb : nullptr);
      BT_LAUNCHED(c, "train_bn_scale", st);
      return BT_OK;
    }
  }
  return BT_OK;
}

// The checks both passes share, before anything is enqueued.
int train_prepare(bt_ctx* c, const char* fn, const void* const* params, int32_t n_params, int32_t B, int32_t L,
                  const bt_train_mode* mode, const void* act, int64_t act_bytes, TrModel* m) {
  if (c->dtype != BT_DTYPE_F32)
    return fail(c, BT_ERR_ARG, "%s: training runs on a BT_DTYPE_F32 context (fp32 CUDA cores)", fn);
  if (B < 1 || L < 1) return fail(c, BT_ERR_ARG, "%s: need B >= 1 and L >= 1, got B=%d L=%d", fn, B, L);
  if (int64_t{B} * L > kMaxChunkCap)
    return fail(c, BT_ERR_ARG, "%s: B * L = %lld frames exceeds %lld", fn, static_cast<long long>(int64_t{B} * L),
                static_cast<long long>(kMaxChunkCap));
  if (mode) {
    for (const float p : {mode->dropout_frontend, mode->dropout_transformer})
      if (!(p >= 0.f && p < 1.f)) return fail(c, BT_ERR_ARG, "%s: dropout rate %g outside [0, 1)", fn, p);
    // the fewest positions a BatchNorm sees is the stem's bn1d: B * L
    if (int64_t{B} * L < 2)
      return fail(c, BT_ERR_ARG, "%s: batch-statistics BatchNorm needs more than one value per channel, B * L = %lld",
                  fn, static_cast<long long>(int64_t{B} * L));
  }
  *m = train_model(c->hp, B, L, mode != nullptr);
  if (n_params != static_cast<int32_t>(m->table.size()))
    return fail(c, BT_ERR_ARG, "%s: %d parameter pointers, the model has %zu (bt_train_param_count)", fn, n_params,
                m->table.size());
  if (!params || !act) return fail(c, BT_ERR_ARG, "%s: null parameter array or activation store", fn);
  for (size_t i = 0; i < m->table.size(); ++i)
    if (!params[i] && m->table[i].ndim > 0)
      return fail(c, BT_ERR_ARG, "%s: parameter %zu (%s) is null", fn, i, m->table[i].name.c_str());
  if (act_bytes < m->floats * static_cast<int64_t>(sizeof(float)))
    return fail(c, BT_ERR_ARG,
                "%s: activation store of %lld bytes, B=%d L=%d in %s mode needs %lld (bt_train_activation_bytes_ex)", fn,
                static_cast<long long>(act_bytes), B, L, mode ? "training" : "eval",
                static_cast<long long>(m->floats * static_cast<int64_t>(sizeof(float))));
  return BT_OK;
}

// The running statistics every BatchNorm updates: the table and its running_mean / running_var entries must be set.
int check_running(bt_ctx* c, const char* fn, const TrModel& m, float* const* running) {
  if (!running) return fail(c, BT_ERR_ARG, "%s: training mode needs the running-statistics table", fn);
  for (size_t i = 0; i < m.table.size(); ++i) {
    const std::string& n = m.table[i].name;
    const bool stat = n.size() > 13 && (n.compare(n.size() - 13, 13, ".running_mean") == 0 ||
                                        n.compare(n.size() - 12, 12, ".running_var") == 0);
    if (stat && !running[i])
      return fail(c, BT_ERR_ARG, "%s: running-statistics entry %zu (%s) is null", fn, i, n.c_str());
  }
  return BT_OK;
}

// bt_grad_pack's and bt_grad_ordered_sum's device table: the entries with elements, packed densely in table order.
int grad_table(bt_ctx* c, const char* fn, const bt_grad_entry* entries, int32_t n, std::vector<GradEntry>* dev,
               int64_t* chunks) {
  if (n < 0 || (n > 0 && !entries)) return fail(c, BT_ERR_ARG, "%s: need n >= 0 entries, got %d", fn, n);
  int64_t off = 0;
  *chunks = 0;
  for (int32_t i = 0; i < n; ++i) {
    const bt_grad_entry& e = entries[i];
    if (e.numel < 0) return fail(c, BT_ERR_ARG, "%s: entry %d has numel %lld", fn, i, static_cast<long long>(e.numel));
    if (e.numel == 0) continue;
    if (!e.grad) return fail(c, BT_ERR_ARG, "%s: entry %d has a null pointer", fn, i);
    dev->push_back(GradEntry{e.grad, e.numel, off, *chunks});
    off += e.numel;
    *chunks += grad_chunks(e.numel);
  }
  if (*chunks > 0x7fffffff)
    return fail(c, BT_ERR_ARG, "%s: %lld blocks exceed the grid", fn, static_cast<long long>(*chunks));
  return BT_OK;
}

int train_scratch(bt_ctx* c, int64_t BL, TrScratch* s) {
  const int64_t n = scratch_floats(BL);
  BT_CUDA(c, c->train_ws.reserve(n * sizeof(float), n * sizeof(float)));
  float* p = c->train_ws.get();
  auto take = [&](int64_t k) {
    float* r = p;
    p += k;
    return r;
  };
  s->dcur = take(BL * 1024), s->s1 = take(BL * 1024), s->s2 = take(BL * 1024), s->big = take(BL * 4096);
  s->dqkv = take(BL * 3072), s->hd1 = take(BL * 32 + 1024), s->hd2 = take(BL * 32 + 1024);
  s->part = take(kTrPartFloats);
  return BT_OK;
}

}  // namespace

extern "C" {

int32_t bt_train_param_count(const bt_hparams* hp) {
  if (!hp) return BT_ERR_ARG;
  return static_cast<int32_t>(train_model(*hp, 0, 0).table.size());
}

int bt_train_param_info(const bt_hparams* hp, int32_t i, char* name, int32_t cap, int64_t* shape, int32_t* ndim,
                        int32_t* trainable) {
  if (!hp || !name || cap < 1 || !shape || !ndim || !trainable) return BT_ERR_ARG;
  const TrModel m = train_model(*hp, 0, 0);
  if (i < 0 || i >= static_cast<int32_t>(m.table.size())) return BT_ERR_ARG;
  const TrParam& p = m.table[i];
  if (static_cast<int32_t>(p.name.size()) >= cap) return BT_ERR_ARG;
  memcpy(name, p.name.c_str(), p.name.size() + 1);
  for (int k = 0; k < 4; ++k) shape[k] = k < p.ndim ? p.shape[k] : 0;
  *ndim = p.ndim;
  *trainable = p.trainable;
  return BT_OK;
}

int64_t bt_train_activation_bytes_ex(const bt_ctx* c, int32_t B, int32_t L, const bt_train_mode* mode) {
  if (!c || B < 1 || L < 1) return BT_ERR_ARG;
  return train_model(c->hp, B, L, mode != nullptr).floats * static_cast<int64_t>(sizeof(float));
}

int64_t bt_train_activation_bytes(const bt_ctx* c, int32_t B, int32_t L) {
  return bt_train_activation_bytes_ex(c, B, L, nullptr);
}

int bt_train_forward_ex(bt_ctx* c, const float* const* params, int32_t n_params, float* const* running,
                        const float* spect_dev, int32_t B, int32_t L, const bt_train_mode* mode, void* act_dev,
                        int64_t act_bytes, float* beat_dev, float* down_dev, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_train_forward_ex";
  TrModel m;
  int r = train_prepare(c, fn, reinterpret_cast<const void* const*>(params), n_params, B, L, mode, act_dev, act_bytes,
                        &m);
  if (r != BT_OK) return r;
  if (!spect_dev || !beat_dev || !down_dev) return fail(c, BT_ERR_ARG, "%s: null spectrogram or logits pointer", fn);
  if (mode && (r = check_running(c, fn, m, running)) != BT_OK) return r;
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  TrRun R{c, st, params, nullptr, static_cast<float*>(act_dev), {}, B, L, nullptr, nullptr, mode, running};
  if ((r = train_scratch(c, int64_t{B} * L, &R.s)) != BT_OK) return r;
  BT_CUDA(c, cudaMemcpyAsync(R.at(m.layers[0].in), spect_dev, sizeof(float) * B * L * c->hp.spect_dim,
                             cudaMemcpyDeviceToDevice, st));
  for (size_t i = 0; i < m.layers.size(); ++i) {
    float* next = i + 1 < m.layers.size() ? R.at(m.layers[i + 1].in) : nullptr;
    if ((r = forward_layer(R, m.layers[i], i, next, beat_dev, down_dev)) != BT_OK) return r;
  }
  return BT_OK;
}

int bt_train_forward(bt_ctx* c, const float* const* params, int32_t n_params, const float* spect_dev, int32_t B,
                     int32_t L, void* act_dev, int64_t act_bytes, float* beat_dev, float* down_dev, void* stream) {
  return bt_train_forward_ex(c, params, n_params, nullptr, spect_dev, B, L, nullptr, act_dev, act_bytes, beat_dev,
                             down_dev, stream);
}

int bt_train_backward_ex(bt_ctx* c, const float* const* params, int32_t n_params, const void* act_dev,
                         int64_t act_bytes, int32_t B, int32_t L, const bt_train_mode* mode, const float* dbeat_dev,
                         const float* ddown_dev, float* const* grads, float* dspect_dev, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_train_backward_ex";
  TrModel m;
  int r = train_prepare(c, fn, reinterpret_cast<const void* const*>(params), n_params, B, L, mode, act_dev, act_bytes,
                        &m);
  if (r != BT_OK) return r;
  if (!dbeat_dev || !ddown_dev || !grads) return fail(c, BT_ERR_ARG, "%s: null logit gradient or gradient array", fn);
  // an entry that takes no gradient is never written, whatever it holds; every other null entry is skipped
  std::vector<float*> g(grads, grads + m.table.size());
  for (size_t i = 0; i < g.size(); ++i)
    if (!m.table[i].trainable) g[i] = nullptr;
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  TrRun R{c,    st, params, g.data(), static_cast<float*>(const_cast<void*>(act_dev)), {}, B, L, dbeat_dev, ddown_dev,
          mode, nullptr};
  if ((r = train_scratch(c, int64_t{B} * L, &R.s)) != BT_OK) return r;
  for (size_t i = m.layers.size(); i-- > 0;)
    if ((r = backward_layer(R, m.layers[i], i, dspect_dev)) != BT_OK) return r;
  return BT_OK;
}

int bt_train_backward(bt_ctx* c, const float* const* params, int32_t n_params, const void* act_dev, int64_t act_bytes,
                      int32_t B, int32_t L, const float* dbeat_dev, const float* ddown_dev, float* const* grads,
                      float* dspect_dev, void* stream) {
  return bt_train_backward_ex(c, params, n_params, act_dev, act_bytes, B, L, nullptr, dbeat_dev, ddown_dev, grads,
                              dspect_dev, stream);
}

int bt_adamw_step(bt_ctx* c, const bt_adamw_entry* entries, int32_t n, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_adamw_step";
  if (n < 0 || (n > 0 && !entries)) return fail(c, BT_ERR_ARG, "%s: need n >= 0 entries, got %d", fn, n);
  std::vector<AdamwEntry> dev;
  int64_t chunks = 0;
  for (int32_t i = 0; i < n; ++i) {
    const bt_adamw_entry& e = entries[i];
    if (!e.param || !e.exp_avg || !e.exp_avg_sq) return fail(c, BT_ERR_ARG, "%s: entry %d has a null pointer", fn, i);
    if (e.numel < 0) return fail(c, BT_ERR_ARG, "%s: entry %d has numel %lld", fn, i, static_cast<long long>(e.numel));
    for (const double h : {e.lr, e.beta1, e.beta2, e.eps, e.weight_decay})
      if (!std::isfinite(h)) return fail(c, BT_ERR_ARG, "%s: entry %d has a non-finite hyperparameter", fn, i);
    if (e.lr < 0 || e.eps < 0 || !(e.beta1 >= 0 && e.beta1 < 1) || !(e.beta2 >= 0 && e.beta2 < 1) || e.step < 1)
      return fail(c, BT_ERR_ARG, "%s: entry %d needs lr >= 0, eps >= 0, betas in [0, 1) and step >= 1", fn, i);
    if (!e.grad || e.numel == 0) continue;  // torch's rule: a parameter without a gradient is not updated
    // the scalars as torch's foreach path derives them in Python (double), then rounded to fp32
    const double t = static_cast<double>(e.step);
    const double bc1 = 1.0 - std::pow(e.beta1, t), bc2 = 1.0 - std::pow(e.beta2, t);
    const auto aligned = [](const void* q) { return reinterpret_cast<uintptr_t>(q) % 16 == 0; };
    AdamwEntry d{e.param, e.grad, e.exp_avg, e.exp_avg_sq, e.numel, chunks,
                 static_cast<float>(1.0 - e.lr * e.weight_decay), static_cast<float>(1.0 - e.beta1),
                 static_cast<float>(e.beta2), static_cast<float>(1.0 - e.beta2), static_cast<float>(std::pow(bc2, 0.5)),
                 static_cast<float>(e.eps), static_cast<float>(e.lr / bc1 * -1.0), e.weight_decay != 0.0,
                 aligned(e.param) && aligned(e.grad) && aligned(e.exp_avg) && aligned(e.exp_avg_sq)};
    chunks += adamw_chunks(e.numel);
    dev.push_back(d);
  }
  if (chunks > 0x7fffffff) return fail(c, BT_ERR_ARG, "%s: %lld blocks exceed the grid", fn, static_cast<long long>(chunks));
  if (dev.empty()) return BT_OK;
  cudaStream_t st;
  int r;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const AdamwEntry* table = nullptr;
  if ((r = stage(c, st, {{dev.data(), dev.size()}}, &table)) != BT_OK) return r;
  launch_adamw(table, static_cast<int>(dev.size()), chunks, st);
  BT_LAUNCHED(c, "adamw", st);
  return BT_OK;
}

int bt_grad_pack(bt_ctx* c, const bt_grad_entry* entries, int32_t n, float* row_dev, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_grad_pack";
  std::vector<GradEntry> dev;
  int64_t chunks = 0;
  int r = grad_table(c, fn, entries, n, &dev, &chunks);
  if (r != BT_OK) return r;
  if (!row_dev) return fail(c, BT_ERR_ARG, "%s: null row", fn);
  if (dev.empty()) return BT_OK;
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const GradEntry* table = nullptr;
  if ((r = stage(c, st, {{dev.data(), dev.size()}}, &table)) != BT_OK) return r;
  launch_grad_pack(table, static_cast<int>(dev.size()), chunks, row_dev, st);
  BT_LAUNCHED(c, "grad_pack", st);
  return BT_OK;
}

int bt_grad_ordered_sum(bt_ctx* c, const bt_grad_entry* entries, int32_t n, const float* const* rows_host, int32_t k,
                        void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_grad_ordered_sum";
  std::vector<GradEntry> dev;
  int64_t chunks = 0;
  int r = grad_table(c, fn, entries, n, &dev, &chunks);
  if (r != BT_OK) return r;
  if (k < 1 || !rows_host) return fail(c, BT_ERR_ARG, "%s: need k >= 1 rows, got %d", fn, k);
  for (int32_t j = 0; j < k; ++j)
    if (!rows_host[j]) return fail(c, BT_ERR_ARG, "%s: row %d is null", fn, j);
  if (dev.empty()) return BT_OK;
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const GradEntry* table = nullptr;
  const float* const* rows = nullptr;
  if ((r = stage(c, st, {{dev.data(), dev.size()}}, &table)) != BT_OK) return r;
  if ((r = stage(c, st, {{rows_host, static_cast<size_t>(k)}}, &rows)) != BT_OK) return r;
  launch_grad_ordered_sum(table, static_cast<int>(dev.size()), chunks, rows, k, st);
  BT_LAUNCHED(c, "grad_ordered_sum", st);
  return BT_OK;
}

int bt_train_running_replay(bt_ctx* c, float* const* running, int32_t n_params, const float* const* stats_host,
                            int32_t k, int32_t B, int32_t L, void* stream) {
  if (!c) return BT_ERR_ARG;
  const char* fn = "bt_train_running_replay";
  if (B < 1 || L < 1 || int64_t{B} * L < 2)
    return fail(c, BT_ERR_ARG, "%s: need B >= 1, L >= 1 and B * L >= 2, got B=%d L=%d", fn, B, L);
  const TrModel m = train_model(c->hp, B, L, true);
  if (n_params != static_cast<int32_t>(m.table.size()))
    return fail(c, BT_ERR_ARG, "%s: %d running-statistics pointers, the model has %zu (bt_train_param_count)", fn,
                n_params, m.table.size());
  int r = check_running(c, fn, m, running);
  if (r != BT_OK) return r;
  if (k < 0 || (k > 0 && !stats_host)) return fail(c, BT_ERR_ARG, "%s: need k >= 0 micro-batches, got %d", fn, k);
  for (int32_t j = 0; j < k; ++j)
    if (!stats_host[j]) return fail(c, BT_ERR_ARG, "%s: statistics of micro-batch %d are null", fn, j);
  if (k == 0) return BT_OK;
  const int64_t tail = train_model(c->hp, B, L, false).floats;  // the statistics follow the eval-mode layout
  cudaStream_t st;
  if ((r = enter(c, fn, stream, &st)) != BT_OK) return r;
  const std::vector<TrBnStat> bns = bn_stat_list(m, c->hp, B, L);
  for (int32_t j = 0; j < k; ++j)
    for (const TrBnStat& b : bns) {
      const float* mean = stats_host[j] + (b.off - tail);
      TR_OK(running_update(c, st, mean, mean + ((b.ch + 3) & ~3), b.N, b.ch, running[b.p + 2], running[b.p + 3]));
    }
  return BT_OK;
}

}  // extern "C"
