// Internal kernel-launcher interface shared by the .cu files of libbeatthis_sm90.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bt {

constexpr int kHeadDim = 32;
constexpr int kMaxSlabs = 6;

// A GEMM over "planes": output row m = p_out * L + t.  The A operand row for slab s is
//   plane = p_out * plane_mul + plane_add[s],  time = t + t_shift[s]   (zero when time is
// outside [0, L)), columns [0, Kslab) of a row-major [planes_in * L, lda] activation.
// Plain linear: nslab 1.  Conv2d k(2,3) s(2,1) p(0,1): nslab 6 (df,dt).  frontend.linear
// over "b c f t -> b t (c f)": nslab 4 (f).  W is [N, nslab * Kslab] row-major.
struct GemmShape {
  int planes_out;
  int L;
  int N;
  int Kslab;
  int nslab;
  int plane_mul;
  int plane_add[kMaxSlabs];
  int t_shift[kMaxSlabs];
  int lda;
};

// Epilogue description (shared by the fp32 CUDA-core GEMM and the 16-bit wgmma GEMM).
struct EpiParams {
  int kind;            // 0 generic, 1 qkv (RoPE + q scaling), 2 attention gates:
                       //   out_f32[m*heads + n] = sigmoid(acc + bias[n]) for n < heads (N padded to 32)
  const float* bias;   // [N] or null
  int gelu;            // exact-erf GELU after bias
  const float* resid;  // fp32 [M, ldr] added after activation (may alias out_f32) or null
  int ldr;
  float* out_f32;      // optional fp32 output [M, ldo_f32]
  int ldo_f32;
  void* out_act;       // optional activation-dtype output [M, ldo_act]
  int ldo_act;
  // kind 1 (qkv): columns [0,C) q, [C,2C) k, [2C,3C) v, head h = (c % C) / 32
  const float* rope_cos;  // [Lmax, 16]
  const float* rope_sin;
  int C;
  int heads;
  int posmode;  // 0: position = m % L (time attention)   1: position = (m / L) % F (freq attention)
  int F;
  float qscale;  // multiplied into q after RoPE
};

struct ChunkSrc;

// Launchers enqueue their kernel(s) and return void, or, when a host step can fail (cudaFuncSetAttribute, an occupancy
// query), that step's cudaError_t (cudaSuccess otherwise).  None checks the launch itself: the caller does.

// ---- fp32 CUDA-core path -------------------------------------------------------------------
void launch_gemm_simt(const float* A, const float* W, const GemmShape& g, const EpiParams& e,
                      cudaStream_t st);
// qkv [seqs*L, 3C] fp32 (q,k roped; q NOT pre-scaled) -> out [seqs*L, C] (gated)
// chunks != nullptr: sequence s belongs to chunk s / seqs_per_chunk and only its first chunks[..].len keys exist
void launch_attn_time_simt(const float* qkv, const float* gates, float* out, int seqs, int L,
                           int heads, cudaStream_t st, const ChunkSrc* chunks = nullptr, int seqs_per_chunk = 1);
// frequency-direction attention: tokens m = (b*F + f)*L + t, sequences over f (F in {8, 16, 32}).
void launch_attn_freq_simt(const float* qkv, const float* gates, float* out, int B, int F, int L, int heads, float scale,
                           cudaStream_t st);
// rows [len_b, L) of every plane of chunk b <- 0 (the zero padding a k(2,3) convolution sees beyond the end of a
// chunk that is shorter than the wave's padded length).  buf: [nchunks * F, L, C] of elem_bytes-sized elements.
void launch_zero_tail(void* buf, int elem_bytes, const ChunkSrc* chunks, int nchunks, int F, int L, int C, cudaStream_t st);

// ---- shared small kernels (templated on activation dtype inside) ---------------------------
// RMSNorm without gamma (folded into the next weight); optionally also the attention gates
// sigmoid(xn . wg[h] + bg[h]) for h < heads (used when heads <= 2; wg is [>=heads, C] fp32).
void launch_norm(const float* x, void* xn, int64_t M, int C, int act_h16, cudaStream_t st, float* gates = nullptr,
                 const float* wg = nullptr, const float* bg = nullptr, int heads = 0);
// per-chunk source description for the stem (chunk gather from per-clip spectrograms)
struct ChunkSrc {
  int64_t frame_base;  // first frame of the clip inside the concatenated spectrogram
  int32_t T;           // frames in the clip
  int32_t start;       // chunk start frame (may be negative)
  int64_t out_base;    // first frame of the clip inside the concatenated outputs
  int32_t write_lo;    // chunk-local frame range [write_lo, write_hi) this chunk owns
  int32_t write_hi;
  int32_t len;         // frames of this chunk (<= the wave's padded length L): rows [len, L) of its planes are padding
  int32_t pad_;
};
void launch_stem(const float* spect, const ChunkSrc* chunks, int nchunks, int L, const float* bn1_scale,
                 const float* bn1_shift, const float* w, const float* bias, float* out,
                 cudaStream_t st);
void launch_head(const float* x, int D, const float* w, const float* b, const ChunkSrc* chunks,
                 int nchunks, int L, float* beat, float* down, int sum_head, cudaStream_t st);
void launch_peakpick(const float* beat, const float* down, const int64_t* frame_off_dev, int n_clips,
                     double* beat_t, int32_t* n_beat, double* down_t, int32_t* n_down,
                     int max_peaks, double fps, cudaStream_t st);
// ---- DBN post-processor on the device (kernels_dbn.cu) ---------------------------------------------------------
// One bar model of the bar-pointer HMM (dbn_model.h BarModel), tables on the device.  State s = b * per_beat +
// first[k] + p (beat b, tempo k, position p < intervals[k]); positions p < nrun[b * n_int + k] observe the (down)beat
// density, all others the "no beat" one.
struct DbnModelDev {
  const int32_t* intervals;  // [n_int]
  const int32_t* first;      // [n_int]
  const int32_t* nrun;       // [beats * n_int]
  const double* log_tempo;   // [n_int * n_int], row = previous tempo
  double init;               // initial value of every state, -log(S) as the host computes it
  int64_t bp_base;           // this model's back pointers: bp[bp_base + frame * beats * n_int + b * n_int + k]
  int32_t beats, n_int, per_beat, pad_;
};
// Per clip (frame offsets fo_dev): act [frames][2] float64 activations (from the fp32 logit pair, or copied from
// act_in when it is non-null), dens [frames][3] log densities (no beat, beat, downbeat), win[clip] = {first frame,
// frames to decode} of the threshold window (0 frames: no beats).
void launch_dbn_prep(const float* beat, const float* down, const double* act_in, const int64_t* fo_dev, int n_clips,
                     double threshold, double observation_lambda, double* act, double* dens, int64_t* win,
                     cudaStream_t st);
// dynamic shared memory of dbn_viterbi for one model
size_t dbn_viterbi_smem(int beats, int n_int, int per_beat);
// Viterbi of every (clip, model): back pointers into bp, res_logp / res_state [clip * n_models + model] = log-probability
// and final state of the best path.  threads >= max beats * n_int (multiple of 32), smem >= max dbn_viterbi_smem.
cudaError_t launch_dbn_viterbi(const DbnModelDev* models_dev, int n_models, int threads, size_t smem, const double* dens,
                               const int64_t* fo_dev, const int64_t* win, int n_clips, uint8_t* bp, double* res_logp,
                               int64_t* res_state, cudaStream_t st);
// Best model, backtrace and beats of every clip: (time, number) pairs at times / numbers + fo[clip], counts[clip]
// (codes: one byte per frame of scratch).  With path_out non-null (one clip, one model) it writes the state path and
// *logp_out instead.
void launch_dbn_backtrace(const DbnModelDev* models_dev, int n_models, const int64_t* fo_dev, const int64_t* win,
                          int n_clips, const uint8_t* bp, const double* res_logp, const int64_t* res_state,
                          const double* act, uint8_t* codes, int correct, double fps, double* times, int32_t* numbers,
                          int64_t* counts, int64_t* path_out, double* logp_out, cudaStream_t st);

// ---- beat-tracking evaluation (kernels_eval.cu) ------------------------------------------------------------------
// The parameters of bt_beat_metric_params (include/beatthis.h); one row of kBeatMetricCols float64 per set.
struct BeatMetricParams {
  double min_beat_time, f_window, cemgil_sigma, phase_threshold, period_threshold;
};
constexpr int kBeatMetricCols = 12;
// Every set s: estimates est[est_off[s], est_off[s+1]), references ref[ref_off[s], ref_off[s+1]) (sorted, finite,
// non-negative) -> out[s * 12 ..].
void launch_beat_metrics(const double* est, const int64_t* est_off_dev, const double* ref, const int64_t* ref_off_dev,
                         int n_sets, const BeatMetricParams& p, double* out, cudaStream_t st);

// ---- training losses (kernels_loss.cu) ----------------------------------------------------------------------------
// The contract of bt_beat_loss (include/beatthis.h).  Rows are CSR over row_off_dev; tile_first_dev[i] is the first CTA
// of row i ([n_rows + 1], prefix of the per-row tile counts the launchers' loss_tiles gives).
constexpr int kLossTile = 256;
constexpr int kLossMaxTolerance = 64;
struct LossParams {
  int kind, tolerance;
  float pos_weight;
};
// CTAs row i needs: scored frames (forward) or frames (backward) over kLossTile
int64_t loss_tiles(int64_t len, const LossParams& p, bool backward);
// forward: one float64 partial per CTA into partials, then one CTA reduces them in a fixed order into row_loss and
// *mean (n_scored: scored frames of all rows).
void launch_beat_loss(const float* x, const float* y, const float* m, const int64_t* row_off_dev,
                      const int64_t* tile_first_dev, int n_rows, int64_t n_tiles, const LossParams& p, double* partials,
                      cudaStream_t st);
void launch_beat_loss_reduce(const double* partials, const int64_t* row_off_dev, const int64_t* tile_first_dev,
                             int n_rows, int64_t n_tiles, int64_t n_scored, const LossParams& p, double* row_loss,
                             float* mean, cudaStream_t st);
// backward: grad[j] for every frame (gather over the windows covering j).  One launch.
void launch_beat_loss_backward(const float* x, const float* y, const float* m, const int64_t* row_off_dev,
                               const int64_t* tile_first_dev, int n_rows, int64_t n_tiles, int64_t n_scored,
                               const LossParams& p, const float* grad_mean, float* grad, cudaStream_t st);

// ---- signal (kernels_signal.cu) ------------------------------------------------------------------------------------
// The contracts of bt_logmel, bt_logmel_config, bt_resample, bt_stft, bt_phase_vocoder and bt_istft
// (include/beatthis.h).  log2n: 6..13.
void launch_logmel(const float* audio, const int64_t* sample_off_dev, const int64_t* frame_off_dev,
                   int n_clips, int64_t max_frames, const float* window, const float* twiddle,
                   const int32_t* fb_start, const int32_t* fb_ptr, const float* fb_w, float* spect,
                   cudaStream_t st);
// bt_logmel_config's tables, output and scalars (logmel_config_kernel); norm_mode as bt_mel_config
struct MelConfigArgs {
  const float* window;
  const float* twiddle;
  const int32_t* fb_start;
  const int32_t* fb_ptr;
  const float* fb_w;
  float* spect;
  int hop, n_mels, norm_mode;
  float power, log_multiplier;
};
cudaError_t launch_logmel_config(int log2n, const float* audio, const int64_t* sample_off_dev,
                                 const int64_t* frame_off_dev, int n_clips, int64_t total_frames,
                                 const MelConfigArgs& p, cudaStream_t st);
// dynamic shared memory resample_kernel needs for the ratio L/M with K taps; the caller keeps it <= kResampleMaxSmem
int64_t resample_smem(int L, int M, int K);
constexpr int64_t kResampleMaxSmem = 200 * 1024;
cudaError_t launch_resample(const float* in, const int64_t* in_off_dev, float* out, const int64_t* out_off_dev,
                            int n_clips, int64_t max_out, const float* coef, int L, int M, int K, cudaStream_t st);
// spec: interleaved complex fp32, n_fft / 2 + 1 bins per frame.
cudaError_t launch_stft(int log2n, const float* audio, const int64_t* sample_off_dev, const int64_t* frame_off_dev,
                        int n_clips, int64_t total_frames, const float* window, const float* twiddle, int hop, float* spec,
                        cudaStream_t st);
// One time-stretched variant: input frames [in_base, in_base + T) at `rate` -> output frames [out_base, out_base + T_out)
struct VocoderVariant {
  int64_t in_base, out_base, T, T_out;
  double rate;
};
void launch_phase_vocoder(const float* spec, const VocoderVariant* variants_dev, int n_variants, int bins, float* out,
                          cudaStream_t st);
// frames: scratch of total_frames * n_fft floats (the windowed inverse transform of every frame), gathered by the second
// launch into out (sequence s: frames frame_off[s].., samples out_off[s]..); n_seqs <= 65535.
cudaError_t launch_istft_frames(int log2n, const float* spec, int64_t total_frames, const float* window,
                                const float* twiddle, float* frames, cudaStream_t st);
void launch_istft_ola(const float* frames, const int64_t* frame_off_dev, const int64_t* out_off_dev, int n_seqs,
                      int64_t max_out, const float* window, int n_fft, int hop, float* out, cudaStream_t st);

// ---- training batches (kernels_data.cu) -----------------------------------------------------------------------------
// The contract of bt_train_batch (include/beatthis.h); all tables on the device, row_map may be null (identity).
void launch_train_batch(const uint16_t* rows, const int64_t* row_off, int n_items, int length, const int32_t* row_map,
                        const int32_t* beats, const int64_t* beat_off, const int32_t* downs, const int64_t* down_off,
                        uint16_t* spect, uint8_t* truth_beat, uint8_t* truth_downbeat, uint8_t* padding_mask,
                        cudaStream_t st);

// ---- optimizer (kernels_optim.cu) -------------------------------------------------------------------------------------
// One entry of bt_adamw_step's device table: n > 0 elements from p, g, m, v; chunk0, its first chunk of the launch
// (prefix sums of adamw_chunks over the entries before it); vec: all four pointers 16-byte aligned.  The scalars are
// the fp32 values of what the host derived in double: decay = 1 - lr wd (applied when decay_on), w1 = 1 - beta1,
// beta2, w2 = 1 - beta2, bc2_sqrt = (1 - beta2^t)^0.5, eps and step_size = -lr / (1 - beta1^t).
struct AdamwEntry {
  float* p;
  const float* g;
  float* m;
  float* v;
  int64_t n, chunk0;
  float decay, w1, beta2, w2, bc2_sqrt, eps, step_size;
  int32_t decay_on, vec;
};
int64_t adamw_chunks(int64_t n);  // blocks of one entry of n elements
void launch_adamw(const AdamwEntry* entries_dev, int n_entries, int64_t chunks, cudaStream_t st);

// ---- data-parallel gradient exchange (kernels_dp.cu) ----------------------------------------------------------------
// One entry of bt_grad_pack's and bt_grad_ordered_sum's device table: n > 0 elements of grad, at element off of a
// packed row; chunk0, its first chunk of the launch (prefix sums of grad_chunks over the entries before it).
struct GradEntry {
  float* grad;
  int64_t n, off, chunk0;
};
int64_t grad_chunks(int64_t n);  // blocks of one entry of n elements
// row[off + i] = grad[i] for every entry
void launch_grad_pack(const GradEntry* entries_dev, int n_entries, int64_t chunks, float* row, cudaStream_t st);
// grad[i] = ((rows[0][off + i] + rows[1][off + i]) + ...) + rows[k - 1][off + i], fp32 adds in row order; rows_dev: k
// device pointers on the device
void launch_grad_ordered_sum(const GradEntry* entries_dev, int n_entries, int64_t chunks, const float* const* rows_dev,
                             int k, cudaStream_t st);

// ---- FLAC decoding (kernels_flac.cu, flac.cuh) ------------------------------------------------------------------------
// One stream of a bt_flac_decode call on the device: its frame bytes and frame table (entries of 24 bytes: offset,
// first sample, bytes, block size, as bt_flac_frame), its int64 scratch [channels][n_samples] and its first output
// element.
struct FlacStreamDev {
  const uint8_t* bytes;
  const void* frames;
  int64_t* scratch;
  int64_t byte_count, n_frames, n_samples, out_off;
  int32_t channels, bits;
};
// one thread per frame: CRC-16, subframes and decorrelation into the scratch; a malformed frame stores BT_ERR_IO in
// status[stream].  Streams whose status is not BT_OK are skipped.
void launch_flac_frames(const FlacStreamDev* streams_dev, int n_streams, int64_t max_frames, int32_t* status,
                        cudaStream_t st);
// one thread per sample: mode 0 mono fp32, mode 1 float64 [time, channels]; zeros for a stream whose status is not BT_OK
void launch_flac_output(const FlacStreamDev* streams_dev, int n_streams, int64_t max_samples, int mode, void* out,
                        const int32_t* status, cudaStream_t st);

// ---- MP3 decoding (kernels_mp3.cu, mp3.cuh) --------------------------------------------------------------------------
// One stream of a bt_mp3_decode call on the device: its compacted main data and frame table (bt_mp3_frame entries),
// its scratch (one granule record per frame, granule and channel; 2 x channels x 32 x 36 fp32 IMDCT values per frame)
// and its output window.
struct Mp3StreamDev {
  const uint8_t* bytes;
  const void* frames;
  void* recs;
  float* blocks;
  int64_t byte_count, n_frames, skip, n_samples, out_off;
  int32_t channels, rate_index;
};
// one thread per (frame, channel): scalefactors and Huffman lines of both granules (lut: mp3.cuh's lookup tables)
void launch_mp3_granules(const Mp3StreamDev* streams_dev, int n_streams, int64_t max_frames, const uint32_t* lut,
                         int32_t* status, cudaStream_t st);
// one CTA per (frame, granule): requantisation, stereo, reorder, alias reduction, IMDCT of both channels (tables:
// mp3.cuh's kFloatTables floats)
void launch_mp3_hybrid(const Mp3StreamDev* streams_dev, int n_streams, int64_t max_frames, const float* tables,
                       const int32_t* status, cudaStream_t st);
// one CTA per granule of output, max_granules covering every stream's skip + n_samples: overlap-add, polyphase
// synthesis, trim, output mode (0 mono fp32, 1 float64 [time, ch]); zeros where a stream is not decoded
void launch_mp3_synth(const Mp3StreamDev* streams_dev, int n_streams, int64_t max_granules, const float* tables,
                      int mode, void* out, const int32_t* status, cudaStream_t st);

// ---- Ogg Vorbis decoding (kernels_vorbis.cu, vorbis.cuh) -------------------------------------------------------------
namespace vorbis {
struct StreamDev;
}
// one thread per packet: floors and residues into the packet's scratch
void launch_vorbis_packets(const vorbis::StreamDev* streams_dev, int n_streams, int64_t max_packets, int32_t* status,
                           cudaStream_t st);
// one CTA per packet: floor curves, inverse coupling, floor x residue, IMDCT and window (tables: vorbis.cuh's signal
// tables)
void launch_vorbis_blocks(const vorbis::StreamDev* streams_dev, int n_streams, int64_t max_packets, const float* tables,
                          const int32_t* status, cudaStream_t st);
// one thread per output sample, max_samples covering every stream's n_samples: overlap-add, trim, output mode (0 mono
// fp32, 1 float64 [time, ch]); zeros where a stream is not decoded
void launch_vorbis_output(const vorbis::StreamDev* streams_dev, int n_streams, int64_t max_samples, int mode, void* out,
                          const int32_t* status, cudaStream_t st);

void launch_f32_to_h16(const float* in, void* out, int64_t n, cudaStream_t st);
void launch_h16_to_f32(const void* in, float* out, int64_t n, cudaStream_t st);
// [seqs, L, heads*32] fp32 q,k,v -> packed qkv buffer [seqs*L, 3C] of the activation dtype
// (test hooks bt_debug_attention and bt_debug_attention_freq)
void launch_pack_qkv_test(const float* q, const float* k, const float* v, void* qkv, int seqs, int L,
                          int heads, float qscale, int act_h16, cudaStream_t st);

// ---- 16-bit (fp16 or bf16 operands) tensor-core path (wgmma GEMM, mma.sync attention) ---------------------------------
struct TcGemmPlan;  // one launch: its epilogue, tensor maps and launch geometry
// The plan keeps e.  Kinds 0 and 1 read the residual and write their results ([planes_out * L] rows) through tensor
// maps of e.resid / e.out_f32 / e.out_act that the plan encodes; the gates GEMM (kind 2) stores from registers.
// resid_epilogue: the tile width policy of a GEMM that adds the fp32 residual (kernels_gemm.cu).
TcGemmPlan* tc_gemm_plan_create(const void* A_h16, const void* W_h16, const GemmShape& g, int planes_in,
                                bool resid_epilogue, const EpiParams& e, char* err, int errlen);
void tc_gemm_plan_destroy(TcGemmPlan*);
void tc_gemm_plan_tile(const TcGemmPlan*, int* bn, int* bk);  // the (BN, BK) tile the plan launches
void launch_gemm_tc(const TcGemmPlan* plan, cudaStream_t st);

struct TcAttnPlan;
TcAttnPlan* tc_attn_plan_create(const void* qkv_h16, int seqs, int L, int heads, char* err, int errlen);
void tc_attn_plan_destroy(TcAttnPlan*);
void launch_attn_time_tc(const TcAttnPlan* plan, const float* gates, void* out_h16, cudaStream_t st,
                         const ChunkSrc* chunks = nullptr, int seqs_per_chunk = 1);

// frequency-direction attention of the frontend blocks (F, heads) = (32, 1), (16, 2) or (8, 4): qkv [B * F * L, 3C] ->
// out [B * F * L, C], the tokens of launch_attn_freq_simt.  Plan creation fails for any other pair.
struct TcFreqPlan;
TcFreqPlan* tc_freq_plan_create(const void* qkv_h16, void* out_h16, int B, int F, int L, int heads, char* err, int errlen);
void tc_freq_plan_destroy(TcFreqPlan*);
void launch_attn_freq_tc(const TcFreqPlan* plan, const float* gates, float scale, cudaStream_t st);

// fused RMSNorm + FFN + residual for C in {32, 64} (frontend), x updated in place (+ optional 16-bit copy)
struct TcFfPlan;
TcFfPlan* tc_ff_plan_create(const void* w1_h16, const void* w2_h16, int C, int64_t M, const void* o_h16,
                            const void* wout_h16, char* err, int errlen);
void tc_ff_plan_destroy(TcFfPlan*);
void launch_fused_ff(const TcFfPlan* plan, float* X, const float* b1, const float* b2, void* xb_out, cudaStream_t st);

// fused RMSNorm + gates + QKV projection + RoPE for C in {32, 64} (frontend attentions)
struct TcQkvPlan;
TcQkvPlan* tc_qkv_plan_create(const void* wqkv_h16, int C, int64_t M, char* err, int errlen);
void tc_qkv_plan_destroy(TcQkvPlan*);
void launch_fused_qkv(const TcQkvPlan* plan, const float* X, const float* wg, const float* bg, const float* rope_cos,
                      const float* rope_sin, void* qkv, float* gates, int L, int F, int posmode, float qscale,
                      cudaStream_t st);

int tc_init(char* err, int errlen);  // resolves cuTensorMapEncodeTiled, sets smem attributes

}  // namespace bt
