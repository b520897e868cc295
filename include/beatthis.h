/*
 * beatthis.h -- C ABI of libbeatthis_sm90.so, the H100 (sm_90a) implementation of the
 * CPJKU/beat_this Audio -> Frames -> Beats inference path.
 *
 * The reference has no FFI: its boundary is the Python API of beat_this/inference.py
 * (Spect2Frames / Audio2Frames / Audio2Beats / File2Beats).  Each entry point below names
 * the reference function (file:line under the reference tree) whose arithmetic it
 * replaces.  beat_this_b200/_lib.py binds these with ctypes; INTEGRATION.md shows the stub
 * a reference maintainer would add.
 *
 * Conventions
 *  - plain C types only; no torch / CUDA types in signatures (streams travel as void*).
 *  - `*_dev` pointers are device pointers on the context's GPU, `*_host` are host pointers.
 *  - ragged batches are CSR style: `offsets[n+1]` (host, int64) into a concatenated buffer.
 *    Offsets never decrease, and offsets[0] is >= 0, or exactly 0 where an entry point says so.
 *    Every ctx entry point checks this before anything is enqueued and returns BT_ERR_ARG
 *    ("<entry point>: <offsets> must ...") otherwise.
 *  - all work is enqueued on the given CUDA stream (cudaStream_t as void*, NULL = default
 *    stream); no hidden device synchronisation except where stated.
 *  - return value: 0 = ok, negative = error (bt_last_error() gives the text).  Nothing
 *    throws across the ABI.  There is NO CPU fallback: without a CUDA device every compute
 *    entry point fails with BT_ERR_CUDA.
 *  - one bt_ctx per GPU; a ctx is not thread-safe (one host thread per ctx).
 */
#ifndef BEATTHIS_H_
#define BEATTHIS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BT_OK 0
#define BT_ERR_ARG (-1)
#define BT_ERR_CUDA (-2)
#define BT_ERR_STATE (-3)
#define BT_ERR_PARAM (-4)
#define BT_ERR_IO (-5)     /* file could not be opened / read */
#define BT_ERR_FORMAT (-6) /* not a file of the container the probe reads (RIFF/WAVE, FLAC, MP3, Ogg Vorbis) that this library decodes
                            * (caller falls back to another decoder) */

#define BT_DTYPE_F32 0  /* fp32 CUDA-core kernels: the reference's float16=False numerics   */
#define BT_DTYPE_H16 1 /* 16-bit tensor-core kernels (wgmma GEMMs, mma.sync attention), fp32 accumulate + fp32 residual stream.  Operand type
                        * fp16 (what the reference's float16=True autocasts to on CUDA, inference.py:245-246);
                        * bt_act_dtype() names it ("f16", or "bf16" for a -DBT_ACT_BF16 build) */

#define BT_SAMPLE_RATE 22050
#define BT_N_FFT 1024
#define BT_HOP 441
#define BT_N_MELS 128
#define BT_CHUNK 1500
#define BT_BORDER 6
#define BT_FPS 50

typedef struct bt_ctx bt_ctx;

/* BeatThis constructor arguments (reference beat_this/model/beat_tracker.py:39-49), as
 * filtered from the checkpoint's hyper_parameters by load_model (inference.py:72-78). */
typedef struct bt_hparams {
  int32_t spect_dim;            /* 128 */
  int32_t transformer_dim;      /* 512 (final*) / 128 (small*) */
  int32_t ff_mult;              /* 4 */
  int32_t n_layers;             /* 6 */
  int32_t head_dim;             /* 32 */
  int32_t stem_dim;             /* 32 */
  int32_t sum_head;             /* 1 */
  int32_t partial_transformers; /* 1 */
} bt_hparams;

/* Library / ABI version (major*100 + minor). */
int bt_version(void);

/* Operand type of the BT_DTYPE_H16 path in this build: "f16" or "bf16". */
const char* bt_act_dtype(void);

/* ---- model lifetime: replaces load_model (inference.py:56-87) ------------------------ */

/* Create a context on CUDA device `device_ordinal` for a model of shape `hp`.
 * compute_dtype: BT_DTYPE_F32 or BT_DTYPE_H16. */
int bt_create(bt_ctx** out, int device_ordinal, const bt_hparams* hp, int compute_dtype);

/* Upload one packed parameter (fp32, host memory, `count` elements) under `name`.
 * The host side (beat_this_b200/weights.py) folds eval-mode BatchNorm and the RMSNorm
 * gamma*sqrt(dim) factors into neighbouring weights and lays convolution / frontend.linear
 * weights out as GEMM operands; names and shapes are listed in DESIGN.md "Packed
 * parameters".  Replaces model.load_state_dict (inference.py:84). */
int bt_set_param(bt_ctx* ctx, const char* name, const float* data_host, int64_t count);

/* Check that every parameter the model shape needs is present, build 16-bit operand copies and TMA
 * descriptors.  After this the weights are immutable.  (model.to(device).eval(), :87)
 * "rope.cos" / "rope.sin" hold the RoPE rotation of positions 0 .. P - 1 ([P, 16] each, rotary_embedding_torch's
 * fp32 cos / sin of pos * freqs); P sets the ctx's maximum chunk length (bt_max_chunk): BT_CHUNK for the reference's
 * inference chunking, more for a model trained on longer sequences.  BT_ERR_PARAM unless both have P x 16 elements
 * with BT_CHUNK <= P <= 256 * BT_CHUNK (the largest frame budget of a wave, bt_set_wave_chunks). */
int bt_finalize(bt_ctx* ctx);

/* The longest chunk this ctx runs (P of its RoPE tables; BT_CHUNK before bt_finalize): bt_spect2frames_chunked,
 * bt_audio2frames_chunked and bt_forward_chunks refuse longer chunks with BT_ERR_ARG before anything is enqueued.
 * BT_ERR_ARG for a NULL ctx. */
int32_t bt_max_chunk(const bt_ctx* ctx);

/* Free everything. */
void bt_destroy(bt_ctx* ctx);

/* Text of the last error on this ctx (or the last bt_create failure when ctx == NULL). */
const char* bt_last_error(const bt_ctx* ctx);

/* ---- host-side planning helpers (pure host, no GPU needed) ---------------------------------- */

/* Number of log-mel frames for `n_samples` samples: 1 + n/441 (torch.stft center=True,
 * preprocessing.py:43-59). */
int64_t bt_num_frames(int64_t n_samples);

/* split_piece (inference.py:100-135) for a piece of T frames with chunk 1500 / border 6 /
 * avoid_short_end: writes up to `cap` chunk starts and lengths, returns the chunk count
 * (or the count needed when cap is too small). */
int64_t bt_plan_chunks(int64_t T, int64_t* starts, int64_t* lens, int64_t cap);

/* How split_predict_aggregate (inference.py:188-230) cuts a piece and stitches it back: split_piece with
 * avoid_short_end=True (:100-135), then aggregate_prediction (:138-185).  bt_plan_chunks, bt_spect2frames and
 * bt_audio2frames use { BT_CHUNK, BT_BORDER, BT_KEEP_FIRST }; PLBeatThis.predict_step (model/pl_module.py:231-266) cuts
 * a border of 2 * tolerance, 0 for the weighted_bce / bce checkpoints. */
#define BT_KEEP_FIRST 0 /* a frame two chunks cover comes from the earlier one */
#define BT_KEEP_LAST 1  /* ... from the later one                              */

typedef struct bt_chunking {
  int32_t chunk_size;   /* model frames per chunk, 1 <= chunk_size <= the maximum chunk (BT_CHUNK, or bt_max_chunk)  */
  int32_t border;       /* frames cut from each side of a chunk's predictions, 0 <= 2 * border < chunk_size       */
  int32_t overlap_mode; /* BT_KEEP_FIRST or BT_KEEP_LAST                                                       */
} bt_chunking;

/* The chunk plan of a piece of T frames under chunking `ck` (c = chunk_size, b = border, step = c - 2b):
 *  - starts s_i = -b + i * step for i = 0 .. ceil(T / step) - 1 (numpy arange(-b, T - b, step)); when T > step the
 *    last start is moved to T - (c - b);
 *  - chunk i covers the piece rows [max(s_i, 0), min(s_i + c, T)), with max(0, -s_i) zero rows on its left and
 *    max(0, min(b, s_i + c - T)) on its right; lens[i] is its length (<= c);
 *  - its predictions lose b frames on each side; what remains lands on [s_i + b, s_i + lens[i] - b), which equals
 *    [s_i + b, s_i + c - b) clipped to [0, T);
 *  - a frame two chunks cover belongs to the earlier chunk (BT_KEEP_FIRST) or the later one (BT_KEEP_LAST):
 *    chunk i owns [own_lo[i], own_hi[i]) in piece frames.
 * No frame is left uncovered (the reference would leave -1000 there): s_0 + b = 0; starts increase and
 * s_{i+1} + b <= s_i + c - b, with s_{i+1} + b < T, so each range reaches the next one's beginning; the last chunk's
 * range ends at T (it starts at T - (c - b), or is the only chunk and T <= step).  Owned ranges are therefore
 * consecutive, non-empty and tile [0, T) exactly.
 * Writes up to `cap` entries of each non-NULL output array and returns the chunk count (the count needed when cap is
 * too small; 0 for T <= 0), or BT_ERR_ARG when ck is NULL or outside the limits above with a maximum chunk of
 * BT_CHUNK.  Pure host: no ctx, no CUDA. */
int64_t bt_plan_chunking(int64_t T, const bt_chunking* ck, int64_t* starts, int64_t* lens, int64_t* own_lo,
                         int64_t* own_hi, int64_t cap);

/* bt_plan_chunking with the maximum chunk `max_chunk` in place of BT_CHUNK (a ctx's bt_max_chunk): the same plan and
 * outputs for 1 <= chunk_size <= max_chunk, BT_ERR_ARG otherwise.  bt_plan_chunking is this with max_chunk =
 * BT_CHUNK.  A piece of T <= chunk_size - 2 * border frames is one chunk: with border 0 and chunk_size >= T the
 * whole piece runs as one sequence, as in the reference. */
int64_t bt_plan_chunking_max(int64_t T, const bt_chunking* ck, int32_t max_chunk, int64_t* starts, int64_t* lens,
                             int64_t* own_lo, int64_t* own_hi, int64_t cap);

/* ---- host front door: Audio2Frames.signal2spect's host half (inference.py:269-276) ------------------ */

#define BT_SIG_F32 0 /* float32 samples                                                         */
#define BT_SIG_F64 1 /* float64 samples (what the reference's load_audio returns)                */
#define BT_SIG_I16 2 /* int16 PCM, scaled by 1/32768 (== soundfile / torchaudio's float decode)  */

/* Mono mix + fp32 cast of n_clips host signals into one host buffer (normally pinned; it is the source of the single
 * H2D copy of a batch): clip i is signals[i], `frames[i]` x `channels[i]` samples, channels-last and contiguous, of
 * type dtypes[i]; its mono fp32 samples land at dst + dst_offsets[i].  The arithmetic is the reference's: the mean
 * over channels in the array's own floating type (numpy `signal.mean(1)`, inference.py:270-271; float64 for PCM),
 * then the cast of `torch.tensor(signal, dtype=torch.float32)` (:276).  Runs on n_threads host threads (<= 0: all);
 * no CUDA, no ctx. */
int bt_stage_audio(const void* const* signals, const int32_t* dtypes, const int64_t* frames,
                   const int32_t* channels, int32_t n_clips, float* dst, const int64_t* dst_offsets,
                   int32_t n_threads);

/* RIFF/WAVE front door of load_audio (preprocessing.py:6-24) for the batched File2Beats path. */
typedef struct bt_wav_info {
  int32_t sample_rate;
  int32_t channels;
  int32_t bytes_per_sample; /* 1, 2, 3, 4 (PCM) or 4, 8 (IEEE float) */
  int32_t is_float;
  int64_t frames;
  int64_t data_offset;      /* byte offset of the first sample in the file */
} bt_wav_info;

/* Parse the header of a WAV file (PCM 8/16/24/32-bit, IEEE float 32/64-bit, incl. WAVE_FORMAT_EXTENSIBLE).
 * BT_ERR_IO: cannot open; BT_ERR_FORMAT: not such a file. */
int bt_wav_probe(const char* path, bt_wav_info* info);

/* Decode n_files probed WAV files on n_threads host threads: samples -> float64 as soundfile would return them
 * (PCM / 2^(bits-1)), mean over channels in float64, fp32 cast -- i.e. load_audio + the host half of
 * signal2spect -- written to dst + dst_offsets[i] (infos[i].frames samples each).  status[i] (optional) receives
 * BT_OK / BT_ERR_IO per file; files that fail are zero-filled and the call returns BT_ERR_IO. */
int bt_stage_wav_files(const char* const* paths, const bt_wav_info* infos, int32_t n_files, float* dst,
                       const int64_t* dst_offsets, int32_t n_threads, int32_t* status);

/* ---- FLAC (ABI 2.17): native decoding of FLAC files (RFC 9639), on the device -------------------------------------
 * The front door of load_audio for FLAC files, and of the batched File2Beats path.  Three steps: bt_flac_probe reads
 * the metadata (host), bt_stage_flac_files reads the frame bytes and finds the frames (host threads), bt_flac_decode
 * decodes every frame of many files in one call (device).  Native FLAC streams only (no Ogg); 1..8 channels, 4..32 bits
 * per sample. */
typedef struct bt_flac_info {
  int32_t sample_rate;
  int32_t channels;        /* 1..8 */
  int32_t bits_per_sample; /* 4..32 */
  int32_t min_block;       /* STREAMINFO's block-size limits */
  int32_t max_block;
  int32_t reserved_;
  int64_t total_samples;   /* samples per channel; 0: unknown (the frames define the length) */
  int64_t frames_offset;   /* byte offset of the first frame in the file */
  int64_t frames_bytes;    /* bytes from there to the end of the file */
  int64_t max_frames;      /* frame-table entries bt_stage_flac_files may need for this file */
  uint8_t md5[16];         /* STREAMINFO's MD5 of the samples (all zero: not given) */
} bt_flac_info;

/* Parse the metadata of a FLAC file: an optional leading ID3v2 tag, the "fLaC" marker, STREAMINFO as the first metadata
 * block, every other block skipped.  max_frames is ceil(total / max(min_block, 16)) + 1 when the total is known, else
 * frames_bytes / 10 + 1 (the shortest frame has 10 bytes).  Host only: no ctx, no GPU.  BT_ERR_IO: cannot open or read;
 * BT_ERR_FORMAT: not a FLAC stream this library decodes (no marker, no or a malformed STREAMINFO, channels or bits per
 * sample outside the limits above, metadata running past the end). */
int bt_flac_probe(const char* path, bt_flac_info* info);

/* One frame of a FLAC file: `offset` bytes from the start of its frame bytes, `bytes` long, holding samples
 * [first_sample, first_sample + block_size) of every channel. */
typedef struct bt_flac_frame {
  int64_t offset;
  int64_t first_sample;
  int32_t bytes;
  int32_t block_size;
} bt_flac_frame;

/* Read n_files probed FLAC files on n_threads host threads (<= 0: all): file i's infos[i].frames_bytes frame bytes go to
 * bytes_dst + byte_offsets[i] (normally pinned memory, the source of one H2D copy), its frame table to frames_dst +
 * frame_offsets[i] (room for infos[i].max_frames entries), its frame count to n_frames[i] and its samples per channel
 * to n_samples[i].  Frames are found by a scan for the sync code; a candidate is a frame only when its header passes
 * CRC-8, its reserved bits and values are valid, its frame number (fixed block size) or sample number (variable)
 * continues the previous frame, and its channels, bits per sample, sample rate and block size agree with STREAMINFO
 * (block size <= max_block).  The first frame starts at the first byte, the last runs to the end of the file.  When
 * STREAMINFO's total is not 0 the block sizes must add up to it.  status[i]: BT_OK, or BT_ERR_IO (cannot read, no valid
 * first frame, a total that disagrees, more frames than max_frames), which leaves n_frames[i] = n_samples[i] = 0; the
 * call returns BT_ERR_IO when a file failed.  No CUDA, no ctx. */
int bt_stage_flac_files(const char* const* paths, const bt_flac_info* infos, int32_t n_files, uint8_t* bytes_dst,
                        const int64_t* byte_offsets, bt_flac_frame* frames_dst, const int64_t* frame_offsets,
                        int64_t* n_frames, int64_t* n_samples, int32_t n_threads, int32_t* status);

/* One stream of a bt_flac_decode call (host table). */
typedef struct bt_flac_stream {
  int64_t byte_offset;  /* its frame bytes start at bytes_dev + byte_offset ... */
  int64_t byte_count;   /* ... and have this many bytes                        */
  int64_t frame_offset; /* its frame table starts at frames_dev + frame_offset  */
  int64_t n_frames;
  int64_t n_samples;    /* per channel                                          */
  int64_t out_offset;   /* element of out_dev where its output starts           */
  int32_t channels;     /* 1..8                                                 */
  int32_t bits_per_sample; /* 4..32                                             */
} bt_flac_stream;

#define BT_FLAC_MONO_F32 0     /* n_samples fp32: the mono mix of bt_stage_wav_files               */
#define BT_FLAC_CHANNELS_F64 1 /* n_samples x channels float64 [time, ch]: what soundfile returns  */

/* Decode n_streams FLAC streams on the device.  For every frame: CRC-16, each subframe (CONSTANT, VERBATIM, FIXED
 * orders 0..4, LPC orders 1..32 with up to 15-bit coefficients and a shift >= 0; wasted bits; Rice residuals with 4- and
 * 5-bit parameters, any partition order, escaped partitions), accumulated in int64; then the channel decorrelation
 * (independent, left/side, side/right, mid/side).  Outputs, per sample t and with v * 2^-(bits-1) taken in float64:
 *  - BT_FLAC_MONO_F32: out_dev (float*)[out_offset + t] = fp32(sum over channels in order / channels), the arithmetic of
 *    bt_stage_wav_files, so a FLAC file and a WAV file of the same samples give the same bits (one channel: one multiply
 *    and one rounding);
 *  - BT_FLAC_CHANNELS_F64: out_dev (double*)[out_offset + t * channels + c].
 * status_dev (n_streams int32, device) is read and written: a stream whose entry is not BT_OK is not decoded and its
 * output is zero-filled; a malformed frame (CRC mismatch, reserved or refused coding, a read past the frame's end, a
 * partition order the block size does not allow, a header that disagrees with the table or the stream, a frame outside
 * the stream's bytes or samples) stores BT_ERR_IO there and zero-fills that stream's output; the other streams still
 * decode.  Every read of a frame is bounded by its own span.  The frame table must cover each stream's samples (what
 * bt_stage_flac_files writes); samples no frame covers are undefined.
 * Needs an int64 scratch of sum(n_samples * channels) values, kept by the ctx and grown on demand (8 bytes per
 * sample and channel: a group of 64 stereo clips of 30 s at 44.1 kHz needs 1.35 GB).  Any ctx will do (a weight-less
 * one too).  Two launches at most, counted and profiled as "flac_frames" (when there is a frame) and "flac_output" (when
 * there is a sample), enqueued on `stream` without synchronisation; the stream table goes through the staging ring.
 * BT_ERR_ARG before anything is enqueued: n_streams < 0 or > 65535, an unknown mode, a NULL pointer (n_streams > 0),
 * a negative count or offset, channels or bits per sample outside the limits. */
int bt_flac_decode(bt_ctx* ctx, const uint8_t* bytes_dev, const bt_flac_frame* frames_dev,
                   const bt_flac_stream* streams_host, int32_t n_streams, int32_t mode, void* out_dev, int32_t* status_dev,
                   void* stream);

/* Test hook: bt_flac_decode's arithmetic on the host, through the same frame decoder (bytes_host, frames_host, out_host
 * and status_host in host memory; the same contract otherwise).  It is a check of the device code on machines without
 * a GPU, not a decoder for the library's callers. */
int bt_debug_flac_decode_host(const uint8_t* bytes_host, const bt_flac_frame* frames_host,
                              const bt_flac_stream* streams_host, int32_t n_streams, int32_t mode, void* out_host,
                              int32_t* status_host);

/* ---- MP3 (ABI 2.18): native decoding of MPEG-1 Layer III files (ISO/IEC 11172-3), on the device --------------------
 * The same three steps as FLAC's: bt_mp3_probe walks the frame headers (host), bt_stage_mp3_files reads each file's
 * frames and lays out their main data (host threads), bt_mp3_decode decodes every frame of many files in one call
 * (device).  32, 44.1 and 48 kHz, mono and stereo; every bitrate, CBR or VBR.  MPEG-2 / 2.5 (LSF), Layers I and II, free
 * format, reserved header values and streams whose rate or channel count changes are refused (BT_ERR_FORMAT). */
typedef struct bt_mp3_info {
  int32_t sample_rate;
  int32_t channels;        /* 1 or 2 */
  int64_t n_frames;        /* audio frames (a Xing / Info frame is not one) */
  int64_t n_samples;       /* output samples per channel, after the gapless trim */
  int64_t skip;            /* decoded samples dropped at the start (encoder delay + 529 when tagged, else 0) */
  int64_t padding;         /* encoder padding of a gapless tag (0: none) */
  int64_t frames_offset;   /* byte range of the audio frames in the file */
  int64_t frames_bytes;
  int64_t max_frames;      /* frame-table entries bt_stage_mp3_files writes for this file */
  int64_t main_bytes;      /* bound on the file's compacted main-data bytes */
  int32_t gapless;         /* 1: a Xing / Info frame with a LAME-style tag whose frame count matches */
  int32_t reserved_;
} bt_mp3_info;

/* Walk the headers of an MP3 file: an optional leading ID3v2 tag (with or without footer), then junk or false syncs
 * until the first header that is followed by two more consistent headers, each at the length the one before gives (or
 * by the end of the file, after a trailing ID3v1 or APEv2 tag); then frame after frame.  Bytes after the last frame with no further frame in
 * them are ignored, and a truncated last frame is dropped.  Host only.  BT_ERR_IO: cannot open or read;
 * BT_ERR_FORMAT: no MPEG-1 Layer III stream as above, or one whose rate or channel count changes.  A stream that loses
 * sync in the middle is probed (n_frames counts the frames before the loss) and refused by bt_stage_mp3_files. */
int bt_mp3_probe(const char* path, bt_mp3_info* info);

/* One frame of a staged MP3 stream. */
typedef struct bt_mp3_frame {
  int64_t main_start;      /* its main data starts at this byte of the stream's compacted main data (may be < 0) */
  int64_t first_sample;    /* its first decoded sample: 1152 x frame index */
  uint32_t header;         /* the 4 header bytes, big-endian */
  int32_t main_bytes;      /* main-data bytes the frame itself carries */
  uint8_t side_info[32];   /* its side info (17 bytes for mono) */
} bt_mp3_frame;

/* Read n_files probed MP3 files on n_threads host threads (<= 0: all): file i's compacted main data (each frame's
 * bytes after header, CRC and side info, back to back; at most infos[i].main_bytes) goes to bytes_dst + byte_offsets[i],
 * its frame table to frames_dst + frame_offsets[i] (infos[i].max_frames entries), the main-data bytes to main_bytes[i]
 * and the frame count to n_frames[i].  status[i]: BT_OK, or BT_ERR_IO (cannot read, lost sync in the middle, a walk
 * that disagrees with the probe), which leaves n_frames[i] = 0; the call returns BT_ERR_IO when a file failed. */
int bt_stage_mp3_files(const char* const* paths, const bt_mp3_info* infos, int32_t n_files, uint8_t* bytes_dst,
                       const int64_t* byte_offsets, bt_mp3_frame* frames_dst, const int64_t* frame_offsets,
                       int64_t* main_bytes, int64_t* n_frames, int32_t n_threads, int32_t* status);

/* One stream of a bt_mp3_decode call (host table). */
typedef struct bt_mp3_stream {
  int64_t byte_offset;  /* its compacted main data starts at bytes_dev + byte_offset ... */
  int64_t byte_count;   /* ... and has this many bytes                                 */
  int64_t frame_offset; /* its frame table starts at frames_dev + frame_offset          */
  int64_t n_frames;
  int64_t skip;         /* decoded samples dropped at the start                          */
  int64_t n_samples;    /* output samples per channel from there                         */
  int64_t out_offset;   /* element of out_dev where its output starts                    */
  int32_t channels;     /* 1 or 2                                                        */
  int32_t sample_rate;  /* 32000, 44100 or 48000                                         */
} bt_mp3_stream;

#define BT_MP3_MONO_F32 BT_FLAC_MONO_F32         /* fp32((sum over channels of double(s_c)) / channels)         */
#define BT_MP3_CHANNELS_F64 BT_FLAC_CHANNELS_F64 /* double(s_c) [time, ch], what torchaudio returns as float64 */

/* Decode n_streams MP3 streams on the device in fp32 (no clipping, no rounding to integers): scalefactors with scfsi,
 * Huffman big-values and count1 regions, requantisation, M/S and intensity stereo, short-block reordering, alias
 * reduction, IMDCT of every block type including mixed blocks, overlap-add and the polyphase synthesis; then decoded
 * samples [skip, skip + n_samples) in the mode's output.  status_dev (n_streams int32, device) is read and written as
 * bt_flac_decode's: a stream whose entry is not BT_OK is not decoded and is zero-filled; a malformed granule
 * (scalefactors or big values past part2_3_length, big_values > 288, table 4 or 14, block type 0 with window switching,
 * main data past the stream's end, a frame entry outside its stream) stores BT_ERR_IO and zero-fills the stream.  A
 * count1 quadruple that overshoots part2_3_length is dropped, and a granule whose main data begins before the stream
 * decodes as zeros (a main-data start more than 511 bytes before the stream is outside it: BT_ERR_IO).  Needs a
 * scratch of 5820 bytes per granule and channel (a 1212-byte granule record and 32 x 36 fp32 IMDCT values), about
 * 20 bytes per output sample of a stereo stream (2.2 GB for 64 stereo clips of 30 s at 44.1 kHz, 14 GB for 64 of four
 * minutes), kept by the ctx and grown on demand.  Three launches at most, counted and profiled as "mp3_granules" and
 * "mp3_hybrid" (when a stream has a frame) and "mp3_synth" (when a stream has an output sample: streams that are not
 * decoded, having no frames or a status that is not BT_OK, are zero-filled by it), enqueued on `stream`.
 * BT_ERR_ARG before anything is enqueued: n_streams < 0 or > 65535, an unknown mode, a NULL pointer (n_streams > 0),
 * a negative count or offset, channels outside 1..2, a sample rate MPEG-1 does not have. */
int bt_mp3_decode(bt_ctx* ctx, const uint8_t* bytes_dev, const bt_mp3_frame* frames_dev,
                  const bt_mp3_stream* streams_host, int32_t n_streams, int32_t mode, void* out_dev, int32_t* status_dev,
                  void* stream);

/* Test hook: bt_mp3_decode's arithmetic on the host, through the same per-lane functions (mp3.cuh); host memory, the
 * same contract otherwise. */
int bt_debug_mp3_decode_host(const uint8_t* bytes_host, const bt_mp3_frame* frames_host,
                             const bt_mp3_stream* streams_host, int32_t n_streams, int32_t mode, void* out_host,
                             int32_t* status_host);

/* ---- Ogg Vorbis (ABI 2.19): native decoding of Vorbis I audio in an Ogg stream, on the device -------------------------
 * The same three steps: bt_vorbis_probe reads the pages and the three Vorbis headers (host), bt_stage_vorbis_files
 * reassembles each file's audio packets and builds its decode tables (host threads), bt_vorbis_decode decodes every
 * packet of many files in one call (device).  1 to 8 channels, block sizes 64 .. 8192, floor type 1, residue types 0, 1
 * and 2.  Floor type 0, more than one logical stream (multiplexed or chained files), a first stream that is not Vorbis
 * (Opus, Ogg FLAC, Speex) and invalid header values are refused (BT_ERR_FORMAT). */
typedef struct bt_vorbis_info {
  int32_t sample_rate;
  int32_t channels;        /* 1 .. 8 */
  int32_t blocksize0;      /* short and long block sizes */
  int32_t blocksize1;
  int64_t n_packets;       /* audio packets: the packet-table entries bt_stage_vorbis_files writes at most */
  int64_t packet_bytes;    /* bound on the audio packets' bytes */
  int64_t table_bytes;     /* the decode tables' bytes */
  int64_t skip;            /* decoded samples dropped at the start (front trim by the first audio page's granule) */
  int64_t n_samples;       /* output samples per channel, after both trims */
} bt_vorbis_info;

/* Read the Ogg pages of a file from byte 0 (capture pattern, version 0, CRC-32 of the header pages, lacing, packets
 * spanning pages) and its identification, comment and setup headers, validating the setup completely; then walk the
 * page headers to the end.  A partial last page is dropped, and the output ends at the granule position of the last
 * whole page.  Host only.  BT_ERR_IO: cannot open or read; BT_ERR_FORMAT: as above. */
int bt_vorbis_probe(const char* path, bt_vorbis_info* info);

/* One audio packet of a staged Vorbis stream. */
typedef struct bt_vorbis_packet {
  int64_t byte_offset;     /* its bytes in the stream's packet bytes */
  int64_t end_sample;      /* decoded samples complete once it is decoded: its own are [the previous one's, this) */
  int64_t block_offset;    /* the block sizes of the stream's packets before it (its scratch) */
  int32_t bytes;
  uint8_t mode;            /* its mode number (as read; the decode refuses one >= the mode count) */
  uint8_t blockflag;       /* 1: a long block */
  uint8_t prev_long;       /* window flags of a long block (0 for a short one) */
  uint8_t next_long;
} bt_vorbis_packet;

/* Read n_files probed Vorbis files on n_threads host threads (<= 0: all), checking every page's CRC and sequence number:
 * file i's audio packets, back to back (at most infos[i].packet_bytes), go to bytes_dst + byte_offsets[i], its decode
 * tables (infos[i].table_bytes) right after them at the next multiple of 4 bytes, its packet table to packets_dst +
 * packet_offsets[i] (infos[i].n_packets entries); the packet bytes to packet_bytes[i], the packet count to n_packets[i]
 * and the sum of the packets' block sizes to block_samples[i].  status[i]: BT_OK, or BT_ERR_IO (cannot read, a CRC or
 * sequence mismatch, a walk that disagrees with the probe), which leaves n_packets[i] = 0; the call returns BT_ERR_IO
 * when a file failed. */
int bt_stage_vorbis_files(const char* const* paths, const bt_vorbis_info* infos, int32_t n_files, uint8_t* bytes_dst,
                          const int64_t* byte_offsets, bt_vorbis_packet* packets_dst, const int64_t* packet_offsets,
                          int64_t* packet_bytes, int64_t* n_packets, int64_t* block_samples, int32_t n_threads,
                          int32_t* status);

/* One stream of a bt_vorbis_decode call (host table). */
typedef struct bt_vorbis_stream {
  int64_t byte_offset;    /* its packet bytes start at bytes_dev + byte_offset ...                  */
  int64_t byte_count;     /* ... and have this many bytes                                           */
  int64_t table_offset;   /* its decode tables start at bytes_dev + table_offset (a multiple of 4)  */
  int64_t table_bytes;
  int64_t packet_offset;  /* its packet table starts at packets_dev + packet_offset                  */
  int64_t n_packets;
  int64_t block_samples;  /* the sum of its packets' block sizes                                    */
  int64_t skip;           /* decoded samples dropped at the start                                   */
  int64_t n_samples;      /* output samples per channel from there                                  */
  int64_t out_offset;     /* element of out_dev where its output starts                             */
  int32_t channels;       /* 1 .. 8                                                                 */
  int32_t sample_rate;
} bt_vorbis_stream;

#define BT_VORBIS_MONO_F32 BT_FLAC_MONO_F32         /* fp32((sum over channels of double(s_c)) / channels)        */
#define BT_VORBIS_CHANNELS_F64 BT_FLAC_CHANNELS_F64 /* double(s_c) [time, ch]                                     */

/* Decode n_streams Vorbis streams on the device in fp32 (no clipping, no rounding to integers): floor1 and residue
 * decode, inverse coupling, floor x residue, IMDCT, window and overlap-add; then decoded samples [skip, skip +
 * n_samples) in the mode's output.  status_dev (n_streams int32, device) is read and written as bt_flac_decode's: a
 * stream whose entry is not BT_OK is not decoded and is zero-filled.  A packet cut short follows the specification's
 * end-of-packet rules (every floor unused when it ends in the floors, the rest of the residue zero when it ends in the
 * residue).  A mode number >= the mode count, a codeword a book does not have and a packet entry outside its stream
 * or out of step with the one before store BT_ERR_IO and zero-fill the stream.  Needs a scratch of 4.5 n + 264 bytes
 * per packet of block size n and channel (about 9.3 bytes per output sample and channel at blocks 256 / 2048: 1.6 GB
 * for 64 stereo clips of 30 s at 44.1 kHz), kept by the ctx and grown on demand.  Three launches at most, counted and
 * profiled as "vorbis_packets" and "vorbis_blocks" (when a stream has a packet) and "vorbis_output" (when a stream has
 * an output sample; streams that are not decoded are zero-filled by it), enqueued on `stream`.  BT_ERR_ARG before
 * anything is enqueued: n_streams < 0 or > 65535, an unknown mode, a NULL pointer (n_streams > 0), a negative count or
 * offset, a table offset that is not a multiple of 4, channels outside 1..8, a sample rate <= 0. */
int bt_vorbis_decode(bt_ctx* ctx, const uint8_t* bytes_dev, const bt_vorbis_packet* packets_dev,
                     const bt_vorbis_stream* streams_host, int32_t n_streams, int32_t mode, void* out_dev,
                     int32_t* status_dev, void* stream);

/* Test hook: bt_vorbis_decode's arithmetic on the host, through the same per-lane functions (vorbis.cuh); host memory,
 * the same contract otherwise. */
int bt_debug_vorbis_decode_host(const uint8_t* bytes_host, const bt_vorbis_packet* packets_host,
                                const bt_vorbis_stream* streams_host, int32_t n_streams, int32_t mode, void* out_host,
                                int32_t* status_host);

/* ---- the hot path ------------------------------------------------------------------------- */

/* LogMelSpect.forward (preprocessing.py:56-59) for n_clips mono 22.05 kHz clips.
 * audio_dev: concatenated fp32 samples; sample_offsets_host[n_clips+1].
 * spect_dev: out, concatenated [T_i,128] fp32 with T_i = bt_num_frames(len_i), laid out
 * at frame_offsets_host[i] (frames; frame_offsets_host[n_clips+1], starting at 0).  Every clip needs more than
 * BT_N_FFT/2 samples.  Any n_clips >= 0 runs in one launch (no limit of the grid applies); n_clips < 0 is BT_ERR_ARG
 * before anything is enqueued, n_clips == 0 does nothing. */
int bt_logmel(bt_ctx* ctx, const float* audio_dev, const int64_t* sample_offsets_host,
              int32_t n_clips, float* spect_dev, const int64_t* frame_offsets_host,
              void* stream);

/* LogMelSpect (preprocessing.py:27-59) with any analysis parameters: torchaudio 2.x MelSpectrogram as the reference
 * constructs it, then log1p(log_multiplier * mel).  Contract, for a mono fp32 clip x of len samples:
 *  - STFT: win_length = n_fft, the caller's window (a periodic Hann window for the reference), center=True with
 *    pad_mode="reflect" (n_fft/2 samples mirrored at each end without repeating the edge), onesided: frame t covers
 *    samples t*hop_length - n_fft/2 ..; T = 1 + len / hop_length frames of n_fft/2 + 1 bins X[t][k].
 *  - normalisation (norm_mode; torchaudio's `normalized`): BT_MEL_NORM_FRAME_LENGTH ("frame_length") scales X by
 *    n_fft^-1/2, BT_MEL_NORM_WINDOW (True or "window") divides it by sqrt(sum window^2), BT_MEL_NORM_NONE (False)
 *    leaves it.  Any other string is a ValueError in Python (torchaudio's _get_spec_norms).
 *  - power: S[t][k] = |X[t][k]|^power for a finite power > 0 (power = 1: the magnitude).  Complex output
 *    (power=None) is not implemented.
 *  - filterbank: torchaudio melscale_fbanks(n_fft/2 + 1, f_min, f_max, n_mels, sample_rate, norm=None, mel_scale) with
 *    mel_scale "slaney" or "htk", frequency grid linspace(0, sample_rate // 2, n_fft/2 + 1) (integer floor: it
 *    matters at odd rates such as 11025 Hz), f_max=None meaning float(sample_rate // 2); f_min > f_max is a
 *    ValueError in Python.  The caller passes it in CSR form: band m has the weights fb_w_dev[fb_ptr_dev[m] ..
 *    fb_ptr_dev[m+1]) on the bins from fb_start_dev[m] on (one contiguous run per band; an all-zero band is an empty
 *    run and gives log1p(0) = 0, as torchaudio does after its warning).
 *  - output: spect_dev [T_i][n_mels] fp32 at frame_offsets_host[i] = log1p(log_multiplier * sum_k S[t][k] fb[k][m]).
 *  - tables (caller-owned, device): window_dev [n_fft], twiddle_dev [n_fft/2] complex fp32 (re, im) pairs
 *    e^{-2 pi i j / n_fft} computed in float64 and rounded, as for bt_logmel's "mel.twiddle".
 * Supported range: n_fft a power of two in [64, 8192], hop_length >= 1, 1 <= n_mels <= 1024, norm_mode one of the
 * three, power finite and > 0, log_multiplier finite; anything else is BT_ERR_ARG (NotImplementedError in Python).
 * Every clip needs more than n_fft/2 samples (torch's reflect padding fails below that); frame_offsets_host must start
 * at 0 and give clip i exactly 1 + len_i / hop_length frames; sample offsets must not decrease.  All of this is
 * checked, and BT_ERR_ARG returned, before anything is enqueued.  Needs no weights (a weight-less ctx is enough).
 * Enqueues only: no synchronisation.  Kernel: logmel_config (profile name). */
#define BT_MEL_NORM_NONE 0
#define BT_MEL_NORM_FRAME_LENGTH 1
#define BT_MEL_NORM_WINDOW 2

typedef struct bt_mel_config {
  int32_t n_fft, hop_length, n_mels, norm_mode;
  float power, log_multiplier;
} bt_mel_config;

int bt_logmel_config(bt_ctx* ctx, const bt_mel_config* cfg, const float* window_dev, const float* twiddle_dev,
                     const int32_t* fb_start_dev, const int32_t* fb_ptr_dev, const float* fb_w_dev,
                     const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                     float* spect_dev, const int64_t* frame_offsets_host, void* stream);

/* Resample front door of Audio2Frames.signal2spect (inference.py:274-275:
 * `soxr.resample(signal, in_rate=sr, out_rate=22050)`), as a device polyphase FIR:
 *   out[n] = sum_k coef[(n*M) mod L][k] * in[floor(n*M/L) - K/2 + 1 + k]   (zeros outside a clip)
 * with sr_out/sr_in = L/M in lowest terms.  coef_dev: [L][K] fp32 bank (the host side designs it,
 * beat_this_b200/preprocessing.py: Kaiser-windowed sinc to soxr-HQ-like targets; parity with
 * soxr itself is unpinned).  in/out: concatenated fp32 clips with host offset arrays
 * [n_clips+1]; out lengths are the caller's (normally round(len*L/M)).  Any n_clips >= 0 runs in one launch (no
 * limit of the grid applies); n_clips < 0, a null pointer, L, M < 1, an odd K or K < 1, bad offsets, or (when any
 * clip has outputs) a ratio whose staged input span of (255*M)/L + K + 2 floats exceeds 200 KB of shared memory is
 * BT_ERR_ARG before anything is enqueued. */
int bt_resample(bt_ctx* ctx, const float* audio_in_dev, const int64_t* in_offsets_host,
                int32_t n_clips, const float* coef_dev, int32_t L, int32_t M, int32_t K,
                float* audio_out_dev, const int64_t* out_offsets_host, void* stream);

/* Host-side Viterbi of the bar-pointer HMM behind Postprocessor(type="dbn") (model/postprocessor.py:29-37,170:
 * madmom DBNDownBeatTrackingProcessor; restated in beat_this_b200/dbn.py, parity with madmom unpinned).
 * No CUDA, no ctx: thread-safe.  log_dens [T][3] = log densities of (no beat, beat, downbeat); the state space is
 * `beats` beats x the positions of every tempo `intervals[n_int]` (frames per beat); log_tempo [n_int][n_int] =
 * log P(tempo f -> tempo k) at a beat boundary; pointers [S] = density column of every state.
 * path_out [T] receives the most probable state sequence, *logp_out its log-probability. */
int bt_dbn_viterbi(const double* log_dens, int64_t T, int32_t beats, int32_t n_int,
                   const int32_t* intervals, const double* log_tempo, const int32_t* pointers,
                   int64_t* path_out, double* logp_out);

/* The whole DBN post-processing step of Postprocessor.postp_dbn (model/postprocessor.py:138-173) for many pieces
 * at once, multi-threaded on the host: activations [total_frames][2] = (beat-but-not-downbeat, downbeat)
 * probabilities as the reference builds them (:159-167), pieces at frame_offsets[n_clips+1].  Model parameters as
 * in madmom's DBNDownBeatTrackingProcessor (reference values: beats_per_bar {3,4}, 55..215 BPM, num_tempi 60,
 * transition_lambda 100, observation_lambda 16, threshold 0.05, correct 1, fps 50).  Piece i writes
 * counts_out[i] (time [s], beat number) pairs at times_out / numbers_out + frame_offsets[i]; downbeats are the
 * entries with number 1.  n_threads <= 0: hardware concurrency. */
int bt_dbn_track(const double* activations, const int64_t* frame_offsets, int32_t n_clips,
                 const int32_t* beats_per_bar, int32_t n_bar_lengths, double min_bpm, double max_bpm,
                 int32_t num_tempi, double transition_lambda, double observation_lambda,
                 double threshold, int32_t correct, double fps, int32_t n_threads,
                 double* times_out, int32_t* numbers_out, int64_t* counts_out);

/* Spect2Frames.spect2frames (inference.py:244-254): split_piece -> BeatThis.forward on
 * every chunk -> aggregate_prediction(keep_first).  spect_dev as produced by bt_logmel.
 * beat_dev / downbeat_dev: out, fp32 logits, concatenated with the same frame offsets. */
int bt_spect2frames(bt_ctx* ctx, const float* spect_dev, const int64_t* frame_offsets_host,
                    int32_t n_clips, float* beat_dev, float* downbeat_dev, void* stream);

/* BeatThis.forward (model/beat_tracker.py:188-192) on n_chunks spectrogram chunks of chunk_frames (<= bt_max_chunk) frames
 * each, chunks_dev = [n_chunks, chunk_frames, 128] fp32: no chunk planning, no borders cut -- the model call inside
 * split_predict_aggregate (inference.py:215), batched.  beat_dev / downbeat_dev: [n_chunks, chunk_frames] fp32. */
int bt_forward_chunks(bt_ctx* ctx, const float* chunks_dev, int32_t n_chunks, int32_t chunk_frames,
                      float* beat_dev, float* downbeat_dev, void* stream);

/* Audio2Frames.__call__ (inference.py:279-281) for already mono, 22.05 kHz fp32 audio:
 * bt_logmel + bt_spect2frames with the spectrogram kept in the ctx workspace. */
int bt_audio2frames(bt_ctx* ctx, const float* audio_dev, const int64_t* sample_offsets_host,
                    int32_t n_clips, float* beat_dev, float* downbeat_dev,
                    const int64_t* frame_offsets_host, void* stream);

/* bt_spect2frames / bt_audio2frames with the pieces cut and stitched by `ck` (see bt_plan_chunking) instead of
 * 1500 / 6 / keep_first: split_predict_aggregate (inference.py:188-230) with any valid chunk_size, border_size and
 * overlap_mode, every chunk of every clip batched into waves.  With { BT_CHUNK, BT_BORDER, BT_KEEP_FIRST } the results
 * are bitwise those of the plain entry points.  BT_ERR_ARG, before anything is enqueued, for an invalid ck; the
 * maximum chunk_size is the ctx's bt_max_chunk. */
int bt_spect2frames_chunked(bt_ctx* ctx, const float* spect_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                            float* beat_dev, float* downbeat_dev, const bt_chunking* ck, void* stream);
int bt_audio2frames_chunked(bt_ctx* ctx, const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips,
                            float* beat_dev, float* downbeat_dev, const int64_t* frame_offsets_host,
                            const bt_chunking* ck, void* stream);

/* Postprocessor("minimal") (model/postprocessor.py:85-136,176-197) on device, for predictions at 50 frames per
 * second: bt_peakpick_fps with fps = 50.
 * Per clip i: beat_times_dev[i*max_peaks ..] (float64 seconds), n_beats_dev[i], same for
 * downbeats.  A clip with more than max_peaks peaks reports the true count (> max_peaks)
 * and stores the first max_peaks. */
int bt_peakpick(bt_ctx* ctx, const float* beat_dev, const float* downbeat_dev,
                const int64_t* frame_offsets_host, int32_t n_clips, double* beat_times_dev,
                int32_t* n_beats_dev, double* down_times_dev, int32_t* n_down_dev,
                int32_t max_peaks, void* stream);

/* Postprocessor("minimal", fps) for predictions at any frame rate (ABI 2.09).  Peaks, the merging of adjacent peaks
 * (float64 running means) and the outputs are those of bt_peakpick; a merged peak frame f becomes the time f / fps,
 * one correctly rounded float64 division, as numpy's beat_frame / fps.  Every downbeat time then moves to the nearest
 * beat time (the first of equally near ones) and the downbeat times are sorted with duplicates removed (np.unique),
 * both on those float64 times.  fps must be finite and > 0: anything else is BT_ERR_ARG before anything is
 * enqueued.  With fps = 50 the outputs are bitwise bt_peakpick's; both launch the same kernel ("peakpick"). */
int bt_peakpick_fps(bt_ctx* ctx, const float* beat_dev, const float* downbeat_dev,
                    const int64_t* frame_offsets_host, int32_t n_clips, double fps, double* beat_times_dev,
                    int32_t* n_beats_dev, double* down_times_dev, int32_t* n_down_dev,
                    int32_t max_peaks, void* stream);

/* Postprocessor("dbn") (model/postprocessor.py:138-173) on the device: the decoder of bt_dbn_track, pinned to it (the
 * same arithmetic, operation for operation, and the same tie-breaks), as three kernels (dbn_prep, dbn_viterbi,
 * dbn_backtrace).  Input is either the fp32 logit pair (sigmoid and clamps of postprocessor.py:139-167 computed on the
 * device in float64) or activations_dev [total][2] float64 as bt_dbn_track takes them; exactly one of the two forms
 * is non-NULL.  Model parameters and the output layout as bt_dbn_track (times/numbers at frame_offsets[i],
 * counts_dev[i]), all on the device.  BT_ERR_ARG, before anything is enqueued, for a model with more than 255 tempi or
 * one whose state space does not fit in the device's shared memory (one CTA holds every state of one bar model).
 * Works on a weight-less ctx.  Enqueues only: no synchronisation (a scratch buffer that has to grow is reallocated). */
int bt_dbn_track_device(bt_ctx* ctx, const float* beat_logits_dev, const float* downbeat_logits_dev,
                        const double* activations_dev, const int64_t* frame_offsets_host, int32_t n_clips,
                        const int32_t* beats_per_bar, int32_t n_bar_lengths, double min_bpm, double max_bpm,
                        int32_t num_tempi, double transition_lambda, double observation_lambda,
                        double threshold, int32_t correct, double fps,
                        double* times_dev, int32_t* numbers_dev, int64_t* counts_dev, void* stream);

/* Test hook (conventions with the others, below bt_debug_tap_count): the device Viterbi alone (dbn_viterbi, then
 * dbn_backtrace for the path), same arguments and meaning as bt_dbn_viterbi (log_dens and the outputs on the device,
 * the model tables on the host).  The pointer table must have the form BarModel builds: in every (beat, tempo) a
 * leading run of 2 (first beat of the bar) or 1 (other beats) followed by 0; anything else is BT_ERR_ARG. */
int bt_debug_dbn_viterbi(bt_ctx* ctx, const double* log_dens_dev, int64_t T, int32_t beats, int32_t n_int,
                         const int32_t* intervals, const double* log_tempo, const int32_t* pointers,
                         int64_t* path_dev, double* logp_dev, void* stream);

/* ---- evaluation: Metrics of model/pl_module.py:320-339 (mir_eval.beat at its defaults) ------------------------- */

typedef struct bt_beat_metric_params {
  double min_beat_time;    /* trim_beats: times < this are dropped from both arrays (reference eval_trim_beats, 5 s) */
  double f_window;         /* F-measure hit window [s] (0.07)                                                       */
  double cemgil_sigma;     /* Cemgil Gaussian width [s] (0.04)                                                      */
  double phase_threshold;  /* continuity phase threshold (0.175)                                                    */
  double period_threshold; /* continuity period threshold (0.175)                                                   */
} bt_beat_metric_params;

#define BT_BEAT_METRIC_COLS 12

/* Beat-tracking scores of n_sets event sets in one launch, one float64 row of BT_BEAT_METRIC_COLS per set at out_dev +
 * 12 * i: n_ref, n_est (after trimming), matches, P, R, F, cemgil, cemgil_max, CMLc, CMLt, AMLc, AMLt.  Set i is the
 * estimates est_dev[est_offsets_host[i], est_offsets_host[i+1]) against the references ref_dev[ref_offsets_host[i], ..).
 * Inputs must be sorted, finite and non-negative (not checked on the device; beat_this_b200/evaluate.py checks).
 * Contract, in float64, mirroring mir_eval.beat:
 *  - trim: keep times >= min_beat_time in both arrays; if either is then empty, every score is 0;
 *  - F-measure: a hit is est - w <= ref <= est + w; matches = size of a maximum matching of hits (greedy over sorted
 *    refs, each taking the earliest unmatched estimate that holds it); P = matches / n_est, R = matches / n_ref,
 *    F = 2PR / (P + R), 0 when P + R == 0;
 *  - variations of the reference: original, off-beat (midpoints r[i] + 0.5 * (r[i+1] - r[i])), double tempo
 *    (r0, m01, r1, ..., r_{n-1}), half tempo r[0::2], half tempo r[1::2];
 *  - Cemgil per variation: sum over its beats of exp(-(d*d) / (2 sigma^2)), d = distance to the nearest estimate, over
 *    0.5 * (n_est + n_variation); cemgil = original, cemgil_max = best of the five;
 *  - continuity per variation: estimate m takes nearest = the lowest index at minimal |e_m - r| (np.argmin).  When
 *    m == 0 or nearest == 0 the intervals are forward (r[k+1] - r[k], e[m+1] - e[m], backward at the last element;
 *    both 0 for a one-element array, as Python's x[-1] makes them), otherwise backward.  m is a candidate when
 *    |d / ref_int| < phase_threshold and |1 - est_int / ref_int| < period_threshold (a zero ref_int fails), and
 *    succeeds when no earlier estimate with the same nearest was a candidate.  Over L = max(n_variation, n_est):
 *    CMLc = longest run of successes / L, CMLt = successes / L on the original; AMLc, AMLt = maxima over the five.
 *    A variation with no beats scores 0 (mir_eval raises there: argmin of an empty array).
 * BT_ERR_ARG, before anything is enqueued, for n_sets < 0, null pointers, offsets that are negative or decrease, or
 * non-finite parameters.  Works on a weight-less ctx.  Enqueues only: no synchronisation. */
int bt_beat_metrics(bt_ctx* ctx, const double* est_dev, const int64_t* est_offsets_host, const double* ref_dev,
                    const int64_t* ref_offsets_host, int32_t n_sets, const bt_beat_metric_params* params,
                    double* out_dev, void* stream);

/* ---- losses: model/loss.py of the reference (MaskedBCELoss, ShiftTolerantBCELoss, SplittedShiftTolerantBCELoss) ---- */

#define BT_LOSS_MASKED_BCE 0           /* MaskedBCELoss, loss.py:9-35                 */
#define BT_LOSS_SHIFT_TOLERANT 1       /* ShiftTolerantBCELoss, loss.py:38-92         */
#define BT_LOSS_SPLIT_SHIFT_TOLERANT 2 /* SplittedShiftTolerantBCELoss, loss.py:95-160 */
#define BT_LOSS_MAX_TOLERANCE 64

typedef struct bt_loss_params {
  int32_t kind;       /* BT_LOSS_*                                                                    */
  int32_t tolerance;  /* t in [0, BT_LOSS_MAX_TOLERANCE]: predictions max-pooled by 2t+1, targets by 4t+1
                       * (ignored by BT_LOSS_MASKED_BCE)                                              */
  float pos_weight;   /* p: weight of positive targets (binary_cross_entropy_with_logits pos_weight) */
} bt_loss_params;

/* Beat tracker training losses over n_rows rows of frames: row i is preds_dev / targets_dev / mask_dev (fp32) at
 * [row_offsets_host[i], row_offsets_host[i+1]).  mask_dev may be NULL (weight 1) except for the split kind.
 * With softplus(z) = log1p(exp(-|z|)) + max(z, 0), the element loss is torch's binary_cross_entropy_with_logits with
 * pos_weight: l(x, y) = (1 - y) x + (1 + (p - 1) y) softplus(-x).  Per kind, for the frames c of a row of length len:
 *  - MASKED_BCE: every frame is scored; term m_c l(x_c, y_c).
 *  - SHIFT_TOLERANT: frames c in [2t, len - 2t) are scored; xs_c = max_{|d|<=t} x_{c+d}, ys_c = max_{|d|<=2t} y_{c+d};
 *    term (y_c + (1 - ys_c)) m_c l(xs_c, y_c).
 *  - SPLIT_SHIFT_TOLERANT: the same frames, xs_c and ys_c; term y_c m_c l(xs_c, y_c) + (1 - ys_c) m_c l(xs_c, ys_c).
 *    Equal to SHIFT_TOLERANT for binary targets, different for soft ones.
 * A loss is the sum of its terms over its number of scored frames (zero-weight frames included, as in torch's mean).
 * row_loss_dev[i] (float64) is the loss of row i alone (the reference's batch-size-1 test step, pl_module.py:99-114,
 * 224-229); *mean_dev (fp32) is the terms of all rows over the scored frames of all rows (for rows of equal length, the
 * reference module's batch mean).  Terms are computed in fp32 and summed in float64, one partial per CTA, the
 * partials reduced in a fixed order by a second launch: results are bitwise repeatable.
 * BT_ERR_ARG, before anything is enqueued, for an unknown kind, a tolerance outside [0, BT_LOSS_MAX_TOLERANCE], a
 * non-finite pos_weight, n_rows < 1, offsets that do not start at 0 or decrease, a row shorter than 4t + 1 frames
 * (1 for MASKED_BCE; torch's max_pool1d raises there), a null pointer, or the split kind without a mask.  Works on a
 * weight-less ctx.  Enqueues only: no synchronisation (the scratch of per-CTA partials grows on demand). */
int bt_beat_loss(bt_ctx* ctx, const float* preds_dev, const float* targets_dev, const float* mask_dev,
                 const int64_t* row_offsets_host, int32_t n_rows, const bt_loss_params* params, double* row_loss_dev,
                 float* mean_dev, void* stream);

/* d(mean)/d(preds) of bt_beat_loss with the same arguments, times the upstream gradient *grad_mean_dev (fp32, read on
 * the device), into grad_preds_dev (every frame written; frames outside the scored range and its pooling windows get
 * 0).  Torch's form per scored frame: ((p y + 1 - y) sigmoid(xs) - p y) w g / N, the sum of the two parts for the split
 * kind; the max-pool routes it to the lowest index that attains the window maximum (max_pool1d_with_indices), and
 * each frame sums the windows it wins in ascending order.  One launch; errors as bt_beat_loss. */
int bt_beat_loss_backward(bt_ctx* ctx, const float* preds_dev, const float* targets_dev, const float* mask_dev,
                          const int64_t* row_offsets_host, int32_t n_rows, const bt_loss_params* params,
                          const float* grad_mean_dev, float* grad_preds_dev, void* stream);

/* ---- tempo and pitch augmentation: the time stretch and pitch shift of launch_scripts/preprocess_audio.py ---------
 * The reference calls pedalboard (Rubber Band) for both; its arithmetic is not in the reference tree, so parity with it
 * is unpinned.  The contract here is the classic phase vocoder as torch.stft -> torchaudio.functional.phase_vocoder ->
 * torch.istft define it, in three calls that share one analysis among any number of variants.  Spectrograms are
 * interleaved complex fp32, n_fft / 2 + 1 bins per frame, the frames of all clips concatenated under CSR frame offsets
 * (host, int64, starting at 0).  window_dev: the periodic Hann window of n_fft fp32 values; twiddle_dev: e^{-2 pi i j /
 * n_fft}, j < n_fft / 2, interleaved fp32.  All three work on a weight-less ctx and only enqueue. */

typedef struct bt_stft_config {
  int32_t n_fft;      /* a power of two in [64, 8192]; win_length = n_fft */
  int32_t hop_length; /* >= 1 */
} bt_stft_config;

#define BT_VOCODER_MIN_RATE 0.25
#define BT_VOCODER_MAX_RATE 4.0

/* Analysis: torch.stft(center=True, pad_mode="reflect", onesided=True, normalized=False).  Clip i (samples
 * [sample_offsets_host[i], sample_offsets_host[i+1]) of audio_dev) gives 1 + len_i / hop_length frames.
 * BT_ERR_ARG, before anything is enqueued, for an unsupported n_fft, hop_length < 1, a negative clip count, a null
 * pointer, frame offsets that do not start at 0 or do not match, or a clip of at most n_fft / 2 samples (reflect
 * padding is undefined there). */
int bt_stft(bt_ctx* ctx, const bt_stft_config* cfg, const float* window_dev, const float* twiddle_dev,
            const float* audio_dev, const int64_t* sample_offsets_host, int32_t n_clips, float* spec_dev,
            const int64_t* frame_offsets_host, void* stream);

/* Phase vocoder: variant v reads the T frames X of clip variant_clip_host[v] at rate r = variant_rate_host[v] (finite,
 * in [BT_VOCODER_MIN_RATE, BT_VOCODER_MAX_RATE]) and writes ceil(T / r) frames (the division and ceil in float64) at
 * out_frame_offsets_host[v].  For output frame j: s_j = j r in float64, i = floor(s_j), alpha = s_j - i, and the frame
 * paired with i is i' = floor(s_j + 1) with the sum rounded to float64 as torchaudio indexes it: i + 1, except where s_j
 * lies within an ulp below an integer, where it is i + 2.  Frames T and T + 1 of X are zero;
 *   magnitude  alpha |X[i']| + (1 - alpha) |X[i]|,
 *   phase      phi_0 = angle X[0],  phi_{j+1} = phi_j + wrap(angle X[i'] - angle X[i] - omega_k) + omega_k,
 * omega_k = pi hop k / (n_fft / 2), wrap(x) = x - 2 pi round(x / 2 pi), angle 0 = 0; output magnitude e^{i phi_j}.
 * Since wrap(x - omega_k) + omega_k = x (mod 2 pi) and only e^{i phi} is written, the kernel accumulates angle X[i'] -
 * angle X[i] in float64, reduced modulo 2 pi after every step, and needs no hop: |error of phi_j| <= (2 j + 1) 2^-21
 * rad (two atan2f of 2 ulp each per step), whatever the size of the unreduced phase.
 * Any number of variants may name the same clip; listing a clip's variants together lets them share its analysis in
 * L2.  Each variant is computed from its own clip and rate alone: bitwise repeatable and independent of the batch.
 * BT_ERR_ARG, before anything is enqueued, for an unsupported n_fft, a null pointer, n_clips or n_variants < 0 or
 * n_variants > 65535, a clip index out of range, a clip without frames, a rate outside the range or not finite, or
 * offsets that do not start at 0 or do not match. */
int bt_phase_vocoder(bt_ctx* ctx, int32_t n_fft, const float* spec_dev, const int64_t* frame_offsets_host,
                     int32_t n_clips, const int32_t* variant_clip_host, const double* variant_rate_host,
                     int32_t n_variants, float* out_dev, const int64_t* out_frame_offsets_host, void* stream);

/* Synthesis: torch.istft(center=True, length=len_s) of each of n_seqs sequences of frames: the inverse real FFT of
 * every frame (the imaginary parts of bins 0 and n_fft / 2 ignored) times the window, overlap-added at p = f
 * hop_length, divided by the envelope sum w^2 of the frames that cover p, the first n_fft / 2 samples removed, cut or
 * zero-extended to len_s = out_sample_offsets_host[s+1] - out_sample_offsets_host[s].  Every output sample gathers its
 * frames in ascending order (no atomics): bitwise repeatable and independent of the batch.  The windowed frames pass
 * through ctx scratch of 4 n_fft bytes per frame, which grows on demand.
 * BT_ERR_ARG, before anything is enqueued, for the bt_stft_config errors, a null pointer, n_seqs < 0 or > 65535,
 * offsets that decrease or frame offsets that do not start at 0, a sequence without frames, or an envelope (of the
 * periodic Hann window, evaluated in float64 on the host) below 1e-11 at a sample some frame covers, as torch.istft
 * refuses it: hop_length >= n_fft, or a length that reaches the last samples of the last frame. */
int bt_istft(bt_ctx* ctx, const bt_stft_config* cfg, const float* window_dev, const float* twiddle_dev,
             const float* spec_dev, const int64_t* frame_offsets_host, int32_t n_seqs, float* audio_out_dev,
             const int64_t* out_sample_offsets_host, void* stream);

/* ---- training batches: BeatTrackingDataset.__getitem__ + default_collate (dataset.py:169-241, augment.py:129-201) --
 * Assembles n_items excerpts of `length` frames whose windows the caller has drawn and staged (ABI 2.11).  Item i owns
 * rows [row_offsets_host[i], row_offsets_host[i+1]) of rows_dev (n_i of them, n_i <= length; a row is BT_N_MELS fp16
 * values) and the same range of row_map_host: the window row each output row t < n_i copies, or -1 for a row a zero
 * mask cleared (NULL: the identity map).  Beat and downbeat frames are CSR tables (beat_offsets_host[n_items + 1] into
 * beat_frames_host, likewise for downbeats), each item's frames sorted, in [0, n_i), duplicates allowed.  Writes
 *   out_spect_dev    [n_items, length, BT_N_MELS] fp16: the mapped row's bits (never converted), 0 for -1 rows and t >= n_i;
 *   truth_beat_dev / truth_downbeat_dev [n_items, length] bytes: 1 where t is one of the item's frames, else 0;
 *   padding_mask_dev [n_items, length] bytes: t < n_i.
 * One launch: every output element is written once (a gather, a binary search per frame), so results are bitwise
 * repeatable.  Works on a weight-less ctx; the tables travel through the ctx's staging ring.
 * BT_ERR_ARG, before anything is enqueued, for n_items < 0, length < 1, a null pointer, offsets that do not start at 0
 * or decrease, n_i > length, a map entry outside [-1, n_i), a frame outside [0, n_i), or an item's frames out of
 * order. */
int bt_train_batch(bt_ctx* ctx, const uint16_t* rows_dev, const int64_t* row_offsets_host, int32_t n_items,
                   int32_t length, const int32_t* row_map_host, const int32_t* beat_frames_host,
                   const int64_t* beat_offsets_host, const int32_t* downbeat_frames_host,
                   const int64_t* downbeat_offsets_host, uint16_t* out_spect_dev, uint8_t* truth_beat_dev,
                   uint8_t* truth_downbeat_dev, uint8_t* padding_mask_dev, void* stream);

/* ---- model gradients: loss.backward() through the reference's BeatThis in eval() mode (train() mode: below) ---------
 * The gradient of the function the inference path computes (BatchNorm on its running statistics, no dropout), in fp32
 * on the CUDA cores (ABI 2.12).  The parameters are the caller's: unfolded fp32 device tensors, one per entry of
 * BeatThis.state_dict(), in the order and shapes of bt_train_param_info, passed on every call as a host array of
 * n_params device pointers.  The entries no kernel reads (the ndim-0 num_batches_tracked counters) may be NULL.  A ctx
 * of any bt_hparams bt_create accepts serves, with BT_DTYPE_F32 and without bt_set_param / bt_finalize; a BT_DTYPE_H16
 * ctx is refused with BT_ERR_ARG.  RoPE angles are computed from each attention's rotary_embed.freqs, so L is bounded
 * only by the activation store (and B * L by 384000 frames). */

/* Entries of the parameter table of a model of shape hp (pure host).  BT_ERR_ARG for a NULL hp. */
int32_t bt_train_param_count(const bt_hparams* hp);
/* Entry i: its state_dict name (NUL-terminated, cap bytes), shape[0 .. *ndim) (the rest 0) and whether it takes a
 * gradient (0 for the BatchNorm running statistics and counters, and rotary_embed.freqs).  Pure host; BT_ERR_ARG for
 * i out of range, a name longer than cap - 1 or a NULL pointer. */
int bt_train_param_info(const bt_hparams* hp, int32_t i, char* name, int32_t cap, int64_t* shape, int32_t* ndim,
                        int32_t* trainable);
/* Bytes of the activation store of one forward pass over [B, L, 128]: what bt_train_backward reads.  BT_ERR_ARG for a
 * NULL ctx or B, L < 1. */
int64_t bt_train_activation_bytes(const bt_ctx* ctx, int32_t B, int32_t L);
/* BeatThis.forward of a dense batch spect_dev [B, L, 128] (fp32; padded frames take part as they do in the reference)
 * -> beat_dev, down_dev [B, L], saving its activations in act_dev (act_bytes >= bt_train_activation_bytes).  The
 * logits equal those of the BT_DTYPE_F32 inference path within its fp32 tolerance. */
int bt_train_forward(bt_ctx* ctx, const float* const* params, int32_t n_params, const float* spect_dev, int32_t B,
                     int32_t L, void* act_dev, int64_t act_bytes, float* beat_dev, float* down_dev, void* stream);
/* From the gradients at the logits (dbeat_dev, ddown_dev [B, L]) and the store of the bt_train_forward call with the
 * same params, B and L: the gradient of every entry into grads[i] (a device buffer of the entry's shape, overwritten,
 * never accumulated).  Entries that take no gradient are never written; a NULL grads[i] skips that gradient.
 * dspect_dev: the gradient at the spectrogram [B, L, 128], or NULL.  Reductions run in a fixed order without atomics:
 * two calls on the same inputs write the same bytes.
 * Both passes: BT_ERR_ARG, before anything is enqueued, for a 16-bit ctx, B or L < 1, n_params other than
 * bt_train_param_count, a NULL pointer, or a store smaller than the batch needs.  Enqueued on `stream` without
 * synchronisation; the ctx's scratch grows on demand. */
int bt_train_backward(bt_ctx* ctx, const float* const* params, int32_t n_params, const void* act_dev, int64_t act_bytes,
                      int32_t B, int32_t L, const float* dbeat_dev, const float* ddown_dev, float* const* grads,
                      float* dspect_dev, void* stream);

/* ---- training mode (ABI 2.14): the reference's BeatThis in train() mode ---------------------------------------------
 * The three calls above are the _ex calls below with mode NULL (eval mode).  With a bt_train_mode, the forward pass is
 * that of the reference's model after .train():
 *  - Dropout at rate dropout_frontend in the three frontend blocks' partial transformers and dropout_transformer in the
 *    main transformer blocks, at four sites per residual branch: an attention's probabilities after the softmax (Attend's
 *    dropout_p) and the output of to_out (to_out.1); a feed-forward's GELU output (net.3) and output (net.5).  Kept values
 *    are scaled by 1 / (1 - p).  Valid rates are 0 <= p < 1; a rate of 0 is no dropout.
 *  - BatchNorm (the stem's bn1d and bn2d, each frontend block's norm) on the batch mean and biased variance over every
 *    position of the batch, zero padding included: B L positions for bn1d, B L F for the others.  The forward pass
 *    updates running_mean and running_var in place, r = 0.9 r + 0.1 batch (the unbiased variance N / (N - 1) for
 *    running_var), through `running`: a host array of device pointers parallel to params, whose running_mean and
 *    running_var entries must be set (the others are not read; it may be params itself).  num_batches_tracked is the
 *    caller's to increment.
 * Dropout masks: element e of dropout site `site` under `seed` is kept iff 32-bit word e mod 4 of
 * Philox4x32-10(counter (lo32(e / 4), hi32(e / 4), site, 0), key (lo32(seed), hi32(seed))) (the rounds of curand's
 * curand_Philox4x32_10) is >= floor(p 2^32), and kept values are multiplied by 1 / (1 - p) rounded to float; p is the
 * float rate as passed (0.9f, not 0.9).
 *  - site: 2 s + k for step s of the model's layer list (stem, then per frontend block attnF, ffF, attnT, ffT and the
 *    block's convolution (without partial transformers only the convolution), frontend.linear, per main block its
 *    attention and feed-forward, the head), k = 0 for an attention's probabilities or a feed-forward's GELU output, 1 for
 *    to_out's or the feed-forward's output.
 *  - e, elementwise sites: row N + col of the step's [M, N] token rows (frontend token row ((b F + f) L + t), main
 *    row b L + t; N = channels, or the FFN hidden width for net.3).
 *  - e, attention probabilities: ((s heads + h) n + i) n + j for query i and key j of sequence s (frequency attention:
 *    s = b L + t over n = F planes; time attention: s = b F + f, or b in the main blocks, over n = L frames).
 * Masks are never stored: the backward pass regenerates them, so it must get the forward's mode (seed and rates), and
 * uses the forward's batch statistics, kept in the store (bt_train_activation_bytes_ex with the same mode sizes it).
 * BT_ERR_ARG before anything is enqueued, beyond the checks above: a rate outside [0, 1) or NaN, a store sized for eval
 * mode, a NULL running table or running_mean / running_var entry (forward), and B L < 2 (a BatchNorm would see one value
 * per channel, which torch refuses in training mode). */
typedef struct bt_train_mode {
  uint64_t seed;
  float dropout_frontend, dropout_transformer;
} bt_train_mode;
/* The activation store's layout (fp32, offsets in floats; each region rounded up to 4 floats, pads never written).
 * Per step of the layer list, in order, with M = B L F token rows of the step's C channels (frontend row
 * ((b F + f) L + t), main row b L + t):
 *   stem       in [B L, 128] (the spectrogram), z [M, C] (the convolution before bn2d)
 *   attention  in [M, C], xn [M, C], inv [M] (1 / ||in||), qkv [M, 3C] (q and k after RoPE), gate logits [M, C/32],
 *              lse [M, C/32] (natural log), o [M, C] (attention output before the gates)
 *   FFN        in [M, C], xn [M, C], inv [M], h [M, mult C] (before GELU), a [M, mult C] (after GELU and dropout)
 *   conv       in [M, C], z [M / 2, 2C] (the convolution before the norm)
 *   linear     in [M, C], xl [B L, C F] (the gathered rows)
 *   head       in [B L, D], xn [B L, D], inv [B L]
 * A step's input is the previous step's output.  Training mode appends, per BatchNorm in layer order (the stem's bn1d
 * then bn2d, each convolution's norm), its batch mean then its biased variance, ch floats each. */
int64_t bt_train_activation_bytes_ex(const bt_ctx* ctx, int32_t B, int32_t L, const bt_train_mode* mode);
int bt_train_forward_ex(bt_ctx* ctx, const float* const* params, int32_t n_params, float* const* running,
                        const float* spect_dev, int32_t B, int32_t L, const bt_train_mode* mode, void* act_dev,
                        int64_t act_bytes, float* beat_dev, float* down_dev, void* stream);
int bt_train_backward_ex(bt_ctx* ctx, const float* const* params, int32_t n_params, const void* act_dev,
                         int64_t act_bytes, int32_t B, int32_t L, const bt_train_mode* mode, const float* dbeat_dev,
                         const float* ddown_dev, float* const* grads, float* dspect_dev, void* stream);

/* ---- optimizer (ABI 2.15): AdamW over a parameter table -------------------------------------------------------------
 * bt_adamw_step updates every entry of `entries_host` (n entries, a host array) in one kernel launch, as
 * torch.optim.AdamW(amsgrad=False, maximize=False) does one step: per element of an entry with t = step,
 *   p <- p (1 - lr wd)                                  (only if wd != 0)
 *   m <- m + (1 - beta1)(g - m)                          (torch's lerp: g - (g - m) beta1 when 1 - beta1 >= 0.5)
 *   v <- beta2 v + (1 - beta2) g g
 *   p <- p - (lr / (1 - beta1^t)) m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
 * op by op in the order of torch's foreach path, each op rounded to fp32 (multiply-adds may be fused).  The scalars
 * 1 - lr wd, 1 - beta1, beta2, 1 - beta2, (1 - beta2^t)^0.5, eps and -lr / (1 - beta1^t) are derived on the host in
 * double, as torch derives them in Python, and rounded to fp32.  `step` is t, the entry's step count after this
 * update (torch increments its state step first).  param, grad, exp_avg and exp_avg_sq are fp32 device arrays of numel
 * elements; grad is read, the other three are updated in place.  An entry whose grad is NULL, or with numel 0, is left
 * untouched (torch skips a parameter without a gradient); when no entry is left, nothing is launched.  Each element
 * is read and written by one thread, without atomics: two calls on the same inputs write the same bytes.
 * BT_ERR_ARG before anything is enqueued: n < 0 (or entries_host NULL with n > 0), a NULL param, exp_avg or exp_avg_sq,
 * numel < 0, a non-finite hyperparameter, lr < 0, eps < 0, a beta outside [0, 1) or step < 1.  The table goes to the
 * device through the ctx's staging ring; the launch is counted and profiled as "adamw".  Any ctx will do (a
 * weight-less one too); enqueued on `stream` without synchronisation. */
typedef struct bt_adamw_entry {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t numel;
  double lr, beta1, beta2, eps, weight_decay;
  int64_t step;
} bt_adamw_entry;
int bt_adamw_step(bt_ctx* ctx, const bt_adamw_entry* entries_host, int32_t n, void* stream);

/* ---- data-parallel training (ABI 2.16): the gradient exchange and the running statistics -----------------------------
 * An optimizer step of k micro-batches on W ranks: each rank runs the micro-batches it owns, packs each one's gradients
 * into a row with bt_grad_pack, the rows travel by all_gather, and every rank sums the k rows in micro-batch order into
 * its gradients with bt_grad_ordered_sum and replays the k micro-batches' BatchNorm statistics with
 * bt_train_running_replay, so every rank holds what one process running the k micro-batches in order would hold.
 *
 * A gradient table: entries_host (n entries, a host array) of fp32 device arrays of numel elements.  Its packed row
 * holds entry i's elements at the sum of the numel of the entries before it, densely in table order (no padding).
 * bt_grad_pack copies every entry's grad into row_dev (the table's total numel floats; nothing else is written).
 * bt_grad_ordered_sum writes every entry's grad as ((r_0 + r_1) + r_2) + ... + r_{k-1} elementwise over the k packed
 * rows rows_host[0 .. k) (a host array of device pointers), in that order: each step one fp32 add rounded to nearest,
 * never fused or reassociated, and r_0 stored as it is (k = 1: a copy).  That is what autograd's AccumulateGrad makes
 * of the same gradients (the first stored, each later one added in place), so the results are bitwise equal to it,
 * signed zeros, infinities, NaNs and subnormals included.  The rows may not overlap the grads.  Each element is read
 * and written by one thread without atomics: two calls on the same inputs write the same bytes.
 * Both: one launch over the whole table (entries with numel 0 are skipped; when no element is left, nothing is
 * launched), counted and profiled as "grad_pack" / "grad_ordered_sum"; the tables go to the device through the ctx's
 * staging ring; any ctx will do (a weight-less one too); enqueued on `stream` without synchronisation.  BT_ERR_ARG
 * before anything is enqueued: n < 0 (or entries_host NULL with n > 0), numel < 0, a NULL grad with numel > 0, a NULL
 * row_dev (pack), k < 1, a NULL rows_host or row (sum), or more than 2^31 - 1 blocks of 2048 elements. */
typedef struct bt_grad_entry {
  float* grad;
  int64_t numel;
} bt_grad_entry;
int bt_grad_pack(bt_ctx* ctx, const bt_grad_entry* entries_host, int32_t n, float* row_dev, void* stream);
int bt_grad_ordered_sum(bt_ctx* ctx, const bt_grad_entry* entries_host, int32_t n, const float* const* rows_host,
                        int32_t k, void* stream);
/* The BatchNorm statistics of k training-mode micro-batches of B x L frames applied to the running statistics in
 * micro-batch order, as k bt_train_forward_ex calls in training mode would have updated them: per micro-batch and per
 * BatchNorm in layer order, r = 0.9 r + 0.1 mean for running_mean and r = 0.9 r + (0.1 N / (N - 1)) var for
 * running_var (N positions), by the same launches the forward pass makes, so the results are bitwise those of the
 * forward passes.  stats_host[j] (a host array of k device pointers) holds micro-batch j's batch statistics: the
 * floats its activation store keeps after the eval-mode layout, (bt_train_activation_bytes_ex with a mode - without) / 4
 * of them, per BatchNorm its batch mean then its biased variance (bt_train_activation_bytes_ex).  running: a host array
 * of device pointers parallel to the parameter table (n_params entries), as bt_train_forward_ex takes it; only its
 * running_mean and running_var entries are read and updated.  num_batches_tracked is the caller's to increment by k.
 * Two launches per BatchNorm and micro-batch, each counted and profiled as "train_reduce" (k = 0: none); any ctx of
 * the model's shape; enqueued on `stream` without synchronisation.  BT_ERR_ARG before anything is enqueued: B or L < 1,
 * B L < 2, n_params other than bt_train_param_count, a NULL running table or running_mean / running_var entry, k < 0,
 * or a NULL stats_host (k > 0) or entry. */
int bt_train_running_replay(bt_ctx* ctx, float* const* running, int32_t n_params, const float* const* stats_host,
                            int32_t k, int32_t B, int32_t L, void* stream);

/* Test hook (fp32 ctx only; BT_ERR_ARG for a 16-bit one): the attention core of one bt_train_forward /
 * bt_train_backward layer alone, on `seqs` time-direction sequences of n positions and `heads` heads of 32.  qkv_dev
 * [seqs * n, 3 * heads * 32] holds q | k | v before RoPE, gates_dev [seqs * n, heads] the gate logits, freqs_dev [16]
 * the rotary frequencies.  Writes y_dev [seqs * n, heads * 32] = softmax(q k^T / sqrt 32) v * sigmoid(gate) (q, k
 * rotated by position * freqs) and, from dy_dev (the gradient at y), the gradients at the pre-RoPE qkv (dqkv_dev) and
 * at the gate logits (dgates_dev).  Seven kernels: RoPE, attention, gate, gate backward, dQ, dK/dV and the inverse
 * RoPE, each counted and profiled under its train_* name.  Synchronises the stream before it returns. */
int bt_debug_attention_backward(bt_ctx* ctx, const float* qkv_dev, const float* gates_dev, const float* freqs_dev,
                                const float* dy_dev, int32_t seqs, int32_t n, int32_t heads, float* y_dev,
                                float* dqkv_dev, float* dgates_dev, void* stream);

/* Test hook (ABI 2.13; fp32 ctx only, BT_ERR_ARG for a 16-bit one): one training kernel alone, through the launcher
 * bt_train_forward / bt_train_backward call, on the caller's fp32 device arrays.  arrays_dev[i] holds counts[i]
 * elements (i < n_arrays; a missing or NULL slot is absent).  The slots of each op, in order (? optional, * written):
 *   GEMM      A, B, C*, bias?, resid?, gelu_out?*, part?*   C[m, n] (ldc) = sum_k A(m, k) B(n, k) (+ bias[n])
 *             (+ resid[m ldr + n]) over M x N x K, A(m, k) = A[m a_rs + k a_cs], B likewise; gelu_out (ldc) = GELU(C).
 *             splits (0: the weight-gradient policy of the training pass) > 1 runs tr_gemm into part [parts, M, N] and
 *             tr_reduce (scale) into C, which then needs ldc = N and no bias, resid or gelu_out.  resid may alias C.
 *   REDUCE    part [splits, M], out* [M]           out = scale sum_z part[z] (masked; + beta out when beta != 0)
 *   COLSUM    A, B?, rs?, part*, out*, shift?      A, B [M, N], rs [M]: part [parts, N] of up to `splits` row ranges
 *             (0: the training pass's policy) of A (* B) (* rs[m]), then out [N] = scale sum of the parts; shift [N]
 *             centres A's columns (A - shift, squared without B)
 *   RMS_FWD   x, gamma, xn*, inv*                  [M, C], gamma [C], inv [M]
 *   RMS_BWD   dxn, x, inv, gamma, dres*            dres [M, C] = (flag ? dres : 0) + dx
 *   BN_GELU_FWD  z, w, b, rm, rv, y*               [M] elements of C channels (index % C), BatchNorm arrays [C]
 *   BN_GELU_BWD  dy, z, w, b, rm, rv, dbn*, dz*
 *   BN_GRADS  s_gz, s_g, w, b, rm, rv, dw?*, db?*  [C]
 *   BN_SCALE  g, w, b, rm, rv, dx*, x?, s_gz?, s_g?  [M] elements of C channels; with x: the batch-statistics input
 *             gradient, rm / rv the batch mean and biased variance over bn_n positions, s_gz / s_g [C] = sum g x, sum g
 *   GELU_BWD  da, h, dh*                           [M]; dh may be da (in place); masked da
 *   IM2COL    in, col*, w?, b?, rm?, rv?           flag: through the 1-d BatchNorm of the input's F S frequencies;
 *             input element (b, f, t, c) of B x (F S) x L x C at b sb + f sf + t st + c sc; col [B F L, C S 3]
 *   COL2IM    dcol, din*                           the adjoint of IM2COL without BatchNorm
 *   CONCAT    src, dst*                            [B F L C] tokens <-> [B L, C F] rows (flag: backward)
 *   ROPE      qkv*, freqs                          qkv [M, 3C] in place, freqs [16]; posmode, L, F; flag: inverse
 *   GATE_FWD  O, g, G*                             O, G [M, C], g [M, C / 32]
 *   GATE_BWD  dG*, O, g, dg*, delta*               dG [M, C] becomes dO; dg, delta [M, C / 32]
 *   HEAD_FWD  o, beat*, down*                      o [M, 2]; flag: sum head
 *   HEAD_BWD  dbeat, ddown, dout*                  dout [M, 2]
 *   ATTN_FWD  qkv, O*, lse*                        over the TrSeqs (seqs, n, heads, seq_in, s_out, s_in, s_pos): token
 *             row r = (s / seq_in) s_out + (s % seq_in) s_in + i s_pos of qkv [*, 3C], O [*, C], lse [*, heads]
 *   ATTN_DQ   qkv, dO, lse, delta, dqkv*           dO [*, C], delta [*, heads]; the q columns of dqkv [*, 3C]
 *   ATTN_DKV  qkv, dO, lse, delta, dqkv*           the k and v columns of dqkv
 * Dropout (p > 0; GEMM unsplit, REDUCE, GELU_BWD, ATTN_*): the mask of `site` under `seed` at element e0 + the op's own
 * element index (GEMM m N + n, REDUCE and GELU_BWD i, attention ((s heads + h) n + i) n + j), as the training pass
 * applies it; GEMM masks gelu_out when given, else the result before resid.  e0 lets a test reach element indices past
 * 2^32 without an array that long.
 * Beyond the hook rules below: a geometry or stride that would take a kernel outside an array's count, a negative
 * stride, a launch grid out of range, or a misaligned pointer where the kernel moves float4 (qkv, O, dO and dqkv of
 * the attention ops) is BT_ERR_ARG with nothing enqueued.  The kernels count and profile under the names the
 * training pass gives them (train_gemm, train_reduce, train_colsum + train_reduce, train_rmsnorm, train_rmsnorm_bwd,
 * train_bn_gelu, train_bn_gelu_bwd, train_bn_grads, train_bn_scale, train_gelu_bwd, train_im2col, train_col2im,
 * train_concat, train_rope, train_gate, train_gate_bwd, train_head, train_attention, train_attention_dq,
 * train_attention_dkv).  Synchronises the stream before it returns. */
enum {
  BT_TRAIN_GEMM, BT_TRAIN_REDUCE, BT_TRAIN_COLSUM, BT_TRAIN_RMS_FWD, BT_TRAIN_RMS_BWD, BT_TRAIN_BN_GELU_FWD,
  BT_TRAIN_BN_GELU_BWD, BT_TRAIN_BN_GRADS, BT_TRAIN_BN_SCALE, BT_TRAIN_GELU_BWD, BT_TRAIN_IM2COL, BT_TRAIN_COL2IM,
  BT_TRAIN_CONCAT, BT_TRAIN_ROPE, BT_TRAIN_GATE_FWD, BT_TRAIN_GATE_BWD, BT_TRAIN_HEAD_FWD, BT_TRAIN_HEAD_BWD,
  BT_TRAIN_ATTN_FWD, BT_TRAIN_ATTN_DQ, BT_TRAIN_ATTN_DKV, BT_TRAIN_OPS
};
typedef struct bt_debug_train_desc {
  int32_t op, splits;  /* BT_TRAIN_*; GEMM / COLSUM: parts (0: policy), REDUCE: parts */
  int64_t M;           /* rows (GEMM, COLSUM, RMS_*, ROPE, GATE_*, HEAD_*), elements (REDUCE, BN_*, GELU_BWD) */
  int32_t N, K, C;     /* GEMM: N x K; COLSUM: N columns; C: channels */
  int32_t flag;        /* RMS_BWD add, IM2COL BatchNorm, CONCAT backward, ROPE inverse, HEAD_* sum head */
  float scale;         /* REDUCE, COLSUM */
  int64_t a_rs, a_cs, b_rs, b_cs, ldc, ldr;  /* GEMM */
  int32_t B, F, L, S, posmode, heads;        /* IM2COL / COL2IM (F: output frequencies), CONCAT, ROPE; attention */
  int64_t sb, sf, st, sc;                    /* IM2COL / COL2IM input strides */
  int32_t seqs, n, seq_in, pad_;             /* attention sequences */
  int64_t s_out, s_in, s_pos;
  /* ABI 2.14; all zero: no dropout, no beta, eval-mode BN_SCALE */
  uint64_t seed;                             /* dropout: the mask's seed */
  float p;                                   /* dropout rate in [0, 1), 0: none */
  uint32_t site;                             /* dropout site */
  int64_t e0;                                /* element index of the op's first element */
  float beta;                                /* REDUCE */
  int32_t pad2_;
  int64_t bn_n;                              /* BN_SCALE with batch statistics: positions per channel */
} bt_debug_train_desc;
int bt_debug_train_kernel(bt_ctx* ctx, const bt_debug_train_desc* desc, float* const* arrays_dev, const int64_t* counts,
                          int32_t n_arrays, void* stream);

/* ---- introspection / tuning ----------------------------------------------------------------- */

/* Upper bound on the chunks processed per wave (1..256, default 128; one wave = one launch of every kernel of the
 * forward pass).  The workspace is budgeted in padded frames: max(chunks x BT_CHUNK, bt_max_chunk) frames (~46 MB per
 * 1500 frames on the 16-bit path), allocated on first use.  Chunks run longest first; a wave is padded to its longest
 * chunk and closes before it would exceed `chunks` chunks or the frame budget, so chunks of up to BT_CHUNK frames
 * form the same waves whatever bt_max_chunk is, and one chunk of bt_max_chunk frames always fits. */
int bt_set_wave_chunks(bt_ctx* ctx, int32_t chunks);

/* Number of kernel launches issued by this ctx since creation (bench.py "gpu_launches"). */
int64_t bt_launch_count(const bt_ctx* ctx);

/* Per-kernel-class device timing for bench.py's roofline line.  While enabled, one CUDA event
 * is recorded on the launch stream after every kernel launch; a launch's duration is the gap
 * to the previous event.  bt_profile_collect synchronises the device and folds the recorded
 * events into per-class totals; bt_profile_get(index) reads class `index` (name, total
 * milliseconds, launches), bt_profile_count the number of classes seen so far. */
int bt_profile_enable(bt_ctx* ctx, int enable);
int bt_profile_collect(bt_ctx* ctx);
int bt_profile_reset(bt_ctx* ctx);
int bt_profile_count(const bt_ctx* ctx);
int bt_profile_get(const bt_ctx* ctx, int index, char* name, int name_cap, double* total_ms,
                   int64_t* launches);

/* Test hook: after the next bt_spect2frames call on a single wave, copy the activation
 * named `tap` (see DESIGN.md "Taps") as fp32 into out_dev (capacity `cap` floats).
 * Returns the element count through *count.  Used only by tests/. */
int bt_debug_request_tap(bt_ctx* ctx, const char* tap, float* out_dev, int64_t cap);
int64_t bt_debug_tap_count(const bt_ctx* ctx);

/* Kernel test hooks: bt_debug_gemm, _attention, _attention_freq, _norm, _fused_qkv, _fused_ff, _stem, _zero_tail,
 * _head (below) and bt_debug_dbn_viterbi (with the DBN entry points) each run the kernel the forward pass or
 * post-processor runs, alone, on the ctx's device and the given stream.  Common to all of them:
 *  - Arguments are checked before anything is enqueued; a bad one returns BT_ERR_ARG and launches nothing.
 *  - Arrays are fp32 on the device unless stated.  The 16-bit context rounds the kernel's 16-bit operands to its
 *    activation type, and runs each 16-bit output through that type: the whole buffer given, so that values the
 *    kernel does not store survive.
 *  - A tensor-core plan the geometry does not fit is refused with the plan's reason: BT_ERR_CUDA, except BT_ERR_ARG
 *    for bt_debug_attention_freq.
 *  - Only the kernel under test counts in bt_launch_count (+1 per call; +2 for bt_debug_dbn_viterbi) and in the
 *    profile, under the name debug_gemm, debug_attention, debug_attention_freq, debug_norm, debug_fused_qkv,
 *    debug_fused_ff, stem, zero_tail, head, or dbn_viterbi and dbn_backtrace.  Under BT_SYNC_DEBUG=1 it is checked as
 *    every launch of the forward pass is.  Rounding and operand packing are neither counted nor profiled.
 *  - Each synchronises the stream before it returns. */

/* Shape and epilogue of one bt_debug_gemm call: the GEMM the forward pass runs for a linear layer, a k(2,3)
 * convolution or frontend.linear (csrc/bt_kernels.h GemmShape / EpiParams).  Output row m = p_out * L + t of N
 * columns; slab s reads plane p_out * plane_mul + plane_add[s] at time t + t_shift[s] (zeros outside [0, L)),
 * columns [0, Kslab) of a row-major [planes_in * L, lda] A.  W is [N, nslab * Kslab].
 * kind 0: (+ bias) (-> GELU) (+ resid) into out_f32 and/or out_act, both [M, N];  kind 1: q|k|v columns of C each,
 * RoPE on q and k at position t (posmode 0) or p_out % F (posmode 1), q scaled by qscale, into out_act [M, N];
 * kind 2: sigmoid(acc + bias) of columns n < heads into out_f32 [M, heads].
 * resid_epilogue: the tile-width policy of a GEMM whose epilogue adds the fp32 residual. */
typedef struct bt_debug_gemm_desc {
  int32_t planes_out, planes_in, L, N, Kslab, nslab, plane_mul, lda;
  int32_t plane_add[6];
  int32_t t_shift[6];
  int32_t resid_epilogue;
  int32_t kind, gelu, C, heads, posmode, F;
  float qscale;
} bt_debug_gemm_desc;

/* One GEMM of shape and epilogue `desc` through the ctx's GEMM kernel (16-bit: gemm_tc_kernel, fp32:
 * gemm_simt_kernel).  bias, resid, out_f32, out_act and the rope tables may be NULL; resid may alias out_f32.  The
 * 16-bit operands are A and W; out_act (out_act_count elements) is the 16-bit output.  tile_out[2] (optional) receives
 * the (BN, BK) tile of the 16-bit plan, (0, 0) in the fp32 context. */
int bt_debug_gemm(bt_ctx* ctx, const bt_debug_gemm_desc* desc, const float* a_dev, const float* w_dev,
                  const float* bias_dev, const float* resid_dev, float* out_f32_dev, float* out_act_dev,
                  int64_t out_act_count, const float* rope_cos_dev, const float* rope_sin_dev, int32_t* tile_out,
                  void* stream);

/* gates * softmax(Q K^T / sqrt(32)) V for `seqs` sequences of length L and `heads` heads of dim 32 through the ctx's
 * time-direction attention kernel.  q/k/v_dev are [seqs, L, heads*32], gates_dev [seqs * L, heads].  o_dev, the 16-bit
 * output, holds o_count >= seqs * L * heads * 32 elements, the first seqs * L * heads * 32 of them the output.
 * key_lens_host (optional): sequence s belongs to chunk s / seqs_per_chunk and attends to the first
 * key_lens_host[chunk] keys only (1 <= len <= L), as in a wave of chunks of different lengths. */
int bt_debug_attention(bt_ctx* ctx, const float* q_dev, const float* k_dev, const float* v_dev,
                       const float* gates_dev, float* o_dev, int64_t o_count, int32_t seqs, int32_t L, int32_t heads,
                       const int32_t* key_lens_host, int32_t seqs_per_chunk, void* stream);

/* The frequency-direction attention of B chunks of F planes of L frames: token m = (b * F + f) * L + t attends over
 * the F tokens of its (b, t), gates * softmax(q k^T / sqrt(32)) v per head.  q/k/v/o_dev are [B * F * L, heads * 32],
 * gates_dev [B * F * L, heads]; F in {8, 16, 32}.  o_dev holds o_count >= B * F * L * heads * 32 elements, as for
 * bt_debug_attention.  The 16-bit context runs the tensor-core kernel of the frontend blocks, whose plan refuses any
 * pair other than (F, heads) = (32, 1), (16, 2), (8, 4). */
int bt_debug_attention_freq(bt_ctx* ctx, const float* q_dev, const float* k_dev, const float* v_dev,
                            const float* gates_dev, float* o_dev, int64_t o_count, int32_t B, int32_t F, int32_t L,
                            int32_t heads, void* stream);

/* The frontend's row kernels.  x, wg, b1 and b2 must be 16-byte aligned, and so must xn of bt_debug_norm in the fp32
 * context (the kernel stores it directly).  The 16-bit operands are wqkv, w1, w2, o and wout; the 16-bit outputs are
 * xn, qkv and xb. */

/* RMSNorm xn = x / max(||x||, 1e-12) of M rows of C in {32, 64, 128, 256, 512, 1024} through norm_kernel, in the
 * ctx's activation type.  With gates_dev (then wg_dev [heads, C], bg_dev [heads], 1 <= heads <= C / 32) also
 * gates [M, heads] = sigmoid(xn . wg[h] + bg[h]); without, heads is 0. */
int bt_debug_norm(bt_ctx* ctx, const float* x_dev, float* xn_dev, int64_t M, int32_t C, const float* wg_dev,
                  const float* bg_dev, float* gates_dev, int32_t heads, void* stream);

/* The fused RMSNorm + gates + QKV + RoPE kernel of the frontend attentions (16-bit context only, C in {32, 64}):
 * x [M, C] -> qkv [M, 3C] = rmsnorm(x) wqkv^T with RoPE on the q and k columns at position m % L (posmode 0) or
 * (m / L) % F (posmode 1), q also scaled by qscale; gates [M, C / 32] as bt_debug_norm gives them.  wqkv [3C, C];
 * wg [C / 32, C] or the padded [32, C]; bg likewise; rope tables [BT_CHUNK, 16]. */
int bt_debug_fused_qkv(bt_ctx* ctx, const float* x_dev, const float* wqkv_dev, const float* wg_dev, const float* bg_dev,
                       const float* rope_cos_dev, const float* rope_sin_dev, float* qkv_dev, float* gates_dev, int64_t M,
                       int32_t C, int32_t L, int32_t F, int32_t posmode, float qscale, void* stream);

/* The fused FFN of the frontend blocks (16-bit context only, C in {32, 64}), in place on x [M, C]:
 * x' = x (+ o wout^T when o_dev and wout_dev are both set: the attention out-projection in front), then
 * x = x' + w2 gelu(w1 rmsnorm(x') + b1) + b2.  w1 [4C, C], b1 [4C], w2 [C, 4C], b2 [C], o [M, C], wout [C, C].
 * xb_dev (optional, [M, C]) receives the 16-bit copy of the result. */
int bt_debug_fused_ff(bt_ctx* ctx, float* x_dev, const float* w1_dev, const float* b1_dev, const float* w2_dev,
                      const float* b2_dev, const float* o_dev, const float* wout_dev, float* xb_dev, int64_t M, int32_t C,
                      void* stream);

/* One entry of the chunk table the forward pass hands its stem, zero_tail and head kernels (one chunk of a wave):
 * the clip is spectrogram frames [frame_base, frame_base + T) and output frames [out_base, out_base + T); the chunk
 * starts at clip frame `start` (may be negative or run past T: those frames are zero before BN1d) and has `len`
 * frames (rows [len, L) of its planes are padding); it owns chunk-local frames [write_lo, write_hi). */
typedef struct bt_debug_chunk {
  int64_t frame_base;
  int32_t T, start;
  int64_t out_base;
  int32_t write_lo, write_hi, len;
} bt_debug_chunk;

/* The kernels that read the chunk table.  Parameters are device arrays, so a weight-less ctx will do; chunks_host is
 * uploaded through the ctx's staging ring, as the forward pass uploads its table.  A table or geometry that would
 * take the kernel outside the buffers described is BT_ERR_ARG.
 *
 * bt_debug_stem: stem_kernel over n_chunks chunks (1..65535) of padded length L (1..384000) gathered from spect_dev
 * [spect_frames, 128]; bn1_scale / bn1_shift [128], w [32, 4, 3] (BN2d folded), bias [32]; out_dev [n_chunks, 32, L,
 * 32] holds out_count >= n_chunks * 32 * L * 32 floats.  spect_dev and out_dev must be 16-byte aligned; every chunk
 * needs T >= 1, 1 <= len <= L and its clip inside [0, spect_frames). */
int bt_debug_stem(bt_ctx* ctx, const float* spect_dev, int64_t spect_frames, const bt_debug_chunk* chunks_host,
                  int32_t n_chunks, int32_t L, const float* bn1_scale_dev, const float* bn1_shift_dev, const float* w_dev,
                  const float* bias_dev, float* out_dev, int64_t out_count, void* stream);

/* bt_debug_zero_tail: zero_tail_kernel: rows [len, L) of every plane of buf_dev [n_chunks, F, L, C] (elements of
 * elem_bytes 2 or 4, buf_bytes bytes, 16-byte aligned) become 0.  Needs C * elem_bytes a multiple of 16, n_chunks,
 * F >= 1 with n_chunks * F < 2^31, 1 <= len <= L <= 384000 for every chunk (only len is read). */
int bt_debug_zero_tail(bt_ctx* ctx, void* buf_dev, int32_t elem_bytes, const bt_debug_chunk* chunks_host,
                       int32_t n_chunks, int32_t F, int32_t L, int32_t C, int64_t buf_bytes, void* stream);

/* bt_debug_head: head_kernel on x_dev [n_chunks, L, D] (D a multiple of 64 in [64, 1024], n_chunks * L < 2^31):
 * o_j = (x . w_j) / max(||x||, 1e-12) + b_j with w [2, D], b [2]; beat = o0 + o1 (sum_head != 0) or o0, down = o1,
 * stored at out_base + start + t for every owned frame t of a chunk.  Each owned range must lie in [0, L] and every
 * owned frame's index in [0, out_count), the length of beat_dev and down_dev. */
int bt_debug_head(bt_ctx* ctx, const float* x_dev, int32_t D, const float* w_dev, const float* b_dev,
                  const bt_debug_chunk* chunks_host, int32_t n_chunks, int32_t L, int32_t sum_head, float* beat_dev,
                  float* down_dev, int64_t out_count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BEATTHIS_H_ */
