/* parakeet_b200.h -- the drop-in boundary: a flat C-ABI over the H100-native hot path
 *
 *     16 kHz PCM -> log-mel -> FastConformer encoder -> CTC / TDT greedy decode
 *
 * The reference (Frikallo/parakeet.cpp @ 40bbd7e) has no C API ("C API" is an
 * unchecked roadmap item, README.md:518); its boundary for this path is C++:
 * parakeet::Transcriber (include/parakeet/transcribe.hpp:55-190) calling
 * preprocess_audio (src/audio.cpp:100), FastConformerEncoder::forward
 * (src/encoder.cpp:253), CTCDecoder::forward + ctc_greedy_decode (src/ctc.cpp:12,40)
 * and tdt_greedy_decode (src/tdt.cpp:36).  Each entry point below names the
 * reference function(s) it replaces.  include/parakeet/transcribe.hpp in this
 * repository is the header-only C++ shim with the reference's class signatures
 * on top of this ABI; INTEGRATION.md shows the binding a maintainer would add.
 *
 * Conventions: plain pointers and sizes only; every call returns pk_status and
 * never throws; the opaque engine owns all device memory, its CUDA stream and
 * graphs; the caller owns host buffers.  One engine per device; calls on one
 * engine are serialised on its stream (thread-compatible, not thread-safe).
 * There is no CPU fallback: without a CUDA device pk_engine_create fails.
 */
#ifndef PARAKEET_B200_H
#define PARAKEET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    PK_OK = 0,
    PK_ERR_INVALID = 1,   /* bad argument / shape */
    PK_ERR_IO = 2,        /* cannot open / parse weights */
    PK_ERR_CUDA = 3,      /* CUDA runtime / driver error */
    PK_ERR_MISSING = 4,   /* tensor missing from the state dict */
    PK_ERR_CAPACITY = 5,  /* batch exceeds the engine's configured capacity */
    PK_ERR_NCCL = 6
} pk_status;

/* PK_DECODER_TDT runs only on a TDT model, PK_DECODER_RNNT only on an RNN-T model (n_durations = 0);
 * PK_DECODER_CTC needs a CTC head (has_ctc).  A mismatch is PK_ERR_INVALID.  PK_DECODER_CTC_BEAM: CTC prefix beam
 * search with optional word n-gram fusion (pk_set_ctc_beam below; DESIGN.md section 14).  PK_DECODER_CTC_ALIGN: CTC forced
 * alignment of known token sequences (pk_set_align_targets below; DESIGN.md section 15). */
typedef enum { PK_DECODER_CTC = 0, PK_DECODER_TDT = 1, PK_DECODER_RNNT = 2, PK_DECODER_CTC_BEAM = 3, PK_DECODER_CTC_ALIGN = 4 } pk_decoder;

/* GEMM arithmetic.  PK_MATH_BF16X3 (default): wgmma MMAs on bf16
 * hi/lo operand splits, 3 MMAs per product (hi*hi + hi*lo + lo*hi), fp32
 * accumulation in registers: ~1e-5 relative, the parity mode.  PK_MATH_BF16X1: hi*hi only
 * (fast, ~4e-3).  PK_MATH_FP32: CUDA-core fp32 GEMM (bring-up / checker). */
typedef enum { PK_MATH_BF16X3 = 0, PK_MATH_BF16X1 = 1, PK_MATH_FP32 = 2 } pk_math;

/* Mirrors EncoderConfig / PredictionConfig / JointConfig / TDTCTCConfig / RNNTConfig
 * (include/parakeet/config.hpp:9-75).  pk_config_110m / pk_config_tdt_600m / pk_config_rnnt_600m
 * fill it with make_110m_config (:77-95) / make_tdt_600m_config (:98-116) / make_rnnt_600m_config
 * (:118-135). */
typedef struct {
    int32_t mel_bins;          /* 80 | 128 */
    int32_t sub_channels;      /* 256 */
    int32_t d_model;           /* 512 | 1024 */
    int32_t n_layers;          /* 17 | 24 */
    int32_t n_heads;           /* 8 */
    int32_t ff;                /* 2048 | 4096 */
    int32_t conv_kernel;       /* 9 */
    int32_t vocab;             /* 1025 | 8193, blank = vocab-1 */
    int32_t pred_hidden;       /* 640 */
    int32_t lstm_layers;       /* 1 | 2 */
    int32_t joint_hidden;      /* 640 */
    int32_t n_durations;       /* 5; 0 = RNN-T joint (ParakeetRNNT: joint_.out_proj_ over the vocab, no
                                  duration head; needs joint_prefix_tdt = 0, has_ctc = 0) */
    int32_t durations[8];      /* {0,1,2,3,4} */
    int32_t has_ctc;           /* ParakeetTDTCTC: 1, ParakeetTDT: 0 */
    int32_t joint_prefix_tdt;  /* 1: keys "tdt_joint_." (tdt_ctc.cpp:5-9); 0: "joint_." (tdt.cpp:28-32) */
    int32_t max_symbols;       /* max_symbols_per_step, 10 (tdt.hpp, rnnt.hpp); RNN-T: 1..64, the decode
                                  advances a frame after this many emissions on it */
    /* engine capacity (not model shape) */
    int32_t max_batch;         /* utterances per call */
    int32_t max_samples;       /* per utterance; with full attention the position tables and the attention grow with
                                  the square of it, with a band (below) linearly */
    int32_t math;              /* pk_math */
    /* Limited-context attention (NeMo's rel_pos_local_attn, DESIGN.md section 16) for long offline utterances: encoder
     * frame i attends to frame j only when -local_att_right <= i - j <= local_att_left, with the same relative-position
     * bias and the softmax over the keys that remain.  Both >= 0 (PK_ERR_INVALID otherwise); 0, 0 = full attention, the
     * default of every preset.  A band engine keeps position tables of 2 min(max(left, right), T'max - 1) + 1 rows (T'max =
     * the encoder frames of max_samples: a band wider than an utterance is full attention, at its cost).  It supports
     * max_samples <= PK_LOCAL_ATT_MAX_SAMPLES (3 h of 16 kHz audio; pk_engine_create returns PK_ERR_CAPACITY past it) and
     * batches of at most the encoder frames of that much audio in all (PK_ERR_CAPACITY from the call otherwise).
     * It runs every offline entry point; pk_stream_open on it is PK_ERR_INVALID, and a Sortformer engine takes no band. */
    int32_t local_att_left;
    int32_t local_att_right;
} pk_config;

#define PK_LOCAL_ATT_MAX_SAMPLES 172800000

typedef struct pk_engine pk_engine;

void pk_config_110m(pk_config *cfg);      /* config.hpp:77-95  */
void pk_config_tdt_600m(pk_config *cfg);  /* config.hpp:98-116 */
void pk_config_rnnt_600m(pk_config *cfg); /* config.hpp:118-135 (mel 80, vocab 1025, n_durations = 0) */
/* make_nemotron_600m_config (nemotron.hpp:33-54): the multilingual STREAMING model, opened with pk_stream_open.
 * d 1024, 24 layers, 8 heads, ff 4096, 80 mels (the preset leaves mel_bins at its default), vocab 8193, 2 LSTM
 * layers, TDT durations {0..4}, keys "encoder_." / "prediction_." / "joint_." (has_ctc 0, joint_prefix_tdt 0).
 * Capacity suits streaming: max_batch 64 streams, max_samples 102400 (81 encoder frames >= left context 70 + the
 * frames of one chunk).  The latency mode (att_context_right) is an argument of pk_stream_open, not of pk_config. */
void pk_config_nemotron_600m(pk_config *cfg);

/* Replaces Transcriber::Transcriber + to_gpu (transcribe.hpp:59-71):
 * safetensors::load (axiom io_safetensors.cpp:123-160) + load_state_dict(strict=false)
 * (axiom module.cpp:24-38) + Module::to(GPU).  Missing tensors for modules on the
 * path are an error (PK_ERR_MISSING); extra tensors are ignored. */
pk_status pk_engine_create(const pk_config *cfg, const char *safetensors_path, int device,
                           pk_engine **out);
void pk_engine_destroy(pk_engine *e);
/* Last error text of this engine (or of the failed create when e == NULL). */
const char *pk_last_error(const pk_engine *e);

/* Shape helpers (operations.cpp:3191-3196 output-length formula). */
int32_t pk_mel_frames(int64_t n_samples);           /* 1 + n/160                       */
int32_t pk_encoder_frames(int32_t n_mel_frames);    /* three stride-2 k3 p1 stages     */

/* Replaces preprocess_audio (src/audio.cpp:100-158) for a batch of utterances.
 * pcm: host fp32, utterance i = pcm[offsets[i] .. offsets[i+1]).
 * feats_out: host fp32, packed (sum_i frames_i, mel_bins); n_frames_out[n_utt]. */
pk_status pk_mel(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt,
                 float *feats_out, int32_t *n_frames_out);

/* Replaces FastConformerEncoder::forward (src/encoder.cpp:253-271).
 * feats: host fp32 packed (sum frames_i, mel_bins); enc_out: host fp32 packed
 * (sum T'_i, d_model); enc_lens_out[n_utt] = T'_i.
 * Optional debug taps (may be NULL): sub_out packed (sum T'_i, d_model) after
 * ConvSubsampling; layers_out (n_layers, sum T'_i, d_model) after each block. */
pk_status pk_encode(pk_engine *e, const float *feats, const int32_t *n_frames, int32_t n_utt,
                    float *enc_out, int32_t *enc_lens_out, float *sub_out, float *layers_out);

/* Token streams of a batch.  Row i holds len[i] entries of ids/start/end/conf
 * at stride `cap`.  start/end are encoder frames (0.08 s, timestamp.hpp:31-35),
 * conf = exp(log-prob) as in ctc.cpp:110 / tdt.cpp:165.  */
typedef struct {
    int32_t cap;        /* in: row capacity (>= max tokens per utterance)   */
    int32_t *ids;       /* [n_utt * cap] */
    int32_t *start;     /* [n_utt * cap] or NULL */
    int32_t *end;       /* [n_utt * cap] or NULL */
    float *conf;        /* [n_utt * cap] or NULL */
    int32_t *len;       /* [n_utt] */
} pk_tokens;

/* Decode-only entry points on a host encoder output (packed (sum T_i, d_model)):
 * CTCDecoder::forward + ctc_greedy_decode(_with_timestamps) (src/ctc.cpp:12-127),
 * tdt_greedy_decode(_with_timestamps) (src/tdt.cpp:36-201) and
 * rnnt_greedy_decode(_with_timestamps) (src/rnnt.cpp:56-177). */
pk_status pk_decode(pk_engine *e, const float *enc, const int32_t *enc_lens, int32_t n_utt,
                    pk_decoder dec, pk_tokens *out);

/* CTC head log-probs (CTCDecoder::forward, src/ctc.cpp:12-25) for inspection:
 * enc packed (sum T_i, d_model) -> logprobs packed (sum T_i, vocab). */
pk_status pk_ctc_logprobs(pk_engine *e, const float *enc, int32_t total_frames, float *logprobs_out);

/* The whole path, replacing the body of Transcriber::transcribe
 * (transcribe.hpp:99-179) for a batch: host PCM in, token streams out.
 * H2D of the PCM and D2H of the tokens happen inside the call. */
pk_status pk_transcribe_batch(pk_engine *e, const float *pcm, const int64_t *offsets,
                              int32_t n_utt, pk_decoder dec, pk_tokens *out);

/* Device-resident variant for throughput measurement: stage PCM once ...
 * Buffer lifetime: when `pcm` is page-locked, the engine DMAs straight from it and pk_stage_pcm returns while
 * the copy may still be in flight -- the buffer must stay valid AND unmodified until the next pk_fetch_tokens /
 * pk_sync on this engine returns (the same holds for a buffer handed to pk_prefetch_pcm).  Pageable buffers are
 * copied before the call returns. */
pk_status pk_stage_pcm(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt);
/* Serving pipeline (no reference counterpart: the reference is synchronous and batch-1).  Starts the
 * host-to-device copy of the NEXT batch into the engine's second PCM buffer on a copy stream and
 * returns at once, so the copy runs under the current batch's kernels:
 *     pk_prefetch_pcm(b0); loop { pk_stage_pcm(b_i); pk_run_staged(); pk_prefetch_pcm(b_{i+1}); pk_fetch_tokens(); }
 * pk_stage_pcm / pk_transcribe_batch with the same (pcm, offsets, n_utt) then adopt the prefetched buffer
 * instead of copying.  The samples are read when this call is made; the buffer must be page-locked and
 * packed back to back (PK_ERR_INVALID otherwise) and must stay valid until the adopting call returns. */
pk_status pk_prefetch_pcm(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt);
/* ... then run the path on the staged batch; tokens stay on the device until
 * pk_fetch_tokens.  Asynchronous on the engine stream. */
pk_status pk_run_staged(pk_engine *e, pk_decoder dec);
pk_status pk_fetch_tokens(pk_engine *e, pk_tokens *out);
pk_status pk_sync(pk_engine *e);

/* Device token buffer of the last run for the single cross-GPU exchange:
 * int32 rows [n_utt][1 + cap] = (len, ids...).  The caller (torch.distributed /
 * NCCL) all-gathers this buffer; see INTEGRATION.md. */
pk_status pk_token_buffer(pk_engine *e, void **dev_ptr, int32_t *rows, int32_t *row_ints);

/* ---- Jobs and the single cross-GPU exchange (SURVEY.md section 8e; BASELINE configs[4]: 8192 clips over 8 GPUs).
 * The reference is single-device and batch-1 (transcribe.hpp:170-171); this is what a sharded host adds around
 * Transcriber::transcribe.  A rank owns a contiguous block of clips and runs it in micro-batches of at most
 * pk_config.max_batch; after every pk_run_staged, pk_job_append copies that micro-batch's token rows
 * (int32 [1 + cap] = len, ids...) into a device-resident job buffer of rows_local rows (asynchronous, engine
 * stream).  pk_allgather_tokens then issues ONE ncclAllGather of the job buffer on the engine stream (no host
 * synchronisation; rows a rank did not fill have len = 0), and pk_job_fetch copies local (gathered = 0) or
 * gathered (gathered = 1: rank-major [world][rows_local]) rows to the host.
 *
 * NCCL is resolved at run time (dlopen "libnccl.so.2": the copy the process already uses); without it these
 * calls return PK_ERR_NCCL.  Either pass the host's own ncclComm_t to pk_allgather_tokens, or let the engine
 * own one: rank 0 calls pk_nccl_unique_id, the host broadcasts the 128 bytes, every rank calls pk_comm_init_rank. */
#define PK_NCCL_UNIQUE_ID_BYTES 128
pk_status pk_job_begin(pk_engine *e, int64_t rows_local, int32_t world);
pk_status pk_job_append(pk_engine *e);
pk_status pk_nccl_unique_id(void *id128);
pk_status pk_comm_init_rank(pk_engine *e, const void *id128, int32_t rank, int32_t world);
pk_status pk_allgather_tokens(pk_engine *e, void *nccl_comm /* ncclComm_t, or NULL: the engine's communicator */);
pk_status pk_job_fetch(pk_engine *e, int32_t gathered, int32_t *rows_out, int64_t n_rows, int32_t *row_ints);
/* Device-resident job input for throughput measurement: copy the PCM of a whole job (any number of utterances,
 * host buffer, packed or not) to the device once, then make micro-batch [first, first + n_utt) the staged batch
 * without a copy (pk_run_staged / pk_job_append follow as usual). */
pk_status pk_job_stage_pcm(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt);
pk_status pk_job_select(pk_engine *e, int32_t first, int32_t n_utt);

/* ---- Streaming (SURVEY.md section 8f row 2; BASELINE configs[3]: eou-120m, 160 ms chunks), replacing
 * StreamingTranscriber::transcribe_chunk / reset (src/eou.cpp:111-149): StreamingAudioPreprocessor::process_chunk
 * (src/audio.cpp:195-259), StreamingFastConformerEncoder::forward_chunk (src/streaming_encoder.cpp:425-472) and
 * rnnt_streaming_decode_chunk (src/eou.cpp:17-98).  The reference advances ONE stream per call; here n_streams streams
 * advance in lock step and share every weight read.  The engine must have been created with max_batch >= n_streams and
 * max_samples large enough that its encoder-frame capacity is >= att_context_left + frames per chunk (6.4 s is plenty
 * for the eou-120m preset: left context 70).  Per-stream state (sample overlap, leftover mel frames, K/V and conv caches,
 * LSTM state, last token, frame offset) lives on the device.
 *   pk_stream_open : allocate the state of n_streams streams (att_context_left / right of StreamingEncoderConfig,
 *                    streaming_encoder.hpp:18-24; the right context / mask is inert in the reference's CPU path and is
 *                    not applied, see DESIGN.md).
 *   pk_stream_step : stream s receives pcm[offsets[s] .. offsets[s+1]) (host fp32; an empty chunk is allowed); `out` rows
 *                    (n = n_streams, may be NULL) receive the tokens emitted BY THIS STEP, start/end = absolute encoder
 *                    frames (the end frame is not clamped to the chunk, eou.cpp:81-84).  Optional taps (may be NULL):
 *                    mel_out packed (sum nf_s, mel_bins) new log-mel frames, n_mel[s] = nf_s; enc_out packed
 *                    (sum C_s, d_model) encoder rows of this step, n_enc[s] = C_s.  A first chunk of 400..511 samples
 *                    returns PK_ERR_INVALID where the reference's STFT throws (fft.cpp:1516-1521).
 *   pk_stream_reset: StreamingTranscriber::reset for one stream (-1: all). */
pk_status pk_stream_open(pk_engine *e, int32_t n_streams, int32_t max_chunk_samples, int32_t att_context_left,
                         int32_t att_context_right);
pk_status pk_stream_reset(pk_engine *e, int32_t stream);
pk_status pk_stream_step(pk_engine *e, const float *pcm, const int64_t *offsets, pk_tokens *out, float *mel_out,
                         int32_t *n_mel, float *enc_out, int32_t *n_enc);
int32_t pk_stream_count(const pk_engine *e);

/* Host-only probe of the checkpoint reader (safetensors::load, axiom io_safetensors.cpp:16-160: F32 / F16 / BF16 / F64
 * tensors, converted to fp32): opens the file (PK_ERR_IO + pk_last_error(NULL) on a malformed header), and if `name` is
 * given converts that tensor into out[0 .. cap) and reports its element count.  Needs no device. */
pk_status pk_safetensors_probe(const char *path, const char *name, float *out, int64_t cap, int64_t *numel);

/* Number of utterances of the last pk_fetch_tokens whose TDT hypothesis was cut at the engine's token capacity
 * (2 T'max + 8 per utterance; only reachable on inputs that livelock the reference's tdt_greedy_decode, which
 * never forces an advance after max_symbols_per_step, src/tdt.cpp:66-104).  Always 0 for an RNN-T model: its
 * capacity is max_symbols T'max + 8, the most an RNN-T decode can emit. */
int32_t pk_truncated_count(const pk_engine *e);

/* CUDA stream of the engine (cudaStream_t as void*), for event timing. */
void *pk_stream(pk_engine *e);
/* Number of kernel launches issued by the engine since creation (the
 * `gpu_launches` claim in bench.py). */
int64_t pk_launch_count(const pk_engine *e);

/* Measurement aids (bench.py): per-kernel-class device time measured with CUDA events on
 * the engine stream between begin/end (classes in pk_profile_names() order, comma
 * separated; ms / launch counts / algorithmic GEMM flops summed per class), and an L2
 * flush (writes a 256 MiB scratch buffer on the engine stream). */
pk_status pk_profile_begin(pk_engine *e);
pk_status pk_profile_end(pk_engine *e, double *ms, int64_t *counts, double *flops, int32_t n);
const char *pk_profile_names(void);
pk_status pk_flush_l2(pk_engine *e);

/* Debug aid: cycles CTA 0 of the last TDT decode spent in {P1, B1, P2, B2, P3, B3, P4}; out8[7] =
 * number of lock-step decode steps. */
pk_status pk_debug_tdt_phases(pk_engine *e, int64_t *out8);
/* Debug aid: cycles CTA 0 spent in the sections of the decode kernel's passes since the previous call:
 * {x staging, products, partial store + cluster barrier, DSMEM gather + finalise, number of passes, 0, 0, 0}. */
pk_status pk_debug_tdt_passes(pk_engine *e, int64_t *out8);

/* GPU self-check of the wgmma GEMM kernel against the fp32 CUDA-core GEMM on seeded
 * random data (epi_kind: EpiKind of csrc/pk_common.cuh; math: PK_MATH_BF16X3 | PK_MATH_BF16X1). */
pk_status pk_selftest_gemm(int device, int M, int N, int K, int epi_kind, int math, uint32_t seed,
                           float *max_err, float *max_ref);

/* Kernel test hooks (csrc/kernel_hooks.cu): each runs ONE launcher of the hot path exactly as the engine calls it, on host fp32
 * arrays, on a private stream, synchronously, and returns every output buffer whole (bf16 planes widened to float).  Every
 * device output sits between 64 KiB guard bands; output and guards start as 0xFF bytes (NaN in fp32 and bf16), so elements
 * the kernel must not write come back NaN, and *guard_bad = the number of guard bytes that changed.
 *
 * GEMM: path 0 = fp32 CUDA-core kernel (math PK_MATH_FP32), 1 = wgmma (cluster 2 | 4: the multicast form, where
 * supported), 2 = the few-row kernel (M <= 128, launched twice).  A [M][K], W [N][K], bias [N] (or NULL).  Output [M][ldo]:
 * out_f32 for the fp32 kinds and GLU (N/2 columns), out_hi (| out_lo, NULL = no lo plane) for the act kinds and the k | v
 * part of EPI_QKV_ACT (whose q columns go to out_f32 [M][qcols]); the act kinds write out_f32 on path 0.  EPI_RESID_F32
 * reads resid [M][ldo]; in_place = 1 starts out_f32 as resid and passes it as both, as the encoder runs it. */
pk_status pk_kernel_gemm(int device, int path, int math, int cluster, int M, int N, int K, int epi_kind, int qcols, int ldo, float alpha,
                         int in_place, const float *A, const float *W, const float *bias, const float *resid, float *out_f32,
                         float *out_hi, float *out_lo, int64_t *guard_bad);
/* Relative-position attention: kernel 0 = fp32 CUDA-core, 1 = mma.sync (default).  qkv [rows_total][3 d] (kernel 1 gets q
 * in fp32 and k | v as bf16 planes, as the EPI_QKV_ACT epilogue lays them out), pp [2 tmax - 1][d], utterance
 * b = rows [row_off[b], row_off[b+1]) (rows outside every utterance may exist).  ctx [rows_total][d]: ctx_f32 with
 * PK_MATH_FP32 (kernel 0 only), else ctx_hi and, with PK_MATH_BF16X3, ctx_lo. */
pk_status pk_kernel_attention(int device, int kernel, int math, int n_utt, const int32_t *row_off, int rows_total, int d_model, int n_heads,
                              int tmax, const float *qkv, const float *pp, const float *pos_u, const float *pos_v, float *ctx_f32,
                              float *ctx_hi, float *ctx_lo, int64_t *guard_bad);
/* The same with a band (left, right), both >= 0 and not both 0, as a band engine runs it: pp [2 tmax - 1][d] holds the
 * relative positions -(tmax-1)..tmax-1, tmax >= max(left, right) + 1 (the engine's table: tmax = max(left, right) + 1 when
 * that is below its T'max); utterances may be longer than tmax.  The table is uploaded between two NaN rows, which the kernel must not read. */
pk_status pk_kernel_attention_local(int device, int kernel, int math, int n_utt, const int32_t *row_off, int rows_total, int d_model,
                                    int n_heads, int tmax, int left, int right, const float *qkv, const float *pp, const float *pos_u,
                                    const float *pos_v, float *ctx_f32, float *ctx_hi, float *ctx_lo, int64_t *guard_bad);
/* LayerNorm of x [M][d] (w2 == NULL: one; else LN2(LN1(x)), the chained form).  want_f32: y1 = LN1(x) written in place over
 * x -> y1_f32.  planes (the operand of the last LayerNorm): 0 none, 1 hi, 2 hi + lo, 3 fp32 -> act_f32. */
pk_status pk_kernel_layernorm(int device, int M, int d, const float *x, const float *w1, const float *b1, const float *w2, const float *b2,
                              int want_f32, int planes, float *y1_f32, float *act_f32, float *hi, float *lo, int64_t *guard_bad);
/* Depthwise conv (ks taps, tap-major w [ks][d], folded BatchNorm bias [d]) + SiLU over packed utterances of g [rows_total][d].
 * Output [rows_total][d]: out_f32 with PK_MATH_FP32, else hi and, with PK_MATH_BF16X3, lo. */
pk_status pk_kernel_dwconv(int device, int math, int n_utt, const int32_t *row_off, int rows_total, int d, int ks, const float *g,
                           const float *w_tapmajor, const float *bias, float *out_f32, float *hi, float *lo, int64_t *guard_bad);
/* CTC head reduction of logits [M][ld]: best [M] (first maximum), conf [M] = exp(max log-prob), logprobs [M][V] (or NULL). */
pk_status pk_kernel_ctc_argmax(int device, int M, int V, int ld, const float *logits, int32_t *best, float *conf, float *logprobs,
                               int64_t *guard_bad);
/* The front end.  pk_kernel_mel: the offline log-mel (and, with normalize = 1, the per-utterance normalisation) of utterances
 * b = pcm[pcm_off[b] .. pcm_off[b+1]) (n >= 400 samples with normalize = 1, >= 2 without), 1 + n / 160 frames each, packed:
 * logmel_out [frames][n_mels] (with normalize = 0 the kernel's only output) and feats_out [frames][n_mels] (NULL with
 * normalize = 0).  n_mels a multiple of 8 up to 640.  pk_kernel_mel_stream: the streaming log-mel of already pre-emphasised
 * signals b = sig[sig_off[b] .. sig_off[b+1]), n_frames[b] frames (frame f reads samples 160 f .. 160 f + 511) into rows
 * out_row[b] + f of logmel_out [rows_total][n_mels]; the other rows are not written. */
pk_status pk_kernel_mel(int device, int n_utt, const int64_t *pcm_off, const float *pcm, int n_mels, int normalize, float *logmel_out,
                        float *feats_out, int64_t *guard_bad);
pk_status pk_kernel_mel_stream(int device, int n_streams, const int64_t *sig_off, const float *sig, const int32_t *n_frames,
                               const int32_t *out_row, int rows_total, int n_mels, float *logmel_out, int64_t *guard_bad);
/* The convolutional front of the subsampling (3x3 kernels, stride 2, zero padding 1; weights [C][9] unless noted).
 * pk_kernel_subsample_conv1: conv1_ (1 -> C) + ReLU + depthwise dw1_ of utterances b = feature rows [frame_off[b], frame_off[b+1])
 * of feats [rows_total][mel] (mel even, C a multiple of 4 up to 1024) -> rows (t2, f2) per utterance, packed, of C channels.
 * pk_kernel_subsample_dw: depthwise dw2_ (tap-major weights [9][C]) of utterances of in_rows[b] x fin rows of C channels
 * packed in `in` -> conv_len(in_rows[b]) x conv_len(fin) rows each, packed.  Output: out_f32 with PK_MATH_FP32, else hi and,
 * with PK_MATH_BF16X3, lo (the engine's activation operand). */
pk_status pk_kernel_subsample_conv1(int device, int math, int n_utt, const int32_t *frame_off, int rows_total, const float *feats, int mel,
                                    int C, const float *w1, const float *b1, const float *wd, const float *bd, float *out_f32, float *hi,
                                    float *lo, int64_t *guard_bad);
pk_status pk_kernel_subsample_dw(int device, int math, int n_utt, const int32_t *in_rows, int fin, int C, const float *in, const float *wd_tapmajor,
                                 const float *bd, float *out_f32, float *hi, float *lo, int64_t *guard_bad);

/* The TDT / RNN-T decode kernel (csrc/tdt.cu) on host fp32 inputs in the reference's layouts, with the TdtParams that the engine
 * builds: Bpad = n_utt rounded up to 32, LSTM weights reordered unit-major and split into bf16 hi/lo rows, the initial h split into
 * state plane 0.  n_dur = 0 is an RNN-T joint (max_sym symbols per frame).  Utterance b = rows [row_off[b], row_off[b+1]) of EP. */
typedef struct {
    int32_t P, J, V, n_dur, durations[8], L, max_sym;
    int32_t n_utt, rows;
    const int32_t *row_off;                /* [n_utt + 1] */
    const float *EP;                       /* [rows][J]   enc_proj(enc) + bias */
    const float *G0;                       /* [V][4P]     W_ih0 . E[token] + b_ih0 */
    const float *W_hh[4], *W_ih[4];        /* [4P][P] gate-major (i, f, g, o); W_ih for layers >= 1 */
    const float *b_ih[4];                  /* [4P], layers >= 1 */
    const float *W_p;                      /* [J][P] */
    const float *W_out, *b_out;            /* [V + n_dur][J], [V + n_dur] */
    int32_t cap, max_steps;
    int32_t carry;                         /* 1: carried state (the streaming decode): the four arrays below are read */
    const float *h0, *c0;                  /* [L][n_utt][P] committed LSTM state */
    const int32_t *tok0, *frame_base;      /* [n_utt] last token, absolute frame of the first row */
    int32_t cluster;                       /* 0 = the engine's choice, 2 / 4 = only that size (PK_ERR_INVALID if it does not fit) */
    int32_t max_ctas;                      /* 0 = every SM, else the SM count the launch plans for */
    int32_t no_stage;                      /* 1: no staging tile: weights that do not fit are read from L2 */
} pk_tdt_hook_in;
/* Outputs (every array guarded; NULL pointers are not fetched).  h, z and the keys are those of the LAST step: h_hi / h_lo
 * [L][2][n_utt][P] are both state planes of every layer (the step's new h sits in the plane the utterance's committed state
 * does not), z_hi / z_lo [n_utt][J]; lab_idx / dur_idx = -1 where no CTA posted a key (the utterance was idle, or no logit
 * was above -inf); lse [n_utt] = the label log-sum-exp from that step's per-CTA (max, sum) partials, combined in double.
 * With carry: c_state [L][n_utt][P], tok_state [n_utt] (h_hi / h_lo plane 0 holds the committed h). */
typedef struct {
    int32_t *tok;                          /* [n_utt][1 + cap]: len, ids */
    int32_t *t_start, *t_end;              /* [n_utt][cap] */
    float *t_conf;                         /* [n_utt][cap] */
    int32_t *overflow;                     /* [n_utt] */
    float *h_hi, *h_lo, *z_hi, *z_lo;
    float *lab_val, *dur_val;              /* [n_utt] */
    int32_t *lab_idx, *dur_idx;            /* [n_utt] */
    double *lse;                           /* [n_utt] */
    float *c_state;
    int32_t *tok_state;
    int32_t steps;
    int32_t grid, cl, upc, opc, out_in_smem, wih_in_smem, staged_ih, wstage_rows;
} pk_tdt_hook_out;
pk_status pk_kernel_tdt_decode(int device, const pk_tdt_hook_in *in, pk_tdt_hook_out *out, int64_t *guard_bad);
/* The same launch with phrase boosting on and a phrase list and score per row, laid out as pk_set_boost_rows takes them
 * (dec.n_dur > 0; n_utt rows).  With dec.carry the trie state on entry is trie_active0 [n_utt][64] / trie_nact0 [n_utt] (the
 * bitmap follows from them); without, every row starts at the root.  Out: the decode's outputs plus the state on exit,
 * trie_active [n_utt][64] (the first trie_nact[b] entries of a row are written), trie_nact [n_utt] and boost_bits
 * [n_utt][(V + 31) / 32], all guarded. */
typedef struct {
    pk_tdt_hook_in dec;
    const int32_t *phrase_ids, *phrase_off, *row_off;
    const float *boost;                    /* [n_utt] */
    const int32_t *trie_active0, *trie_nact0;
} pk_tdt_boost_hook_in;
typedef struct {
    pk_tdt_hook_out dec;
    int32_t *trie_active, *trie_nact;
    uint32_t *boost_bits;
} pk_tdt_boost_hook_out;
pk_status pk_kernel_tdt_decode_boosted(int device, const pk_tdt_boost_hook_in *in, pk_tdt_boost_hook_out *out, int64_t *guard_bad);
/* Streaming kernels as pk_stream_step launches them for one layer.  n_active of n_streams streams take part:
 * act_stream[a] is stream a's id, its rows are [row_off[a], row_off[a+1]) of the packed step (rows_total in all).
 * Per-stream state is indexed by stream id and updated in place; the updated state comes back in the *_out arrays.
 * pk_kernel_stream_attention: cached attention (streaming_encoder.cpp:160-272) of qkv [rows_total][3 d] (q | k | v),
 *   keys = [ring rows (oldest first) | the chunk's rows]; the ring of stream s is kc/vc [s][L][d] holding cache_len[s] rows
 *   from slot ring_start[s] on (mod L); pp [(2 tmax - 1)][d] the projected position table, pos_u / pos_v [d].  Needs
 *   L + max chunk rows <= tmax.  Output ctx [rows_total][d]: ctx_f32 with PK_MATH_FP32, else hi and, with
 *   PK_MATH_BF16X3, lo; kc_out / vc_out [n_streams][L][d] the rings after the chunk's rows went in.
 * pk_kernel_stream_dwconv: cached causal depthwise conv + folded BatchNorm + SiLU (streaming_encoder.cpp:41-80) of
 *   glu [rows_total][d]; w [d][ks] (channel-major), bias [d]; cache [n_streams][ks - 1][d] the last ks - 1 inputs of
 *   every stream.  Output as above; cache_out [n_streams][ks - 1][d]. */
pk_status pk_kernel_stream_attention(int device, int math, int n_streams, int n_active, const int32_t *act_stream, const int32_t *row_off,
                                     int rows_total, const int32_t *cache_len, const int32_t *ring_start, int L, int d_model, int n_heads,
                                     int tmax, const float *qkv, const float *pp, const float *pos_u, const float *pos_v, const float *kc,
                                     const float *vc, float *ctx_f32, float *ctx_hi, float *ctx_lo, float *kc_out, float *vc_out,
                                     int64_t *guard_bad);
pk_status pk_kernel_stream_dwconv(int device, int math, int n_streams, int n_active, const int32_t *act_stream, const int32_t *row_off,
                                  int rows_total, int d, int ks, const float *glu, const float *w, const float *bias, const float *cache,
                                  float *out_f32, float *hi, float *lo, float *cache_out, int64_t *guard_bad);

/* Host-side text helpers (pure C++ host code; no device work):
 * Tokenizer::load/decode (src/vocab.cpp:10-64), group_timestamps (src/timestamp.cpp:24-75). */
typedef struct pk_vocab pk_vocab;
pk_status pk_vocab_load(const char *vocab_path, pk_vocab **out);
void pk_vocab_free(pk_vocab *v);
int32_t pk_vocab_size(const pk_vocab *v);
/* Longest piece in bytes: pk_detokenize / pk_group_words never write more than n * (that + 1) + 1 bytes for n tokens. */
int32_t pk_vocab_max_piece_bytes(const pk_vocab *v);
/* Writes NUL-terminated UTF-8 into buf (truncated to cap-1); returns full length. */
int32_t pk_detokenize(const pk_vocab *v, const int32_t *ids, int32_t n, char *buf, int32_t cap);
/* Words are written '\n'-separated into buf; returns the number of words. */
int32_t pk_group_words(const pk_vocab *v, const int32_t *ids, const int32_t *start,
                       const int32_t *end, const float *conf, int32_t n, char *buf, int32_t cap,
                       float *w_start, float *w_end, float *w_conf);

/* Tokenizer::encode (src/vocab.cpp:76-117): U+2581-prefixed, spaces -> U+2581, greedy longest piece match on
 * bytes, unknown bytes skipped.  Writes at most cap ids; returns the full count. */
int32_t pk_tokenize(const pk_vocab *v, const char *text, int32_t *ids, int32_t cap);

/* Phrase-boosted CTC greedy decode of ONE utterance on the host (widening row: SURVEY.md section 8f(3)), replacing
 * ctc_greedy_decode_boosted / ctc_greedy_decode_with_timestamps_boosted (src/phrase_boost.cpp:70-176) and the
 * ContextTrie they use (:9-66).  logprobs = (n_frames, vocab) row-major as returned by pk_ctc_logprobs; the
 * phrases are token-id sequences (pk_tokenize), phrase p = phrase_ids[phrase_off[p] .. phrase_off[p+1]).
 * Every frame takes argmax_v(logprob[v] + boost * [v continues an active phrase]) (first maximum), the trie
 * advances on emissions, confidences are exp of the UNboosted log-prob.  start / end / conf may be NULL.
 * Returns the number of tokens (at most `cap` are written) or -1 on invalid arguments. */
int32_t pk_ctc_decode_boosted(const float *logprobs, int32_t n_frames, int32_t vocab, int32_t blank,
                              const int32_t *phrase_ids, const int32_t *phrase_off, int32_t n_phrases, float boost,
                              int32_t *ids, int32_t *start, int32_t *end, float *conf, int32_t cap);

/* Phrase boosting ON THE DEVICE for both decoders (widening row: SURVEY.md section 8f(3)), replacing the decode loops of
 * ctc_greedy_decode(_with_timestamps)_boosted and tdt_greedy_decode(_with_timestamps)_boosted (src/phrase_boost.cpp:70-352)
 * as Transcriber::transcribe uses them when TranscribeOptions::boost_phrases is set (transcribe.hpp:110-137, :158-165).
 * The phrases are token-id sequences (pk_tokenize), phrase p = phrase_ids[phrase_off[p] .. phrase_off[p+1]); the engine builds the
 * ContextTrie (:9-66) and keeps it on the device.  While set, every decode of this engine (pk_transcribe_batch,
 * pk_run_staged, pk_decode; CTC and TDT) adds `boost` to the label scores of the tokens that continue an active phrase;
 * the trie state is per utterance and advances on emissions; confidences stay exp(raw log-prob).  n_phrases = 0 clears
 * it.  This call gives every utterance the SAME list and score (and synchronises the engine stream); pk_set_boost_rows
 * gives each utterance its own, pk_stream_set_boost each stream.  At most 64 simultaneously active trie states per
 * utterance.  The reference has no boosted RNN-T decode: on an RNN-T model a non-empty phrase list is PK_ERR_INVALID.
 * pk_stream_open is also PK_ERR_INVALID there (streaming decodes eou's TDT joint). */
pk_status pk_set_boost(pk_engine *e, const int32_t *phrase_ids, const int32_t *phrase_off, int32_t n_phrases, float boost);
/* Phrase lists per utterance, as TranscribeOptions::boost_phrases / boost_score belong to one transcribe() call of the
 * reference (transcribe.hpp:38-43): for the following decodes (pk_transcribe_batch, pk_run_staged, pk_decode; CTC and TDT) row i
 * of the batch uses phrases [row_off[i], row_off[i+1]) of (phrase_ids, phrase_off) with score boost[i], and decodes as the
 * reference's *_boosted functions do on that utterance alone.  An empty range = that row decodes unboosted, bit for bit
 * as with boosting off; rows >= n_rows of a later batch decode unboosted.  n_rows = 0 clears.  Replaces, and is replaced by,
 * pk_set_boost.  Each row's trie lives in a slot of PK_BOOST_ROW_NODES nodes (root included): a longer list is
 * PK_ERR_CAPACITY (the message names the row) and leaves the previous lists in force; n_rows > max_batch likewise.  The
 * upload is ordered on the engine stream and does not synchronise, and changing lists re-captures no CUDA graph, so the call
 * can be made for every batch of the pk_stage_pcm / pk_run_staged / pk_prefetch_pcm / pk_fetch_tokens pipeline.  RNN-T model
 * with any phrase, Sortformer engine: PK_ERR_INVALID. */
#define PK_BOOST_ROW_NODES 1024
pk_status pk_set_boost_rows(pk_engine *e, const int32_t *phrase_ids, const int32_t *phrase_off, const int32_t *row_off,
                            const float *boost, int32_t n_rows);
/* The same for ONE open stream (0 <= stream < n_streams of pk_stream_open): takes effect from the next pk_stream_step, puts
 * that stream's trie state back at the root, leaves its encoder caches / LSTM state / tokens and every other stream alone.
 * n_phrases = 0 turns boosting off for the stream.  A boosted stream decodes as rnnt_streaming_decode_chunk (src/eou.cpp:17-98)
 * with the label arg-max, trie advance and confidence of tdt_greedy_decode_with_timestamps_boosted (src/phrase_boost.cpp:266-352);
 * the active trie states are carried from chunk to chunk (a phrase may straddle chunks) and pk_stream_reset returns them to
 * the root, keeping the list (DESIGN.md section 8). */
pk_status pk_stream_set_boost(pk_engine *e, int32_t stream, const int32_t *phrase_ids, const int32_t *phrase_off,
                              int32_t n_phrases, float boost);

/* ---- CTC prefix beam search with word n-gram (ARPA) shallow fusion (DESIGN.md section 14 defines the decode).
 * Per frame every beam is extended by the `width` best non-blank tokens of the frame; candidates with the same token
 * sequence merge; each is ranked by ln P(prefix) + lm, lm = alpha ln(10) sum log10 p(word | history) + beta (words scored),
 * over the completed words (a piece starting with U+2581 starts a word; words are the UTF-8 of their pieces without that
 * mark, compared as bytes; a word the LM lacks scores as <unk>).  At the end the unfinished word and </s> are scored and the
 * best beam is backtracked into the greedy layout of pk_tokens (start = frame the token was appended, end = next start - 1,
 * conf = exp(log-prob at start)).
 *
 * The LM is a host object: pk_lm_load reads an ARPA file of order 1..6 (\data\ counts, \k-grams: sections of
 * "log10prob w1 .. wk [log10backoff]", \end\).  PK_ERR_IO, with the line in pk_last_error(NULL), for a count that does not
 * match its section, an n-gram whose context (or word) is not in the file, a field that does not parse, a missing \end\,
 * or two words with the same 64-bit FNV-1a hash.  Without <unk> one is added (log10 p = -10, backoff 0).  Scoring is
 * standard ARPA back-off from the longest present suffix of the history, starting from the <s> unigram when present.
 *   pk_lm_count          : number of n-grams of `order` (1..pk_lm_order), <unk> included when it was added.
 *   pk_lm_sentence_log10 : log10 p of the space-separated words followed by </s>, starting from <s> (NaN: bad argument).
 *   pk_set_ctc_beam      : the beam width (1..PK_CTC_BEAM_MAX) for PK_DECODER_CTC_BEAM on this engine, and the LM (NULL:
 *                          none; then vocab may be NULL and alpha / beta are unused) with the tokenizer whose pieces the
 *                          model emits.  The LM's tables are copied to the device, so the pk_lm may be freed afterwards.
 *                          They are copied only when the LM (a new pk_lm_load) or the vocabulary's pieces differ from the
 *                          tables in place: that call synchronises the engine stream and frees the previous tables.  A call
 *                          that repeats the LM and vocabulary (say, once per request) copies nothing and does not
 *                          synchronise; width, alpha and beta may change on any call.  PK_DECODER_CTC_BEAM is PK_ERR_INVALID before this call, on a
 *                          model without a CTC head, on a Sortformer engine, and while phrase boosting is set. */
#define PK_CTC_BEAM_MAX 32
typedef struct pk_lm pk_lm;
pk_status pk_lm_load(const char *arpa_path, pk_lm **out);
void pk_lm_free(pk_lm *lm);
int32_t pk_lm_order(const pk_lm *lm);
int64_t pk_lm_count(const pk_lm *lm, int32_t order);
double pk_lm_sentence_log10(const pk_lm *lm, const char *space_separated_words);
pk_status pk_set_ctc_beam(pk_engine *e, int32_t width, const pk_lm *lm_or_null, const pk_vocab *vocab, float alpha, float beta);
/* Kernel test hook (conventions of the pk_kernel_* hooks): the two beam-search kernels as the engine launches them, on host
 * log-probs [rows][V] (blank = V - 1), utterance b = rows [row_off[b], row_off[b+1]).  lm / vocab as pk_set_ctc_beam.
 * Outputs, all guarded: tok [n_utt][1 + cap] (len, ids), t_start / t_end / t_conf [n_utt][cap], topk_id / topk_lp
 * [rows][width] (absent entries: id -1), blank_lp [rows], bp [rows][width] (back-pointers: parent slot << 24 | (token + 1),
 * written for the slots alive after each frame).  Any output but tok may be NULL. */
pk_status pk_kernel_ctc_beam(int device, int n_utt, const int32_t *row_off, int rows, int V, const float *logprobs, int width,
                             const pk_lm *lm, const pk_vocab *vocab, float alpha, float beta, int cap, int32_t *tok, int32_t *t_start,
                             int32_t *t_end, float *t_conf, int32_t *topk_id, float *topk_lp, float *blank_lp, int32_t *bp,
                             int64_t *guard_bad);

/* ---- CTC forced alignment (DESIGN.md section 15 defines it): the timestamps of a KNOWN token sequence y_1..y_L per
 * utterance, by the Viterbi pass over the CTC trellis of z = (blank, y_1, blank, ..., y_L, blank) (blank = vocab - 1),
 * S = 2L + 1 states, on the fp32 log-probs lp[t][v] of the CTC head, accumulated in double:
 *   delta_0(0) = lp[0][blank], delta_0(1) = lp[0][y_1], other states -inf;
 *   delta_t(s) = lp[t][z_s] + max(delta_{t-1}(s), delta_{t-1}(s-1), delta_{t-1}(s-2)), the s-2 term only when z_s is not
 *   blank and z_s != z_{s-2}; ties prefer s, then s-1, then s-2.  The path ends in S-1 or S-2, whichever is larger (a tie
 *   goes to S-1); the alignment score is that maximum.  The CTC log-likelihood log p(y | x) is the same trellis with
 *   log-sum-exp in place of max, lse(alpha_{T-1}(S-1), alpha_{T-1}(S-2)).
 * A row with T < L + R frames (R = number of i with y_i = y_{i+1}), or whose best path has probability 0, cannot be aligned:
 * it gets zero tokens and both scores are -inf (a per-row outcome, not an error).  L = 0 aligns every frame to blank.
 * The path's label of every frame goes through the greedy CTC collapse, so a row of pk_tokens has the layout and meaning of
 * a greedy CTC row: start = first frame of the token, end = the frame before the next token's (the last token ends at
 * T-1), conf = exp(lp[start][token]).  Aligning the greedy transcript gives back the greedy row.
 *   pk_set_align_targets  : the token ids of each row of the next PK_DECODER_CTC_ALIGN run, row i = ids[offsets[i] ..
 *                           offsets[i+1]), n_rows <= max_batch (n_rows = 0 clears them; ids and offsets may then be NULL).  The
 *                           ids are copied (ordered on the engine stream, no synchronisation) into buffers that never move,
 *                           so one CUDA graph per batch shape serves every set of targets.  PK_ERR_INVALID: an id outside
 *                           0..vocab-2 (the blank included; pk_last_error names the row), decreasing offsets, a model without
 *                           a CTC head, a Sortformer engine.  PK_ERR_CAPACITY: a row of more than PK_ALIGN_MAX_TOKENS ids.
 *                           Either error leaves the previous targets in force.
 *   pk_fetch_align_scores : the alignment score and log p(y | x) of each row of the last run (either pointer may be NULL);
 *                           PK_ERR_INVALID when the last run was not an alignment.
 * PK_DECODER_CTC_ALIGN works through pk_run_staged, pk_transcribe_batch, pk_decode and jobs; it is PK_ERR_INVALID without
 * targets, with a number of target rows other than the batch's, on a model without a CTC head, on a Sortformer engine, and
 * in pk_transcribe_diarize_batch / pk_run_transcribe_diarize_staged.  Phrase boosting does not change an alignment. */
#define PK_ALIGN_MAX_TOKENS 2048
pk_status pk_set_align_targets(pk_engine *e, const int32_t *ids, const int32_t *offsets, int32_t n_rows);
pk_status pk_fetch_align_scores(pk_engine *e, double *score, double *loglik);
/* Kernel test hook (conventions of the pk_kernel_* hooks): the alignment kernel and the greedy collapse as the engine
 * launches them, on host log-probs [rows][V] (blank = V - 1), utterance b = rows [row_off[b], row_off[b+1]), with targets
 * b = tgt[tgt_off[b] .. tgt_off[b+1]).  Outputs, all guarded: tok [n_utt][1 + cap] (len, ids), t_start / t_end / t_conf
 * [n_utt][cap], score / loglik [n_utt], path [rows] (the best path's state of every frame, -1 in an infeasible row).  Any
 * output but tok may be NULL.  Errors as pk_set_align_targets. */
pk_status pk_kernel_ctc_align(int device, int n_utt, const int32_t *row_off, int rows, int V, const float *logprobs, const int32_t *tgt,
                              const int32_t *tgt_off, int cap, int32_t *tok, int32_t *t_start, int32_t *t_end, float *t_conf, double *score,
                              double *loglik, int32_t *path, int64_t *guard_bad);

/* Offline speaker diarization: Sortformer (include/parakeet/sortformer.hpp, src/sortformer.cpp:42-122 of the reference).
 * PCM -> log-mel WITHOUT per-bin normalisation (main.cpp:514-517) -> NEST encoder (the offline FastConformer under keys
 * "nest_encoder_.", subsampling output times sqrt(d_model), streaming_encoder.cpp:399-423) -> projection_ -> transformer_
 * (post-norm blocks, head_dim 24, transformer.cpp:15-62) -> sigmoid(output_proj_(ReLU(first_hidden_(ReLU(.))))).
 * enc: the NEST encoder's shape plus the engine capacity and math (decoder fields are ignored). */
typedef struct {
    pk_config enc;
    int32_t t_hidden;       /* 192 */
    int32_t t_layers;       /* 18 */
    int32_t t_heads;        /* 8 (head_dim 24: the only one the attention kernel takes) */
    int32_t t_ff;           /* 768 */
    int32_t max_speakers;   /* 4 */
} pk_sortformer_config;
/* make_sortformer_117m_config (sortformer.hpp:43-72): NEST 17 x d 512, 8 heads, ff 2048, 128 mels, 256 subsampling channels;
 * transformer 18 x d 192, 8 heads, ff 768; 4 speakers.  Capacity: 16 utterances of 90 s, bf16x3. */
void pk_config_sortformer_117m(pk_sortformer_config *cfg);
/* An engine in diarization mode.  Required keys: nest_encoder_.*, projection_, transformer_.layers_.{i}.{norm1_, mha_.{q,k,v,out}_proj,
 * norm2_, fc1_, fc2_}, first_hidden_, output_proj_ (hidden_to_spks_ is not used and not required).  On it pk_mel, pk_encode
 * (the NEST encoder output), pk_stage_pcm, the profile calls and pk_last_error work; the decode, boosting and ASR streaming
 * (pk_stream_*) entry points return PK_ERR_INVALID.  Its streams are the pk_diar_stream_* calls below. */
pk_status pk_sortformer_create(const pk_sortformer_config *cfg, const char *safetensors_path, int device, pk_engine **out);
/* Sortformer::forward on a batch of features (packed (sum frames_i, mel_bins), as pk_mel returns them): probs_out packed
 * (sum T'_i, max_speakers) sigmoid activities, t_out[n_utt] = T'_i (may be NULL). */
pk_status pk_sortformer_forward(pk_engine *e, const float *feats, const int32_t *n_frames, int32_t n_utt, float *probs_out, int32_t *t_out);
/* The whole path from 16 kHz PCM (utterance i = pcm[offsets[i] .. offsets[i+1])); outputs as pk_sortformer_forward. */
pk_status pk_diarize_batch(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, float *probs_out, int32_t *t_out);
/* Device-resident form (measurement): pk_stage_pcm, then pk_run_diarize_staged (one CUDA graph per batch shape after the front
 * end), then pk_fetch_probs. */
pk_status pk_run_diarize_staged(pk_engine *e);
pk_status pk_fetch_probs(pk_engine *e, float *probs_out, int32_t *t_out);
/* Sortformer::probs_to_segments (sortformer.cpp:70-113) for one utterance, on the host: probs [T][S]; a frame is active when
 * p > threshold; a segment is [start frame, last active frame] in seconds (frame * 0.08 s); segments sorted by start, equal
 * starts by speaker id.  Writes at most cap segments; returns their full number, or -1 on invalid arguments. */
int32_t pk_diar_segments(const float *probs, int32_t T, int32_t S, float threshold, int32_t *spk, float *start, float *end, int32_t cap);
/* Speaker-attributed transcription (DiarizedTranscriber, include/parakeet/diarize.hpp; diarize.cpp of the reference): one batch
 * through an ASR engine and a Sortformer engine on the same device.  The PCM is copied to the device once, into asr's buffer
 * (pk_stage_pcm's staging); diar's front end reads it from there, and asr does not overwrite or swap that buffer (next
 * pk_stage_pcm, pk_prefetch_pcm) before diar has read it.  tokens_out as pk_transcribe_batch on asr, probs_out / t_out as
 * pk_diarize_batch on diar.  PK_ERR_INVALID: engines on different devices, asr a Sortformer or RNN-T engine, diar not a
 * Sortformer engine, dec not CTC or TDT.  An n_utt or utterance length over either engine's capacity: PK_ERR_CAPACITY, with
 * nothing staged.  Errors are reported by pk_last_error(asr).  Phrase boosting set on asr applies as in pk_transcribe_batch. */
pk_status pk_transcribe_diarize_batch(pk_engine *asr, pk_engine *diar, const float *pcm, const int64_t *offsets, int32_t n_utt,
                                      pk_decoder dec, pk_tokens *tokens_out, float *probs_out, int32_t *t_out);
/* Device-resident form (measurement): pk_stage_pcm(asr, ...) (or pk_prefetch_pcm + pk_stage_pcm), then
 * pk_run_transcribe_diarize_staged, then pk_fetch_tokens(asr) and pk_fetch_probs(diar).  diar keeps no PCM of this batch:
 * pk_run_diarize_staged on it needs a pk_stage_pcm of its own first. */
pk_status pk_run_transcribe_diarize_staged(pk_engine *asr, pk_engine *diar, pk_decoder dec);
/* diarize_transcription (diarize.cpp:10-48) on the host: word w gets the speaker with the largest summed overlap
 * min(end) - max(start) (float32 seconds; only overlaps > 0 count) over the segment list in its order, or -1 when none
 * overlaps; exact ties resolve as the reference's std::unordered_map does (DESIGN.md section 13). */
pk_status pk_diarize_transcription(const float *word_start, const float *word_end, int32_t n_words, const int32_t *seg_spk,
                                   const float *seg_start, const float *seg_end, int32_t n_segs, int32_t *word_spk);
/* One utterance of DiarizedTranscriber::transcribe after the models: the segments of probs [T][S] in the reference's own
 * order (per speaker, then std::sort by start: above 16 segments equal starts need not stay in speaker order, unlike
 * pk_diar_segments) -- at most seg_cap of them written -- and word_spk[n_words] from pk_diarize_transcription on them.
 * Word times in seconds (pk_group_words).  Returns the number of segments, or -1 on invalid arguments. */
int32_t pk_diarize_words(const float *probs, int32_t T, int32_t S, float threshold, const float *word_start, const float *word_end,
                         int32_t n_words, int32_t *word_spk, int32_t *seg_spk, float *seg_start, float *seg_end, int32_t seg_cap);
/* Streaming diarization: Sortformer::diarize_chunk (sortformer.cpp:124-150) with one EncoderCache and AOSCCache per stream,
 * n_streams streams in lock step on a Sortformer engine (the pk_stream_* conventions).  Per stream and step: the chunk's own
 * centred log-mel without normalisation (preprocess_audio(chunk, {n_mels = mel_bins, normalize = false}); nothing carries
 * over between chunks), the NEST encoder's forward_chunk (leftover mel frames, K/V rings of att_context_left rows, conv
 * caches), then projection_ -> transformer_ -> speaker head on THIS chunk's encoder rows only (no context across chunks, as
 * in the reference), and the AOSC update (a speaker arrives the first time its p > 0.5; within a frame in index order).
 *   pk_diar_stream_open : capacity as pk_stream_open: n_streams <= max_batch, att_context_left + encoder frames per chunk
 *                         <= the engine's encoder-frame capacity (PK_ERR_CAPACITY otherwise).  On an ASR engine: PK_ERR_INVALID.
 *   pk_diar_stream_step : stream s receives pcm[offsets[s] .. offsets[s+1]) (16 kHz; empty = no input this step; a chunk
 *                         over max_chunk_samples is PK_ERR_CAPACITY, a 1-sample chunk PK_ERR_INVALID: the reference's
 *                         reflect pad does not terminate there).  probs_out packed (sum C_s, max_speakers) sigmoid
 *                         activities of this step, n_out[s] = C_s (0: the reference returns {} and the AOSC is not
 *                         updated), frame_base_out[s] = the absolute encoder frame of the stream's first row (probs are
 *                         chunk-local: segments restart at frame 0 in every chunk).  enc_out (may be NULL): debug tap of
 *                         the NEST encoder rows, packed (sum C_s, d_model).  Any output pointer may be NULL.
 *   pk_diar_stream_step_feats : the same from host features, stream s = n_frames[s] rows of feats packed (sum, mel_bins)
 *                         (diarize_chunk's own input; n_frames[s] <= 1 + max_chunk_samples / 160).
 *   pk_diar_stream_speakers : AOSCCache::speaker_order of one stream; writes at most cap ids, returns their number (-1 on
 *                         invalid arguments).
 *   pk_diar_stream_reset : a fresh EncoderCache and AOSCCache::reset for one stream (-1: all). */
pk_status pk_diar_stream_open(pk_engine *e, int32_t n_streams, int32_t max_chunk_samples, int32_t att_context_left);
pk_status pk_diar_stream_reset(pk_engine *e, int32_t stream);
pk_status pk_diar_stream_step(pk_engine *e, const float *pcm, const int64_t *offsets, float *probs_out, int32_t *n_out,
                              int32_t *frame_base_out, float *enc_out);
pk_status pk_diar_stream_step_feats(pk_engine *e, const float *feats, const int32_t *n_frames, float *probs_out, int32_t *n_out,
                                    int32_t *frame_base_out, float *enc_out);
int32_t pk_diar_stream_speakers(const pk_engine *e, int32_t stream, int32_t *order, int32_t cap);
int32_t pk_diar_stream_count(const pk_engine *e);
/* Kernel test hooks (conventions of the pk_kernel_* hooks above).  pk_kernel_mha: the transformer attention on qkv [rows_total][3 d]
 * fp32 (q | k | v), head_dim 24 only (else PK_ERR_INVALID); ctx [rows_total][d] in ctx_f32 with PK_MATH_FP32, else ctx_hi and,
 * with PK_MATH_BF16X3, ctx_lo.  pk_kernel_speaker_head: x [M][D], w1 [D][D], b1 [D], w2 [S][D], b2 [S] -> probs [M][S]. */
pk_status pk_kernel_mha(int device, int math, int n_utt, const int32_t *row_off, int rows_total, int d_model, int n_heads, const float *qkv,
                        float *ctx_f32, float *ctx_hi, float *ctx_lo, int64_t *guard_bad);
pk_status pk_kernel_speaker_head(int device, int M, int D, int S, const float *x, const float *w1, const float *b1, const float *w2,
                                 const float *b2, float *probs, int64_t *guard_bad);

/* Sample-rate conversion (widening row: SURVEY.md section 8f(4)), replacing parakeet::resample / sinc_resample
 * (src/audio_io.cpp:123-195, :238-251): 32-tap Kaiser (beta 7.857) windowed sinc in double, output length
 * ceil(n * dst / src) (pk_resample_len), implemented as a POLYPHASE filter: the weights depend only on the phase
 * (i * down) mod up, so they are tabulated once per rate pair (csrc/resample.cu).
 *   pk_stage_pcm_rate : like pk_stage_pcm for a batch recorded at `src_rate`: the raw samples go to the device and are
 *                       converted there straight into the staged 16 kHz batch (read_audio's resampling, audio_io.cpp:227-232,
 *                       without a host pass).  Utterance lengths are checked at 16 kHz.
 *   pk_resample_batch : device conversion of a batch between arbitrary rates, results back to the host
 *                       (out_offsets = prefix sums of pk_resample_len per utterance).
 *   pk_resample       : the same filter evaluated on the host for engine-less callers (parakeet::resample of the C++
 *                       shim); writes at most `cap` samples, returns the full length or -1 on invalid arguments. */
int64_t pk_resample_len(int64_t n, int32_t src_rate, int32_t dst_rate);
int64_t pk_resample(const float *in, int64_t n, int32_t src_rate, int32_t dst_rate, float *out, int64_t cap);
pk_status pk_stage_pcm_rate(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, int32_t src_rate);
pk_status pk_resample_batch(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, int32_t src_rate,
                            int32_t dst_rate, float *out, const int64_t *out_offsets);

#ifdef __cplusplus
}
#endif
#endif /* PARAKEET_B200_H */
