// kernels.h -- host-callable launchers of the sm_90a kernels (one .cu per op group).
#pragma once
#include <cuda.h>

#include <algorithm>
#include <functional>
#include <string>
#include <vector>

#include "pk_common.cuh"

#define PK_MAX_LSTM 4

struct pk_lm;
struct pk_vocab;

namespace pk {

// ------------------------------------------------------------------ mel.cu (K1, K2)
struct MelTables {
    const float *window;    // [400] symmetric Hann (fp32 of the double formula)
    const float2 *tw256;    // [256] exp(-2 pi i m / 256)
    const float2 *tw512;    // [257] exp(-2 pi i k / 512)
    const float *fb_w;      // non-zero filterbank weights, filter-major
    const int32_t *fb_start, *fb_len, *fb_off;   // [n_mels]
    int fb_nnz;
};
// The tables for n_mels bins, built on the host; every array goes through upload(host, bytes) -> device pointer
// (nullptr: out of memory).
MelTables build_mel_tables(int n_mels, const std::function<void *(const void *, size_t)> &upload);
// K2 runs MEL_NORM_THREADS / n_mels frame groups of n_mels threads: the normalisation needs n_mels <= MEL_NORM_THREADS.
constexpr int MEL_NORM_THREADS = 640;
size_t mel_smem_bytes(const MelTables &tb);
// part: scratch of mel_part_floats(n_utt, n_mels) floats (per-chunk statistics of the normalisation), one slice per utterance
size_t mel_part_floats(int n_utt, int n_mels);
// normalize = false (Sortformer: preprocess_audio with AudioConfig::normalize off, main.cpp:514-517): K1 only, the
// log-mel lands in feats and logmel / part are not used.
void launch_mel(const float *pcm, const int64_t *pcm_off, const int32_t *frame_off, int n_utt, int max_frames,
                int n_mels, const MelTables &tb, float *logmel, float *feats, float *part, cudaStream_t st, bool normalize = true);

// streaming variant (StreamingAudioPreprocessor::process_chunk, src/audio.cpp:195-259): `sig` holds, per stream, the
// already pre-emphasised samples [overlap | chunk]; frame f = window . sig[f*160 .. f*160+512) (center = False, no
// reflection), n_frames[b] frames, log-mel WITHOUT normalisation written to logmel rows out_row[b] + f.
void launch_mel_stream(const float *sig, const int64_t *sig_off, const int32_t *n_frames, const int32_t *out_row, int n_streams,
                       int max_frames, int n_mels, const MelTables &tb, float *logmel, cudaStream_t st);

// ------------------------------------------------------------------ stream.cu (streaming eou path)
constexpr int STREAM_OVL_CAP = 512;   // overlap buffer per stream (< 400 samples are ever kept, audio.cpp:225-240)
struct StreamPlan {                   // one row per stream and step, computed on the host from the chunk sizes
    int64_t chunk_off;                // offset of this stream's chunk in the packed chunk buffer
    int64_t sig_off;                  // offset of [overlap | pre-emphasised chunk] in the signal scratch
    int32_t chunk_len, ovl_len;       // samples in the chunk / carried overlap
    int32_t consumed;                 // samples covered by the frames of this step (0: none; overlap = whole signal)
    int32_t nf;                       // new mel frames (the reference's STFT yields one fewer than its own count, DESIGN.md)
    int32_t left;                     // leftover mel frames from the previous steps (< 8)
    int32_t min_off;                  // first row of [leftover | new] frames in mel_in
    int32_t take;                     // frames consumed by the subsampling this step (multiple of 8)
    int32_t feat_off;                 // first row in the packed encoder input (valid if take > 0)
};
struct StreamState {
    float *ovl;                       // [S][STREAM_OVL_CAP]
    float *last;                      // [S] pre-emphasis carry (audio.cpp:206-213)
    float *melq;                      // [S][8][n_mels] leftover mel frames (streaming_encoder.cpp:348-385)
};
void launch_stream_prep(const float *chunk, const StreamPlan *plan, StreamState st, int n_streams, float *ssig, float *mel_in,
                        int n_mels, cudaStream_t s);
void launch_stream_post(const float *chunk, const StreamPlan *plan, StreamState st, int n_streams, const float *ssig,
                        const float *mel_in, int n_mels, float *feats, cudaStream_t s);
// Sortformer streams: per stream, [melq (plan.left rows) | mel_new rows plan.min_off .. + plan.nf] -> the first plan.take
// rows to feats row plan.feat_off, the rest (< 8) back into melq.  No sample overlap, no pre-emphasis carry.
void launch_diar_stream_join(const StreamPlan *plan, const float *mel_new, float *melq, int n_streams, int n_mels, float *feats,
                             cudaStream_t s);
bool launch_stream_attention(const float *qkv, int ld_qkv, const int32_t *row_off, const int32_t *act_stream, int n_active,
                             int max_C, const int32_t *cache_len, const int32_t *ring_start, float *kc, float *vc, int L,
                             int n_heads, int hd, int d_model, const float *pp, int tmax, const float *bu, const float *bv,
                             ActBuf out, cudaStream_t s);
bool launch_stream_dwconv(const float *glu, const int32_t *row_off, const int32_t *act_stream, int n_active, float *cache, int d,
                          int ks, const float *w, const float *bias, ActBuf out, cudaStream_t s);

// ------------------------------------------------------------------ resample.cu (front-of-path rate conversion)
// utterance b: in[in_off[b] .. in_off[b+1]) at src_rate -> out[out_off[b] .. out_off[b+1]) at dst_rate (lengths = pk_resample_len)
bool launch_resample(const float *in, const int64_t *in_off, const int64_t *out_off, int n_utt, int64_t max_out, int src_rate,
                     int dst_rate, float *out, cudaStream_t st);

// ------------------------------------------------------------------ subsample.cu (K3, K4)
void launch_subsample_conv1_dw1(const float *feats, const int32_t *frame_off, const int32_t *s2_off, int n_utt,
                                int max_t2, int mel, int C, const float *w1, const float *b1, const float *wd,
                                const float *bd, ActBuf out, cudaStream_t st);
void launch_subsample_dw(const float *in, const int32_t *in_rows, const int32_t *in_off, const int32_t *out_off,
                         int n_utt, int fin, int C, const float *wd, const float *bd, ActBuf out,
                         int total_out_rows, cudaStream_t st);

// ------------------------------------------------------------------ gemm_simt.cu / gemm_tc.cu (K5)
void launch_gemm_simt(const float *A, int lda, const float *W, int ldw, int M, int N, int K,
                      const EpiParams &epi, cudaStream_t st);

// wgmma path (gemm_tc.cu): a K-major bf16 matrix [rows][K] as TMA tensor maps of its hi
// (and lo) split planes, box = 64 (K) x box_rows, SWIZZLE_128B.
struct TcOperand {
    CUtensorMap hi, lo;
    bool has_lo = false;
    uint32_t box_rows = 0;
};
bool make_tc_operand(TcOperand *out, const bf16 *hi, const bf16 *lo, uint64_t rows, uint64_t K, uint32_t box_rows);
int tc_tile_n(int N);        // N-tile (= box_rows of the weight operand) chosen for an [N][K] weight
// cl = 2 | 4 with A_slice = the A operand with a 128 / cl-row box: clusters of cl CTAs along N that share (TMA multicast) the
// A tile; taken when gemm_tc_cluster_supported(N, epi.kind, cl), else the plain persistent kernel.
bool gemm_tc_cluster_supported(int N, int epi_kind, int cl);
cudaError_t launch_gemm_tc(const TcOperand &A, const TcOperand &W, int M, int N, int K, bool split3,
                           const EpiParams &epi, cudaStream_t st, int cl = 1, const TcOperand *A_slice = nullptr);

// ------------------------------------------------------------------ gemm_skinny.cu (M <= 128: the streaming path's GEMMs)
size_t gemm_skinny_ws_floats(int max_n, int max_splits);
cudaError_t launch_gemm_skinny(const bf16 *Ahi, const bf16 *Alo, int lda, const bf16 *Whi, const bf16 *Wlo, int M, int N, int K, bool split3,
                               const EpiParams &epi, float *ws, size_t ws_floats, unsigned int *tickets, int n_tickets, int num_sms,
                               cudaStream_t st);

// ------------------------------------------------------------------ norm_conv.cu (K6, K8)
// fp32 -> bf16 hi/lo operand planes (n multiple of 4)
void launch_split(const float *x, size_t n, ActBuf out, cudaStream_t st);
void launch_layernorm(const float *x, int M, int d, const float *w1, const float *b1, float *out1_f32,
                      ActBuf out1_act, const float *w2, const float *b2, ActBuf out2_act, cudaStream_t st);
bool launch_dwconv_bn_silu(const float *g, const int32_t *row_off, int n_utt, int max_T, int d, int ks,
                           const float *w, const float *bias, ActBuf out, cudaStream_t st);

// ------------------------------------------------------------------ attention.cu (K7)
// Both relative-position attention launchers take a band (att_left, att_right), both >= 0: query i attends to key j only
// when -att_right <= i - j <= att_left.  (0, 0) is full attention.  pp holds the relative positions -(tmax-1)..tmax-1; a
// band needs tmax >= max(att_left, att_right) + 1.  A negative band: false.
inline bool attention_band(int att_left, int att_right, int *left, int *right) {
    if (att_left < 0 || att_right < 0) return false;
    constexpr int kFull = 1 << 30;          // wider than any utterance, small enough that i0 + BQ + kFull stays an int
    const bool full = att_left == 0 && att_right == 0;
    *left = full ? kFull : std::min(att_left, kFull);
    *right = full ? kFull : std::min(att_right, kFull);
    return true;
}
bool launch_relpos_attention(const float *qkv, int ld_qkv, const int32_t *row_off, int n_utt, int max_T,
                             int n_heads, int head_dim, const float *pp, int tmax, int att_left, int att_right,
                             const float *bu, const float *bv, int d_model, ActBuf out, cudaStream_t st);

// tensor-core variant (attention_tc.cu, head_dim 64): pp as bf16 hi/lo planes
// From the EPI_QKV_ACT GEMM epilogue: q32 = fp32 q [M, d] (the kernel adds pos_u / pos_v), kv_hi / kv_lo = bf16 planes
// [M, ld_kv = 2 d] = [k | v].
bool launch_relpos_attention_tc(const float *q32, const float *pos_u, const float *pos_v, const bf16 *kv_hi, const bf16 *kv_lo,
                                int ld_kv, const int32_t *row_off, int n_utt, int max_T, int n_heads, int head_dim, const bf16 *pp_hi,
                                const bf16 *pp_lo, int tmax, int att_left, int att_right, int d_model, ActBuf out, cudaStream_t st);

// ------------------------------------------------------------------ attention_mha.cu / speaker_head.cu (Sortformer)
// Plain multi-head attention (transformer.cpp:15-50) over packed utterances, head_dim 24 only (false otherwise): qkv fp32
// [M][ld_qkv] = q | k | v, out ctx [M][d_model].
bool launch_mha_attention(const float *qkv, int ld_qkv, const int32_t *row_off, int n_utt, int max_T, int n_heads, int head_dim,
                          int d_model, ActBuf out, cudaStream_t st);
// Tensor-core form (bf16x3 with kv_lo, bf16x1 without): q32 fp32 [M][d_model], kv_hi / kv_lo = k | v bf16 planes [M][ld_kv] as
// the EPI_QKV_ACT epilogue writes them.  head_dim 24 only (false otherwise).
bool launch_mha_attention_tc(const float *q32, const bf16 *kv_hi, const bf16 *kv_lo, int ld_kv, const int32_t *row_off, int n_utt, int max_T,
                             int n_heads, int head_dim, int d_model, ActBuf out, cudaStream_t st);
// probs [M][S] = sigmoid(W2 . ReLU(W1 . ReLU(x) + b1) + b2) (sortformer.cpp:59-67); w1t = W1 transposed [D][D], w2 [S][D].
// D % 32 == 0, D <= 256, S <= 64 (false otherwise).
size_t speaker_head_smem(int D, int S);
bool launch_speaker_head(const float *x, int M, int D, int S, const float *w1t, const float *b1, const float *w2, const float *b2,
                         float *probs, int num_sms, cudaStream_t st);

// ContextTrie (src/phrase_boost.cpp:9-66) in CSR form on the device: node 0 = root; the edges of node i are
// [first[i], first[i+1]) = (token, child node), sorted by token.
// One trie per row (pk_set_boost_rows / pk_stream_set_boost): row b's arrays start b * node_stride (first) and
// b * edge_stride (tok, child) ints further, node ids are local to the row, and a row whose root has no edges
// (first[0] == first[1]) is not boosted.  Strides 0: one trie for every row (pk_set_boost).
struct DeviceTrie {
    const int32_t *first = nullptr, *tok = nullptr, *child = nullptr;
    int32_t n_nodes = 0;
    int32_t node_stride = 0, edge_stride = 0;
    // score added to the boosted label logits of row b: boost_rows[b], or `boost` for every row when boost_rows is null
    const float *boost_rows = nullptr;
    float boost = 0.f;
};
constexpr int BOOST_MAX_ACTIVE = 64;          // simultaneously active trie states per row
constexpr int BOOST_SLOT_NODES = 1024;        // capacity of one row's trie: nodes (root included) ...
constexpr int BOOST_SLOT_EDGES = BOOST_SLOT_NODES - 1;                           // ... and edges (a trie has nodes - 1)
constexpr int BOOST_SLOT_INTS = BOOST_SLOT_NODES + 1 + 2 * BOOST_SLOT_EDGES;     // slot = [first][tok][child]
#ifdef __CUDACC__
struct TrieRow {                              // the trie of one row
    const int32_t *first, *tok, *child;
    float boost;
    __device__ __forceinline__ bool empty() const { return first[0] == first[1]; }
};
__device__ __forceinline__ TrieRow trie_row(const DeviceTrie &t, int b) {
    return {t.first + (size_t)b * t.node_stride, t.tok + (size_t)b * t.edge_stride, t.child + (size_t)b * t.edge_stride,
            t.boost_rows ? t.boost_rows[b] : t.boost};
}
#endif
// Tries of fixed capacity on the device, one slot per row (utterance of a batch, or stream): slot = [first: NODES + 1]
// [tok: EDGES][child: EDGES] with slot-local node ids, plus a score per row.  The buffers never move, so captured graphs
// stay valid when the lists change.
struct BoostSlots {
    int32_t *slots = nullptr;                  // [rows][BOOST_SLOT_INTS]
    float *val = nullptr;                      // [rows]
    int rows = 0;
    DeviceTrie trie() const {
        DeviceTrie t;
        t.first = slots; t.tok = slots + BOOST_SLOT_NODES + 1; t.child = t.tok + BOOST_SLOT_EDGES;
        t.n_nodes = BOOST_SLOT_NODES; t.node_stride = t.edge_stride = BOOST_SLOT_INTS; t.boost_rows = val;
        return t;
    }
};
// The ContextTrie of phrases [p0, p1) (phrase p = phrase_ids[phrase_off[p] .. phrase_off[p+1])) in that CSR form, built on the
// host (engine.cu).  false: phrase_off decreases.
bool boost_trie_csr(const int32_t *phrase_ids, const int32_t *phrase_off, int32_t p0, int32_t p1, std::vector<int32_t> &first,
                    std::vector<int32_t> &tok, std::vector<int32_t> &child);
// Trie state of rows [row0, row0 + n) back to the root: active = {root}, bitmap = the root's children (ContextTrie's
// initial state, phrase_boost.cpp:9-51).  bits [rows][(V+31)/32], active [rows][64], nact [rows].
void launch_boost_state_reset(const DeviceTrie &trie, int V, int row0, int n, uint32_t *bits, int32_t *active, int32_t *nact, cudaStream_t st);

// ------------------------------------------------------------------ ctc.cu (K9)
// best / conf: the raw per-frame arg-max of launch_ctc_frame_argmax, decoded as is by the rows whose trie is empty
void launch_ctc_boosted_decode(const float *logprobs, const int32_t *best, const float *conf, const int32_t *row_off, int n_utt, int V, int blank, int cap,
                               const DeviceTrie &trie, int32_t *tok, int32_t *t_start, int32_t *t_end, float *t_conf,
                               cudaStream_t st);
void launch_ctc_frame_argmax(const float *logits, int M, int V, int ld, int32_t *best, float *conf,
                             float *logprobs, cudaStream_t st);
void launch_ctc_collapse(const int32_t *best, const float *conf, const int32_t *row_off, int n_utt, int blank,
                         int cap, int32_t *tok, int32_t *t_start, int32_t *t_end, float *t_conf, cudaStream_t st);

// ------------------------------------------------------------------ ctc_beam.cu (CTC prefix beam search, DESIGN.md section 14)
// Word n-gram LM in open-addressing tables (built on the host by lm.cpp): words by 64-bit FNV-1a hash of their bytes,
// n-grams by (context entry + 1) << 32 | word id.  Entry 0 is the empty context; an entry's suffix is its longest present
// proper suffix.  Empty slots hold key 0.  word_key == nullptr: no LM.
struct DeviceLM {
    const unsigned long long *word_key = nullptr;
    const int32_t *word_id = nullptr;
    const unsigned long long *ng_key = nullptr;
    const int32_t *ng_val = nullptr;
    const double *prob = nullptr, *backoff = nullptr;   // log10
    const int32_t *suffix = nullptr, *order = nullptr;
    uint32_t word_mask = 0, ng_mask = 0;
    int32_t max_order = 0, start = 0, unk = 0, eos = 0;
    double alpha_ln10 = 0.0, beta = 0.0;
    void set_weights(float alpha, float beta_) {
        alpha_ln10 = (double)alpha * 2.302585092994045684;
        beta = (double)beta_;
    }
};
// Token pieces for word boundaries: the bytes of token v are bytes[off[v] .. off[v+1]) with a leading U+2581 removed;
// starts[v] = 1 when the piece began with it.
struct DevicePieces {
    const uint8_t *bytes = nullptr;
    const int32_t *off = nullptr;
    const uint8_t *starts = nullptr;
};
constexpr int CTC_BEAM_THREADS = 256;
// Per frame: the `width` best non-blank (id, log-prob) pairs, ties to the lower id, into topk_id / topk_lp [M][width]
// (id -1 = absent: fewer than `width` finite values), and lp[blank] into blank_lp [M].
void launch_ctc_frame_topk(const float *logprobs, int M, int V, int width, int32_t *topk_id, float *topk_lp, float *blank_lp,
                           cudaStream_t st);
// The device form of an LM (or none: lm == NULL) and of the vocabulary's pieces; the weights are set by
// DeviceLM::set_weights.  Every table goes through upload(host, bytes) -> device pointer (nullptr: out of memory).  Returns
// an error message, empty on success.
std::string ctc_beam_tables(const pk_lm *lm, const pk_vocab *vocab, int V, const std::function<void *(const void *, size_t)> &upload,
                            DeviceLM *lm_out, DevicePieces *pc_out);
// What the tables of ctc_beam_tables(lm, vocab, V) are made from: 0 without an LM, else a 64-bit identity of the LM
// object (each pk_lm_load gives a new one) and of the vocabulary's first V - 1 pieces.
uint64_t ctc_beam_tables_id(const pk_lm *lm, const pk_vocab *vocab, int V);
// One CTA per utterance: the beam search over its frames; back-pointers bp [M][width]; tokens in the greedy layout.
void launch_ctc_beam(const float *logprobs, const int32_t *topk_id, const float *topk_lp, const float *blank_lp,
                     const int32_t *row_off, int n_utt, int V, int width, int cap, const DeviceLM &lm, const DevicePieces &pieces,
                     int32_t *bp, int32_t *tok, int32_t *t_start, int32_t *t_end, float *t_conf, cudaStream_t st);

// ------------------------------------------------------------------ ctc_align.cu (CTC forced alignment, DESIGN.md section 15)
constexpr int CTC_ALIGN_THREADS = 256;
// Dynamic shared memory of the alignment kernel: double-buffered Viterbi and forward rows of 2 PK_ALIGN_MAX_TOKENS + 1
// states, and the targets.
size_t ctc_align_smem_bytes();
// One CTA per utterance b: the targets tgt[tgt_off[b] .. tgt_off[b+1]) (ids in 0..V-2, at most PK_ALIGN_MAX_TOKENS) aligned
// to the log-probs of rows [row_off[b], row_off[b+1]).  Back-pointers bp [rows][bp_stride] (bp_stride >= 2 L + 1 of every
// feasible row); the best path's label and exp(log-prob) of every frame into best / conf (blank everywhere in an
// infeasible row), the Viterbi score and the log-likelihood into score / loglik [n_utt] (-inf: infeasible), and, when path
// is not NULL, the path's state of every frame (-1: infeasible).
void launch_ctc_align(const float *logprobs, const int32_t *row_off, int n_utt, int V, const int32_t *tgt, const int32_t *tgt_off,
                      uint8_t *bp, int bp_stride, int32_t *best, float *conf, double *score, double *loglik, int32_t *path,
                      cudaStream_t st);

// ------------------------------------------------------------------ tdt.cu (K10)
struct TdtParams {
    int P, J, V, D, L, Bpad, n_utt, cap, max_steps, n_dur;
    int max_sym;                                      // RNN-T (n_dur == 0): max_symbols_per_step; unused by TDT
    int out_in_smem, wih_in_smem, smem_lstm_floats;   // filled by launch_tdt_decode
    int wstage_rows;                                  // rows of the shared-memory staging tile for weights that stay in L2 (0: none)
    int durations[8];
    const float *EP;                          // [M][J] enc_proj(enc) + bias
    const int32_t *row_off;                   // [n_utt+1]
    const float *G0;                          // [V][4P] W_ih0 . E[token] + b0
    // weights pre-split for the tensor-core products (launch_tdt_split_rows): row = [hi: K][lo: K] bf16
    const bf16 *Whh[PK_MAX_LSTM];             // [P*4] rows, K = P, unit-major: row = unit*4 + gate(i,f,g,o)
    const bf16 *Wih[PK_MAX_LSTM];             // [P*4] rows, K = P, unit-major (layers >= 1)
    const float *bih[PK_MAX_LSTM];            // [4P]    (layers >= 1)
    const bf16 *Wp;                           // [J] rows, K = P
    const bf16 *Wout;                         // [V+D] rows, K = J
    const float *bout;                        // [V+D]
    float *hbuf;                              // bf16 [hi|lo][L][2][Bpad][P] LSTM h (two state planes per utterance), zeroed
    float *z;                                 // bf16 [hi|lo][Bpad][J]       joint hidden
    int32_t *overflow;                        // [Bpad]
    float *pl_max, *pl_sum;                   // [3][grid][Bpad] per-CTA (max, sum-exp) partials
    unsigned long long *key_lab, *key_dur;    // [3][Bpad] packed (value, index) arg-max keys
    unsigned int *bar;                        // grid barrier counter
    long long *dbg;                           // [8] optional: CTA-0 cycles per phase, steps
    int32_t *tok;                             // [n_utt][1+cap]
    int32_t *t_start, *t_end;                 // [n_utt][cap]
    float *t_conf;
    // Carried decode state (rnnt_streaming_decode_chunk, src/eou.cpp:17-98): the LSTM state, the last token and the
    // absolute frame number survive from chunk to chunk.  carry = 1: hbuf plane 0 holds the committed h on entry and on
    // exit, c_state [L][Bpad][P] the committed cell state, tok_state [Bpad] the last emitted token; emitted frames are
    // frame_base[b] + t and the end frame is NOT clamped to the chunk (eou.cpp:81-84); utterances with no frames idle.
    int carry;
    float *c_state;
    int32_t *tok_state;
    const int32_t *frame_base;
    // Phrase boosting (tdt_greedy_decode(_with_timestamps)_boosted, src/phrase_boost.cpp:177-352): boost_on = 1 adds the row's
    // score to the label logits of the tokens that continue an active state of the row's trie (durations are not boosted);
    // boost_bits [Bpad][(V+31)/32] is the per-utterance bitmap of those tokens, trie_active [Bpad][64] / trie_nact [Bpad] the
    // active states; all three are maintained by the CTA that owns the utterance.  Confidence stays exp(raw log-prob).
    // A row with an empty trie decodes exactly as with boost_on = 0.  carry = 0: the launch starts every row at the root;
    // carry = 1: the three arrays are stream state like c_state (read on entry, left for the next chunk; rows without
    // frames keep theirs) and whoever resets a stream resets them (launch_boost_state_reset).
    int boost_on;
    DeviceTrie trie;
    uint32_t *boost_bits;
    int32_t *trie_active, *trie_nact;
};
// Geometry controls of one decode launch (kernel tests only) and the geometry the launch chose.
struct TdtLaunchCtl {
    int cluster = 0;          // in: 0 = the engine's choice, 2 / 4 = only that cluster size (no fallback)
    bool no_stage = false;    // in: no staging tile: weights that do not fit are read from L2
    int grid = 0, CL = 0, UPC = 0, OPC = 0;                    // out (grid = 0: nothing was launched)
    int out_in_smem = 0, wih_in_smem = 0, staged_ih = 0, wstage_rows = 0;   // out; staged_ih as decided by cluster 0
};
// ctl = nullptr: the engine's choice, decided per launch from the shapes and the occupancy query.
cudaError_t launch_tdt_decode(TdtParams p, int num_sms, cudaStream_t st, TdtLaunchCtl *ctl = nullptr);
// gate-major LSTM weight [4P][P] (gate order i, f, g, o) -> unit-major [4P][P] (row = unit*4 + gate), the row order
// tdt_decode_kernel expects
void lstm_unit_major(const float *src, int P, float *dst);
void tdt_pass_profile(long long *out8, bool reset);   // measurement aid: section cycles of cluster_pass (CTA 0), summed since the last reset
// fp32 [rows][K] -> [rows][2 K] bf16 = [hi: K][lo: K]
void launch_tdt_split_rows(const float *src, int rows, int K, bf16 *dst, cudaStream_t st);

}  // namespace pk
