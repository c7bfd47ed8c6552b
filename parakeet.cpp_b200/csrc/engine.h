// engine.h -- the engine object behind the C-ABI (include/parakeet_b200.h), shared by engine.cu (offline path,
// jobs) and stream_engine.cu (streaming eou path).  See engine.cu for the reference call stack being replaced.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/parakeet_b200.h"
#include "kernels.h"
#include "nccl_dl.h"
#include "safetensors.h"

using namespace pk;


namespace pk_detail {

std::string &create_err();   // last error of a failed pk_engine_create / engine-less call (thread-local, engine.cu)

#define PK_CUDA(expr)                                                                         \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            return fail(PK_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));     \
        }                                                                                     \
    } while (0)

inline int conv_len(int L) { return (L - 1) / 2 + 1; }  // k3 s2 p1 (operations.cpp:3191-3196)
inline int enc_frames(int mel_frames) { return conv_len(conv_len(conv_len(mel_frames))); }   // the three stride-2 convs

// A linear layer's parameters on the device: fp32 master [N][K] + bias, and (wgmma
// modes) the bf16 hi/lo split planes of the weight.
struct GemmWeight {
    float *w = nullptr;
    bf16 *hi = nullptr, *lo = nullptr;
    float *bias = nullptr;
    int N = 0, K = 0;
    TcOperand tc;   // TMA tensor maps of hi/lo (wgmma modes)
};

// An activation buffer that feeds GEMMs, with its TMA tensor maps (wgmma modes).
struct Act : ActBuf {
    TcOperand tc;
    TcOperand tc32, tc64;   // the same planes with a 32- / 64-row box (A tiles fetched in slices and TMA-multicast across a 4- / 2-CTA cluster)
};

struct LayerW {
    float *ffn_ln_w[2], *ffn_ln_b[2];
    GemmWeight fc1[2], fc2[2];
    float *att_ln_w, *att_ln_b;
    GemmWeight qkv, out;
    float *pos_u, *pos_v;
    float *pp;  // [(2*pos_tmax-1)][d] projected relative-position table
    bf16 *pp_hi = nullptr, *pp_lo = nullptr;   // its bf16 split planes (tensor-core attention)
    float *conv_ln_w, *conv_ln_b;
    GemmWeight pw1, pw2;
    float *dw_w, *dw_b;  // BatchNorm folded; [d][k]
    float *dw_wt;        // the same weights tap-major [k][d] (offline kernel: one float4 per tap and 4 channels)
    float *fin_ln_w, *fin_ln_b;
};

// One post-norm block of Sortformer's transformer_ (transformer.cpp:15-62).
struct TLayerW {
    GemmWeight qkv, out, fc1, fc2;   // q/k/v fused [3 d][d]
    float *n1_w, *n1_b, *n2_w, *n2_b;
};

static_assert(BOOST_SLOT_NODES == PK_BOOST_ROW_NODES, "the slot capacity is part of the C-ABI");

}  // namespace pk_detail
using namespace pk_detail;

// The open streams of an engine (stream_engine.cu): ASR streams (pk_stream_open) or Sortformer streams (pk_diar_stream_open).
struct StreamSet {
    int S = 0, L = 70, R = 1, max_chunk = 0;
    int nf_max = 0, take_max = 0, c_max = 0;
    // host bookkeeping
    std::vector<int32_t> ovl_len, left, cache_len, ring_start, frame_base;
    std::vector<int32_t> act, take, nC;                       // this step: active stream ids, frames taken, encoder frames
    // device state
    StreamState st{};
    float *kc = nullptr, *vc = nullptr;                        // [layers][S][L][d]
    float *convc = nullptr;                                    // [layers][S][k-1][d]
    float *c_state = nullptr;                                  // [lstm][Bpad][P]
    float *hbuf = nullptr;                                     // bf16 planes [hi|lo][lstm][2][Bpad][P]
    int32_t *tok_state = nullptr;
    // Phrase boosting per stream (pk_stream_set_boost): a trie slot and score per stream, and the trie state of the decode
    // kernel, carried from chunk to chunk like the LSTM state.
    BoostSlots boost;
    uint32_t *boost_bits = nullptr;                            // [Bpad][(V+31)/32]
    int32_t *trie_active = nullptr, *trie_nact = nullptr;      // [Bpad][64], [Bpad]
    std::vector<uint8_t> boosted;                              // stream has a list
    int n_boosted = 0;
    // per-step device scratch
    float *d_chunk = nullptr, *ssig = nullptr, *mel_in = nullptr;
    StreamPlan *d_plan = nullptr, *h_plan = nullptr;           // h_plan pinned
    int64_t *d_sig_off = nullptr, *h_sig_off = nullptr;
    int32_t *d_meta = nullptr, *h_meta = nullptr;              // the step's metadata (Meta), h_meta pinned
    float *h_chunk = nullptr;                                  // pinned staging of the chunk samples
    cudaEvent_t ev_up = nullptr;                               // uploads of the previous step consumed
    size_t state_bytes = 0;
    // Sortformer streams (pk_diar_stream_open): no sample overlap, LSTM or token state; d_chunk / d_sig_off hold the packed
    // PCM and its offsets.
    bool diar = false;
    float *mel_new = nullptr, *h_mel = nullptr;                // this step's log-mel frames [S * nf_max][mel] (h_mel pinned)
    std::vector<uint64_t> spk_seen;                            // AOSCCache::speaker_active_ (max_speakers <= 64)
    std::vector<std::vector<int32_t>> arrival;                 // AOSCCache::arrival_order_

    StreamSet() = default;
    StreamSet(const StreamSet &) = delete;
    StreamSet &operator=(const StreamSet &) = delete;
    ~StreamSet() {                                             // the device buffers belong to the engine (pk_engine::allocs)
        if (h_plan) cudaFreeHost(h_plan);
        if (h_sig_off) cudaFreeHost(h_sig_off);
        if (h_meta) cudaFreeHost(h_meta);
        if (h_chunk) cudaFreeHost(h_chunk);
        if (h_mel) cudaFreeHost(h_mel);
        if (ev_up) cudaEventDestroy(ev_up);
    }

    // The segments of h_meta / d_meta, S ints each and row_off S + 1: nf | out_row | act | cache_len | ring_start |
    // frame_base | row_off, meta_ints() uploaded per step.  Sortformer streams keep the mel frame offsets of the step's
    // chunks (S + 1 ints, mel_off) in place of nf | out_row.
    enum Meta : int { NF, OUT_ROW, ACT, CACHE_LEN, RING_START, FRAME_BASE, ROW_OFF, MEL_OFF = NF };
    int32_t *meta_h(Meta k) const { return h_meta + (size_t)k * S; }
    int32_t *meta_d(Meta k) const { return d_meta + (size_t)k * S; }
    size_t meta_ints() const { return (size_t)ROW_OFF * S + S + 1; }

    // After a step that gave stream i the encoder rows [row_off[i], row_off[i+1]): its K / V rings hold the last L rows,
    // cache_len of them from ring_start on (streaming_encoder.cpp:185-208), which the cached attention reads next step.
    void advance(const int32_t *row_off) {
        for (int i = 0; i < S; ++i) {
            const int C = row_off[i + 1] - row_off[i], kv = cache_len[i] + C;
            if (kv > L) ring_start[i] = (ring_start[i] + kv - L) % L;
            cache_len[i] = std::min(kv, L);
            frame_base[i] += C;
        }
    }
    // CUDA-graph key of a step: every kernel argument depends only on which streams take how many frames.  The tag keeps
    // the caches of different step kinds apart.
    std::string graph_key(char tag) const {
        std::string key(1, tag);
        key.append(reinterpret_cast<const char *>(act.data()), act.size() * sizeof(int32_t));
        key.append(reinterpret_cast<const char *>(take.data()), take.size() * sizeof(int32_t));
        return key;
    }
};

struct pk_engine {
    pk_config cfg;
    // ---- diarization mode (pk_sortformer_create): the NEST encoder is cfg's encoder under keys "nest_encoder_.", its
    // subsampling output scaled by sqrt(d) (xscaling, folded into proj_), features not normalised; no decoder.
    bool diar = false;
    pk_sortformer_config sf{};
    std::string enc_prefix = "encoder_.";
    GemmWeight t_proj;                         // projection_ [t_hidden][d]
    std::vector<TLayerW> tlayers;
    float *head_w1t = nullptr, *head_b1 = nullptr, *head_w2 = nullptr, *head_b2 = nullptr;   // first_hidden_ (transposed), output_proj_
    float *t_x = nullptr, *t_qkv = nullptr, *probs = nullptr;   // [Mx][t_hidden] residual stream, [Mx][3 t_hidden], [Mx][S]
    Act t_ln, t_ctx, t_ff;                     // GEMM operands: LayerNorm output, attention context, ReLU(fc1)
    bf16 *t_kv_hi = nullptr, *t_kv_lo = nullptr;   // [Mx][2 t_hidden] k | v planes of the tensor-core attention (q in t_qkv)
    bool probs_valid = false;                  // probs hold the run of the staged batch
    float *h_probs = nullptr;                  // pinned [Mx][S]
    pk_status run_diar_head();                 // projection_ .. sigmoid on the encoder output in x
    int device = 0;
    int num_sms = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_h2d = nullptr;              // recorded after the staging copies of a batch
    // Host PCM arrives in H2D_CHUNKS utterance groups on `copy_stream`; the front end (mel, conv1+dw1)
    // of group i runs on `stream` as soon as its samples have landed, i.e. under the DMA of group i+1.
    static constexpr int H2D_CHUNKS = 8;
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_chunk[H2D_CHUNKS] = {}, ev_front = nullptr;
    bool front_done = false;                   // front end of the staged batch already launched (chunked path)
    std::string err;
    int64_t launches = 0;
    std::vector<void *> allocs;
    void *l2_scratch = nullptr;
    size_t l2_scratch_bytes = 0;
    int64_t l2_flushes = 0;

    // ---- capacity
    int Bmax = 0, Fmax = 0, Tmax = 0;          // per-utterance max mel frames / encoder frames
    int pos_tmax = 0;                          // position tables cover -(pos_tmax-1)..pos_tmax-1: Tmax, or W + 1 for a band
                                               // (cfg.local_att_left / _right, W = the larger of the two)
    int f1n = 0, f2n = 0, f3n = 0;
    int cap = 0;                               // token capacity per utterance

    // ---- weights
    MelTables mel_tb{};
    float *c1_w, *c1_b, *dw1_w, *dw1_b, *dw2_w, *dw2_b;
    float *dw2_wt = nullptr;                   // dw2_ weights tap-major [9][C]: one float4 per tap and 4 channels
    GemmWeight conv2, conv3, proj;
    std::vector<LayerW> layers;
    GemmWeight ctc_head;
    GemmWeight enc_proj;                       // joint enc_proj_ [J][d] + bias
    float *G0 = nullptr;                       // [V][4P]
    float *Whh[PK_MAX_LSTM] = {}, *Wih[PK_MAX_LSTM] = {}, *bih[PK_MAX_LSTM] = {};
    float *Whh_um[PK_MAX_LSTM] = {}, *Wih_um[PK_MAX_LSTM] = {};   // unit-major copies (decode kernel)
    float *Wp = nullptr, *Wout = nullptr, *bout = nullptr;
    bf16 *Whh_s[PK_MAX_LSTM] = {}, *Wih_s[PK_MAX_LSTM] = {}, *Wp_s = nullptr, *Wout_s = nullptr;   // pre-split rows (tdt.cu)

    // ---- workspace
    float *d_pcm = nullptr;
    float *d_pcm_alt = nullptr;               // second PCM buffer (pk_prefetch_pcm); swapped with d_pcm on adoption
    cudaEvent_t ev_pcm_free[2] = {}, ev_prefetch = nullptr;   // [k]: last front end reading buffer k has run; prefetch copy done
    int pcm_cur = 0;                           // which physical buffer d_pcm currently is
    cudaEvent_t ev_join = nullptr;             // pk_run_transcribe_diarize_staged: recorded here for the other engine of the pair to wait on
    struct { const float *pcm = nullptr; int32_t n = 0; std::vector<int64_t> off; bool valid = false; } pref;
    int64_t *d_pcm_off = nullptr;
    int32_t *d_frame_off = nullptr, *d_s2_off = nullptr, *d_row_off = nullptr, *d_t2_rows = nullptr;
    float *logmel = nullptr, *feats = nullptr;
    float *mel_part = nullptr;                 // per-chunk statistics of the mel normalisation (mel.cu K2), one slice per utterance
    Act sub1, sub3, sub4, ln, ffh, ctx, cv;
    float *sub2 = nullptr, *x = nullptr, *qkv = nullptr, *glu = nullptr, *logits = nullptr, *EP = nullptr;
    bf16 *qkvp_hi = nullptr, *qkvp_lo = nullptr;   // [Mx, 2 d] planes [k | v] for the tensor-core attention (q stays fp32 in `qkv`)
    int32_t *best = nullptr;
    float *bconf = nullptr;
    int32_t *tok = nullptr, *t_start = nullptr, *t_end = nullptr;
    float *t_conf = nullptr;
    // TDT state
    int Bpad = 0;
    float *hbuf = nullptr, *cbuf = nullptr, *zbuf = nullptr, *pl_max = nullptr, *pl_sum = nullptr;
    int32_t *tdt_ints = nullptr;               // overflow[Bpad] | barrier counter
    unsigned long long *tdt_keys = nullptr;    // arg-max keys: label[3][Bpad] | duration[3][Bpad]
    // pinned host staging
    float *h_pcm = nullptr;
    int32_t *h_meta = nullptr;                 // offsets staging
    int32_t *h_tok = nullptr, *h_ts = nullptr, *h_te = nullptr;
    float *h_tc = nullptr;

    // ---- CUDA graphs of the staged pipeline, keyed by (decoder, utterance lengths)
    struct GraphEntry { cudaGraphExec_t exec = nullptr; int64_t launches = 0; int seen = 0; };
    std::map<std::string, GraphEntry> graphs;
    bool use_graphs = true;
    bool attn_tc = true;                       // mma.sync attention for head_dim 64 / 128 (PK_ATTN_TC=0: fp32 kernel)

    // ---- the staged batch
    int n_utt = 0;
    std::vector<int64_t> pcm_off;
    std::vector<int32_t> frame_off, s2_off, row_off, t2_rows;
    int maxF = 0, maxT2 = 0, maxT = 0, M = 0, M2 = 0;

    // ---- a JOB: many micro-batches on this GPU, ONE exchange at the end (SURVEY.md section 8e, BASELINE configs[4])
    int32_t *job_tok = nullptr, *job_all = nullptr;   // [job_cap_rows][1 + cap] local rows; [job_world * job_cap_rows][1 + cap] gathered
    int64_t job_cap_rows = 0, job_rows = 0, job_alloc_rows = 0;   // rows per rank of this job / appended so far / allocated (x world)
    int job_world = 1;
    int32_t *h_job = nullptr;                          // pinned staging of the gathered rows
    size_t h_job_ints = 0;
    float *job_pcm = nullptr;                          // device-resident PCM of a whole job (pk_job_stage_pcm)
    size_t job_pcm_cap = 0;
    std::vector<int64_t> job_off;
    const float *pcm_src = nullptr;                    // front end reads this instead of d_pcm (a slice of job_pcm)
    float *d_raw = nullptr;                            // input at its own sample rate (pk_stage_pcm_rate / pk_resample_batch)
    size_t d_raw_cap = 0;
    int64_t *d_raw_off = nullptr;                      // [Bmax + 1] offsets of the raw utterances
    void *nccl_comm = nullptr;                         // ncclComm_t (pk_comm_init_rank) -- owned
    int nccl_rank = 0, nccl_world = 1;
    bool last_tdt = false;                             // the token buffer holds a TDT decode (overflow flags are valid)
    int32_t truncated = 0;                             // utterances of the last fetch whose TDT hypothesis hit the token capacity

    // ---- phrase boosting: ContextTrie on the device + per-utterance trie state of the TDT kernel
    DeviceTrie trie{};                                 // pk_set_boost: one trie and score for every utterance
    bool boost_on = false;
    int boost_gen = 0;                                 // bumps on every pk_set_boost (part of the CUDA-graph key)
    uint32_t *boost_bits = nullptr;                    // [Bpad][(V+31)/32]
    int32_t *trie_active = nullptr, *trie_nact = nullptr;
    BoostSlots brows;                                  // pk_set_boost_rows: a trie and score per utterance of the batch
    bool brows_on = false;                             // some row of brows has a list (replaces, and is replaced by, boost_on)
    int brows_hi = 0;                                  // rows [0, brows_hi) of brows may hold a list on the device
    // List uploads go through two pinned buffers used in turn ([rows][BOOST_SLOT_INTS] ints, then [rows] scores), so an
    // upload never waits for the stream unless two earlier ones are still queued.
    int32_t *h_bstage[2] = {};
    cudaEvent_t ev_bstage[2] = {};
    int bstage_rows = 0, bstage_next = 0;
    pk_status boost_state_alloc();                     // boost_bits / trie_active / trie_nact
    // Rows [row0, row0 + n) of `dst` <- the tries of lists i = phrases [row_off[i], row_off[i+1]) with scores boost[i]; the
    // n_clear rows after them <- empty.  Stream-ordered, no synchronisation.  Nothing is uploaded when a list is invalid
    // or over the slot capacity (PK_ERR_CAPACITY naming the row).  *any: some list has an edge.
    pk_status boost_upload(const char *fn, BoostSlots &dst, int row0, int n, int n_clear, const int32_t *phrase_ids,
                           const int32_t *phrase_off, const int32_t *row_off, const float *boost, bool *any);
    bool boosting() const { return boost_on || brows_on; }
    DeviceTrie boost_trie() const { return brows_on ? brows.trie() : trie; }

    // ---- CTC beam search (pk_set_ctc_beam)
    int beam_w = 0;                                    // 0: not set
    int beam_gen = 0;                                  // bumps when the device tables are replaced (part of the CUDA-graph key)
    uint64_t beam_tab_id = 0;                          // ctc_beam_tables_id of the tables on the device (0: no LM)
    std::vector<void *> beam_tab;                      // their device buffers, freed when they are replaced
    DeviceLM beam_lm{};
    DevicePieces beam_pc{};
    // [Bmax Tmax][PK_CTC_BEAM_MAX] top-W ids / log-probs and back-pointers, [Bmax Tmax] blank log-probs (allocated once)
    int32_t *beam_topk_id = nullptr, *beam_bp = nullptr;
    float *beam_topk_lp = nullptr, *beam_blank = nullptr;

    // ---- CTC forced alignment (pk_set_align_targets), buffers allocated by its first call and never moved
    int align_rows = 0;                                // rows of the targets in place (0: none)
    int32_t *align_ids = nullptr, *align_off = nullptr;   // [Bmax][PK_ALIGN_MAX_TOKENS] packed ids, [Bmax + 1] offsets
    uint8_t *align_bp = nullptr;                       // [Bmax Tmax][align_stride] back-pointers
    int align_stride = 0;                              // 2 min(Tmax, PK_ALIGN_MAX_TOKENS) + 1
    double *align_score = nullptr, *align_loglik = nullptr;   // [Bmax] each
    bool align_last = false;                           // the token buffer holds an alignment (pk_fetch_align_scores)

    // ---- optional per-kernel-class timing (CUDA events on the engine stream)
    enum { CAT_MEL, CAT_SUBSAMPLE, CAT_GEMM, CAT_LAYERNORM, CAT_ATTENTION, CAT_DWCONV, CAT_CTC, CAT_TDT, CAT_MHA, CAT_HEAD, CAT_N };
    struct ProfRec { int cat; cudaEvent_t a, b; double flops; };
    bool prof_on = false;
    std::vector<ProfRec> prof;
    std::vector<cudaEvent_t> ev_pool;
    cudaEvent_t prof_event() {
        if (!ev_pool.empty()) { cudaEvent_t e = ev_pool.back(); ev_pool.pop_back(); return e; }
        cudaEvent_t e; cudaEventCreate(&e); return e;
    }
    struct Scope {
        pk_engine *e; int idx = -1;
        Scope(pk_engine *e_, int cat, double flops = 0.0) : e(e_) {
            if (!e->prof_on) return;
            ProfRec r{cat, e->prof_event(), e->prof_event(), flops};
            cudaEventRecord(r.a, e->stream);
            idx = (int)e->prof.size();
            e->prof.push_back(r);
        }
        ~Scope() { if (idx >= 0) cudaEventRecord(e->prof[idx].b, e->stream); }
    };

    pk_status fail(pk_status s, const std::string &m) {
        err = m;
        return s;
    }
    template <typename T>
    T *dalloc(size_t n) {
        void *p = nullptr;
        if (cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return nullptr;
        allocs.push_back(p);
        return static_cast<T *>(p);
    }
    template <typename T>
    T *upload(const std::vector<T> &h) {
        T *d = dalloc<T>(h.size());
        // On the engine's own (non-blocking) stream, then wait: a legacy-stream cudaMemcpy from
        // pageable memory may still be in flight when a kernel on `stream` starts.
        if (d && !h.empty()) {
            cudaMemcpyAsync(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, stream);
            cudaStreamSynchronize(stream);
        }
        return d;
    }
    // [rows][K] activation that feeds a GEMM as the A operand
    Act act_alloc(size_t rows, size_t K) {
        Act a;
        const size_t n = rows * K;
        if (cfg.math == PK_MATH_FP32) {
            a.f32 = dalloc<float>(n);
        } else {
            a.hi = dalloc<bf16>(n);
            if (cfg.math == PK_MATH_BF16X3) a.lo = dalloc<bf16>(n);
            if (a.hi && (!make_tc_operand(&a.tc, a.hi, a.lo, rows, K, 128) || !make_tc_operand(&a.tc32, a.hi, a.lo, rows, K, 32) || !make_tc_operand(&a.tc64, a.hi, a.lo, rows, K, 64))) a.hi = nullptr;   // reported by the caller
        }
        return a;
    }

    pk_status load(const char *path);
    pk_status make_weight(const SafeTensors &st, const std::string &wname, const std::string &bname, int N, int K,
                          GemmWeight &out, const std::vector<int> *row_perm = nullptr,
                          const std::vector<int> *col_perm = nullptr, float scale = 1.0f);
    pk_status finish_weight(std::vector<float> &w, std::vector<float> *b, int N, int K, GemmWeight &out);
    pk_status get_vec(const SafeTensors &st, const std::string &name, int n, float **out);
    pk_status alloc_workspace();
    pk_status band_rows_ok();
    pk_status set_batch_shapes(const int32_t *n_frames_or_null, const int64_t *offsets_or_null, int n);
    pk_status upload_shapes();
    void gemm(const Act &A, int lda, const GemmWeight &W, int M_, EpiParams epi);
    // LayerNorm of the M rows of `in` [M][width] (layernorm_kernel) into out1 / act1; with w2, a second LayerNorm of that
    // result into act2.
    void layernorm(const float *in, int width, const float *w1, const float *b1, float *out1, ActBuf act1, const float *w2 = nullptr,
                   const float *b2 = nullptr, ActBuf act2 = {});
    int gemm_cluster = 0;                      // PK_GEMM_CLUSTER=2|4: wide GEMMs (fc1, q/k/v, pw1) run as clusters of 2 | 4 CTAs along N with the A tile multicast
    // few-row GEMMs (M <= 128: streaming steps, short utterances) go to gemm_skinny.cu (offline diarization keeps it off)
    bool skinny = true;
    float *skinny_ws = nullptr;
    size_t skinny_ws_floats = 0;
    unsigned int *skinny_tickets = nullptr;
    static constexpr int SKINNY_TICKETS = 1024;
    pk_status gemm_err = PK_OK;
    pk_status run_mel(int u0 = 0, int u1 = -1);
    pk_status run_conv1(int u0 = 0, int u1 = -1);
    pk_status run_graphed(const std::string &key, const std::function<pk_status()> &body);
    pk_status run_subsample_tail();
    pk_status run_encoder(float *sub_out_host, float *layers_out_host);
    // The Conformer blocks on the rows in x; cached: a step of the open streams (attention over their K / V rings, causal
    // conv over their conv caches).  layers_out_host (offline only, may be null) receives x after every block.
    pk_status run_blocks(bool cached, float *layers_out_host);
    // streaming eou path (stream_engine.cu); on a Sortformer engine the streams of pk_diar_stream_open
    StreamSet *ss = nullptr;
    // dec: PK_DECODER_CTC, _CTC_BEAM or _CTC_ALIGN; logprobs_dev_or_null: where the log-probs land (null: where the decoder needs them)
    pk_status run_ctc(pk_decoder dec, float *logprobs_dev_or_null);
    pk_status run_tdt();
    pk_status tdt_decode(TdtParams &p);               // enc_proj and the decode kernel; p holds what the caller's decode sets
    pk_status run_decoder(pk_decoder dec) {           // (dec already checked)
        const bool ctc = dec == PK_DECODER_CTC || dec == PK_DECODER_CTC_BEAM || dec == PK_DECODER_CTC_ALIGN;
        return ctc ? run_ctc(dec, nullptr) : run_tdt();
    }
    pk_status fetch(pk_tokens *out);
};

void pk_stream_free(pk_engine *e);   // stream_engine.cu
