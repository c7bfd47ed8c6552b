// stream_engine.cu -- the STREAMING path behind the C-ABI (SURVEY.md section 8f row 2, BASELINE configs[3]: eou-120m,
// 160 ms chunks).  Reference call stack being replaced (one stream, one chunk at a time, host round trips throughout):
//   StreamingTranscriber::transcribe_chunk                 src/eou.cpp:111-143
//   StreamingAudioPreprocessor::process_chunk              src/audio.cpp:195-259
//   StreamingFastConformerEncoder::forward_chunk           src/streaming_encoder.cpp:425-472
//     CausalConvSubsampling::forward_cached                :339-385
//     StreamingConformerAttention::forward_cached          :160-272
//     CausalConformerConvModule::forward_cached            :41-80
//   rnnt_streaming_decode_chunk                            src/eou.cpp:17-98
//
// Design: the reference advances ONE stream by 1-2 encoder frames per call, which is weight-bandwidth-bound (435 MB of
// fp32 weights per chunk).  Here S streams advance in LOCK STEP: a step takes one chunk of every stream, and all
// streams' frames form one packed row block M = sum_s C_s that runs through the same wgmma GEMMs / LayerNorm kernels as
// the offline path (weights are read once per step for all streams).  Per-stream state is resident in HBM: sample
// overlap + pre-emphasis carry, leftover mel frames, per layer a ring of the last att_context_left K / V rows and the
// last k-1 GLU outputs, the LSTM state, the last token and the absolute frame offset.  All lengths depend only on the
// chunk sizes, so the host computes them (StreamPlan) and the kernels never synchronise with it.  Sortformer streams
// (pk_diar_stream_*) share the open, reset and step below.
#include "engine.h"

namespace {

using Meta = StreamSet::Meta;

// The open of either kind once the kind's own checks passed (s: kind, S, L, R, max_chunk and nf_max set): the capacity
// checks and the state both kinds carry.  `what` names the state in the allocation-failure messages.
pk_status stream_alloc(pk_engine *e, const char *fn, const char *what, StreamSet &s) {
    if (e->ss) return e->fail(PK_ERR_INVALID, std::string(fn) + ": streams are already open on this engine");
    const pk_config &c = e->cfg;
    s.take_max = ((7 + s.nf_max) / 8) * 8;                   // + up to 7 leftover frames
    s.c_max = enc_frames(std::max(s.take_max, 8));
    if (s.S > e->Bmax) return e->fail(PK_ERR_CAPACITY, std::string(fn) + ": more streams than pk_config.max_batch");
    if (s.take_max > e->Fmax || s.L + s.c_max > e->Tmax)
        return e->fail(PK_ERR_CAPACITY, std::string(fn) + ": pk_config.max_samples too small (needs encoder frames >= att_context_left + frames per chunk)");
    const int S = s.S, d = c.d_model, nl = c.n_layers;
    s.ovl_len.assign(S, 0); s.left.assign(S, 0); s.cache_len.assign(S, 0); s.ring_start.assign(S, 0); s.frame_base.assign(S, 0);
    s.st.melq = e->dalloc<float>((size_t)S * 8 * c.mel_bins);
    s.kc = e->dalloc<float>((size_t)nl * S * s.L * d);
    s.vc = e->dalloc<float>((size_t)nl * S * s.L * d);
    s.convc = e->dalloc<float>((size_t)nl * S * (c.conv_kernel - 1) * d);
    s.d_chunk = e->dalloc<float>((size_t)S * s.max_chunk + 8);
    s.d_plan = e->dalloc<StreamPlan>(S);
    s.d_sig_off = e->dalloc<int64_t>(S + 1);
    s.d_meta = e->dalloc<int32_t>(s.meta_ints() + 7);
    if (!s.st.melq || !s.kc || !s.vc || !s.convc || !s.d_chunk || !s.d_plan || !s.d_sig_off || !s.d_meta)
        return e->fail(PK_ERR_CUDA, std::string("cudaMalloc failed (") + what + " state)");
    if (cudaMallocHost(&s.h_plan, sizeof(StreamPlan) * S) != cudaSuccess || cudaMallocHost(&s.h_sig_off, sizeof(int64_t) * (S + 1)) != cudaSuccess ||
        cudaMallocHost(&s.h_meta, sizeof(int32_t) * (s.meta_ints() + 7)) != cudaSuccess ||
        cudaMallocHost(&s.h_chunk, sizeof(float) * ((size_t)S * s.max_chunk + 8)) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.ev_up, cudaEventDisableTiming) != cudaSuccess)
        return e->fail(PK_ERR_CUDA, std::string("cudaMallocHost failed (") + what + " staging)");
    return PK_OK;
}

// Installs the fully allocated streams and runs their first reset; on a failure nothing stays open.
pk_status stream_install(pk_engine *e, std::unique_ptr<StreamSet> s, pk_status (*reset)(pk_engine *, int32_t)) {
    e->ss = s.release();
    const pk_status ps = reset(e, -1);
    if (ps) pk_stream_free(e);
    return ps;
}

// The reset of either kind for one stream (or all: stream = -1): the host bookkeeping, and the conv caches back to zeros
// (streaming_encoder.cpp:52-56); K / V rings and mel queues are empty (lengths 0).  extra(s0, s1) resets the kind's own
// state of streams [s0, s1).
template <class Extra>
pk_status stream_reset(pk_engine *e, const char *fn, int32_t stream, Extra extra) {
    StreamSet &s = *e->ss;
    const pk_config &c = e->cfg;
    if (stream < -1 || stream >= s.S) return e->fail(PK_ERR_INVALID, std::string(fn) + ": bad stream index");
    const int s0 = stream < 0 ? 0 : stream, s1 = stream < 0 ? s.S : stream + 1;
    cudaEventSynchronize(s.ev_up);
    cudaError_t ce = cudaSuccess;
    for (int i = s0; i < s1 && ce == cudaSuccess; ++i) {
        s.ovl_len[i] = s.left[i] = s.cache_len[i] = s.ring_start[i] = s.frame_base[i] = 0;
        for (int l = 0; l < c.n_layers && ce == cudaSuccess; ++l)
            ce = cudaMemsetAsync(s.convc + ((size_t)l * s.S + i) * (c.conv_kernel - 1) * c.d_model, 0,
                                 sizeof(float) * (c.conv_kernel - 1) * c.d_model, e->stream);
    }
    if (ce == cudaSuccess) ce = extra(s0, s1);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(ce));
    return PK_OK;
}

// One step of either kind: every stream's input is checked before any state changes, then the plan (pure integer
// bookkeeping, audio.cpp:216-240, streaming_encoder.cpp:348-385, :185-208) is uploaded, the front end launched, the taps
// filled, the host state advanced and the encoder run on the active streams' rows (s.act, empty if none).  Per kind:
// chunk(i, p) checks and stages stream i's input and sets p.nf and p's front-end fields; upload(st) sends the staged
// input; front(max_nf) leaves every active stream's p.take frames at row p.feat_off of feats; head() runs on the
// encoder rows in the step's graph.
template <class Chunk, class Upload, class Front, class Head>
pk_status stream_step(pk_engine *e, const char *fn, char tag, int32_t *n_mel, int32_t *n_enc, int32_t *frame_base_out, float *enc_out,
                      Chunk chunk, Upload upload, Front front, Head head) {
    StreamSet &s = *e->ss;
    const int S = s.S;
    if (pk_status g = e->gemm_err) return g;
    cudaEventSynchronize(s.ev_up);                 // the previous step has consumed the pinned staging buffers
    int32_t *m_act = s.meta_h(Meta::ACT), *m_cl = s.meta_h(Meta::CACHE_LEN), *m_rs = s.meta_h(Meta::RING_START),
            *m_fb = s.meta_h(Meta::FRAME_BASE), *m_ro = s.meta_h(Meta::ROW_OFF);
    s.act.clear(); s.take.clear(); s.nC.clear();
    m_ro[0] = 0;
    int foff = 0, max_nf = 0;
    for (int i = 0; i < S; ++i) {
        StreamPlan &p = s.h_plan[i];
        memset(&p, 0, sizeof(p));
        p.left = s.left[i];
        if (pk_status ps = chunk(i, p)) return ps;
        p.take = ((p.left + p.nf) / 8) * 8;
        p.feat_off = foff;
        m_cl[i] = s.cache_len[i]; m_rs[i] = s.ring_start[i]; m_fb[i] = s.frame_base[i];
        int C = 0;
        if (p.take > 0) {
            C = enc_frames(p.take);
            s.act.push_back(i); s.take.push_back(p.take); s.nC.push_back(C);
            foff += p.take;
        }
        m_ro[i + 1] = m_ro[i] + C;
        max_nf = std::max(max_nf, p.nf);
    }
    const int n_act = (int)s.act.size();
    for (int a = 0; a < n_act; ++a) m_act[a] = s.act[a];
    cudaStream_t st = e->stream;
    cudaError_t ce = cudaMemcpyAsync(s.d_plan, s.h_plan, sizeof(StreamPlan) * S, cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(s.d_meta, s.h_meta, sizeof(int32_t) * s.meta_ints(), cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = upload(st);
    if (ce == cudaSuccess) ce = cudaEventRecord(s.ev_up, st);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string(fn) + " upload: " + cudaGetErrorString(ce));
    front(max_nf);
    // ---- taps, and the host state of the next step: the samples the new frames did not cover (none on Sortformer
    // streams, whose plans keep their sample fields zero) and the frames the encoder did not take
    for (int i = 0; i < S; ++i) {
        const StreamPlan &p = s.h_plan[i];
        if (n_mel) n_mel[i] = p.nf;
        if (n_enc) n_enc[i] = m_ro[i + 1] - m_ro[i];
        if (frame_base_out) frame_base_out[i] = s.frame_base[i];
        s.ovl_len[i] = p.ovl_len + p.chunk_len - p.consumed;
        s.left[i] = p.left + p.nf - p.take;
    }
    s.advance(m_ro);
    if (n_act == 0) return PK_OK;
    // ---- the active streams' frames as an ordinary packed batch (CausalConvSubsampling runs the plain zero-padded subsampling)
    pk_status ps;
    if ((ps = e->set_batch_shapes(s.take.data(), nullptr, n_act))) return ps;
    if ((ps = e->upload_shapes())) return ps;
    auto body = [&]() -> pk_status {
        const bool sk = e->skinny;
        e->skinny = true;                          // few rows per step: the weight-streaming GEMM
        pk_status q = e->run_conv1();
        if (!q) q = e->run_subsample_tail();
        if (!q) q = e->run_blocks(true, nullptr);
        if (!q && enc_out) {
            cudaError_t c2 = cudaMemcpyAsync(enc_out, e->x, sizeof(float) * (size_t)e->M * e->cfg.d_model, cudaMemcpyDeviceToHost, st);
            if (c2 != cudaSuccess) q = e->fail(PK_ERR_CUDA, std::string(fn) + " tap: " + cudaGetErrorString(c2));
        }
        if (!q) q = head();
        e->skinny = sk;
        return q;
    };
    // every kernel argument of the step depends only on which streams take how many frames (debug tap: plain launches)
    if ((ps = enc_out ? body() : e->run_graphed(s.graph_key(tag), body))) return ps;
    return e->gemm_err;
}

}  // namespace

extern "C" {

pk_status pk_stream_open(pk_engine *e, int32_t n_streams, int32_t max_chunk_samples, int32_t att_context_left, int32_t att_context_right) {
    if (!e || n_streams < 1 || max_chunk_samples < 1 || att_context_left < 1) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_stream_open: a Sortformer engine opens its streams with pk_diar_stream_open");
    const pk_config &c = e->cfg;
    if (c.n_durations == 0) return e->fail(PK_ERR_INVALID, "pk_stream_open: streaming decodes a TDT joint; this is an RNN-T model");
    // the cached attention reads position tables that cover the whole context (Tmax); a band engine keeps only -W..W
    if (c.local_att_left || c.local_att_right) return e->fail(PK_ERR_INVALID, "pk_stream_open: not on a limited-context (local_att_*) engine");
    auto s = std::make_unique<StreamSet>();
    s->S = n_streams; s->L = att_context_left; s->R = att_context_right; s->max_chunk = max_chunk_samples;
    const int tot_max = 399 + max_chunk_samples;
    s->nf_max = tot_max >= 512 ? ((((tot_max - 400) / 160) * 160 + 400) - 512) / 160 + 1 : 0;
    if (pk_status ps = stream_alloc(e, "pk_stream_open", "stream", *s)) return ps;
    const int S = n_streams, P = c.pred_hidden, LL = c.lstm_layers;
    s->st.ovl = e->dalloc<float>((size_t)S * STREAM_OVL_CAP);
    s->st.last = e->dalloc<float>(S);
    s->c_state = e->dalloc<float>((size_t)LL * e->Bpad * P);
    s->hbuf = e->dalloc<float>((size_t)P * e->Bpad * 2 * LL);
    s->tok_state = e->dalloc<int32_t>(e->Bpad);
    s->boost.slots = e->dalloc<int32_t>((size_t)S * BOOST_SLOT_INTS);
    s->boost.val = e->dalloc<float>(S);
    s->boost.rows = S;
    s->boost_bits = e->dalloc<uint32_t>((size_t)e->Bpad * ((c.vocab + 31) / 32));
    s->trie_active = e->dalloc<int32_t>((size_t)e->Bpad * BOOST_MAX_ACTIVE);
    s->trie_nact = e->dalloc<int32_t>(e->Bpad);
    s->boosted.assign(S, 0);
    s->ssig = e->dalloc<float>((size_t)S * (max_chunk_samples + STREAM_OVL_CAP) + 8);
    s->mel_in = e->dalloc<float>((size_t)S * (8 + s->nf_max) * c.mel_bins);
    if (!s->st.ovl || !s->st.last || !s->c_state || !s->hbuf || !s->tok_state || !s->boost.slots || !s->boost.val || !s->boost_bits ||
        !s->trie_active || !s->trie_nact || !s->ssig || !s->mel_in)
        return e->fail(PK_ERR_CUDA, "cudaMalloc failed (stream state)");
    // every slot empty (first[0] == first[1]): no stream is boosted until pk_stream_set_boost
    if (cudaMemsetAsync(s->boost.slots, 0, (size_t)S * BOOST_SLOT_INTS * sizeof(int32_t), e->stream) != cudaSuccess ||
        cudaMemsetAsync(s->boost_bits, 0, (size_t)e->Bpad * ((c.vocab + 31) / 32) * sizeof(uint32_t), e->stream) != cudaSuccess)
        return e->fail(PK_ERR_CUDA, "cudaMemset failed (stream boost state)");
    return stream_install(e, std::move(s), pk_stream_reset);
}

// StreamingTranscriber::reset (eou.cpp:145-149) for one stream (or all: stream = -1)
pk_status pk_stream_reset(pk_engine *e, int32_t stream) {
    if (!e || !e->ss) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_stream_reset: a Sortformer engine's streams reset with pk_diar_stream_reset");
    StreamSet &s = *e->ss;
    const pk_config &c = e->cfg;
    return stream_reset(e, "pk_stream_reset", stream, [&](int s0, int s1) {
        const int P = c.pred_hidden, Bp = e->Bpad, LL = c.lstm_layers;
        cudaError_t ce = cudaSuccess;
        for (int i = s0; i < s1 && ce == cudaSuccess; ++i) {
            ce = cudaMemsetAsync(s.st.last + i, 0, sizeof(float), e->stream);
            // LSTM state zero, last token = blank (eou.cpp:22-33)
            for (int l = 0; l < LL && ce == cudaSuccess; ++l) {
                ce = cudaMemsetAsync(s.c_state + ((size_t)l * Bp + i) * P, 0, sizeof(float) * P, e->stream);
                bf16 *hb = reinterpret_cast<bf16 *>(s.hbuf);
                const size_t HS = (size_t)P * Bp, lo = (size_t)LL * 2 * HS;
                for (int pl = 0; pl < 2 && ce == cudaSuccess; ++pl) {
                    ce = cudaMemsetAsync(hb + (size_t)(l * 2 + pl) * HS + (size_t)i * P, 0, sizeof(bf16) * P, e->stream);
                    if (ce == cudaSuccess) ce = cudaMemsetAsync(hb + lo + (size_t)(l * 2 + pl) * HS + (size_t)i * P, 0, sizeof(bf16) * P, e->stream);
                }
            }
        }
        // the phrase trie restarts at the root (the stream keeps its list)
        if (ce == cudaSuccess) {
            launch_boost_state_reset(s.boost.trie(), c.vocab, s0, s1 - s0, s.boost_bits, s.trie_active, s.trie_nact, e->stream);
            ce = cudaGetLastError();
        }
        if (ce == cudaSuccess) {
            const std::vector<int32_t> blank(s1 - s0, c.vocab - 1);
            ce = cudaMemcpyAsync(s.tok_state + s0, blank.data(), sizeof(int32_t) * (s1 - s0), cudaMemcpyHostToDevice, e->stream);
        }
        return ce;
    });
}

// One step = StreamingTranscriber::transcribe_chunk (eou.cpp:111-143) for every stream: stream s receives the samples
// pcm[offsets[s] .. offsets[s+1]) (an empty chunk is allowed).  out rows (n = n_streams) hold the tokens emitted BY THIS
// STEP with absolute frame numbers.  Optional taps (may be NULL): mel_out packed (sum nf_s, mel_bins) = the new log-mel frames
// of this step, n_mel[s] = nf_s; enc_out packed (sum C_s, d_model) = the encoder rows of this step, n_enc[s] = C_s.
pk_status pk_stream_step(pk_engine *e, const float *pcm, const int64_t *offsets, pk_tokens *out, float *mel_out, int32_t *n_mel,
                         float *enc_out, int32_t *n_enc) {
    if (!e || !e->ss || !offsets || (!pcm && offsets[e->ss->S] > offsets[0])) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_stream_step: a Sortformer engine's streams step with pk_diar_stream_step");
    StreamSet &s = *e->ss;
    const pk_config &c = e->cfg;
    const int S = s.S;
    // Stream i's signal is [overlap | chunk] from sample sig_off; its frames go to mel_in after its leftover frames.
    int64_t coff = 0, soff = 0;
    int moff = 0;
    auto chunk = [&](int i, StreamPlan &p) -> pk_status {
        const int64_t n64 = offsets[i + 1] - offsets[i];
        if (n64 < 0 || n64 > s.max_chunk) return e->fail(PK_ERR_CAPACITY, "pk_stream_step: chunk longer than max_chunk_samples");
        const int n = (int)n64, total = s.ovl_len[i] + n;
        p.chunk_off = coff; p.sig_off = soff; p.chunk_len = n; p.ovl_len = s.ovl_len[i]; p.min_off = moff;
        if (total >= 400) {                        // audio.cpp:225-229: below one window, keep everything
            const int nfh = (total - 400) / 160 + 1;
            p.consumed = (nfh - 1) * 160 + 400;
            // fft::stft(center = false) is called with n_fft = 512 on `consumed` samples: the reference throws below 512
            // (fft.cpp:1516-1521) and otherwise returns (consumed - 512) / 160 + 1 frames -- one fewer than nfh (DESIGN.md)
            if (p.consumed < 512) return e->fail(PK_ERR_INVALID, "pk_stream_step: stft: signal length is less than n_fft (the reference throws here: first chunk of 400..511 samples)");
            p.nf = (p.consumed - 512) / 160 + 1;
        }
        s.meta_h(Meta::NF)[i] = p.nf;
        s.meta_h(Meta::OUT_ROW)[i] = p.min_off + p.left;
        s.h_sig_off[i] = soff;
        if (n > 0) memcpy(s.h_chunk + coff, pcm + offsets[i], sizeof(float) * n);
        coff += n; soff += total; moff += p.left + p.nf;
        return PK_OK;
    };
    auto upload = [&](cudaStream_t st) {
        s.h_sig_off[S] = soff;
        cudaError_t ce = cudaMemcpyAsync(s.d_sig_off, s.h_sig_off, sizeof(int64_t) * (S + 1), cudaMemcpyHostToDevice, st);
        if (ce == cudaSuccess && coff > 0) ce = cudaMemcpyAsync(s.d_chunk, s.h_chunk, sizeof(float) * coff, cudaMemcpyHostToDevice, st);
        return ce;
    };
    auto front = [&](int max_nf) {
        cudaStream_t st = e->stream;
        launch_stream_prep(s.d_chunk, s.d_plan, s.st, S, s.ssig, s.mel_in, c.mel_bins, st);
        {
            pk_engine::Scope sc(e, pk_engine::CAT_MEL);
            launch_mel_stream(s.ssig, s.d_sig_off, s.meta_d(Meta::NF), s.meta_d(Meta::OUT_ROW), S, max_nf, c.mel_bins, e->mel_tb, s.mel_in, st);
        }
        launch_stream_post(s.d_chunk, s.d_plan, s.st, S, s.ssig, s.mel_in, c.mel_bins, e->feats, st);
        e->launches += 3;
        if (mel_out) {      // debug tap: the new frames of every stream, packed
            size_t o = 0;
            for (int i = 0; i < S; ++i) {
                const StreamPlan &p = s.h_plan[i];
                if (p.nf > 0 && cudaMemcpyAsync(mel_out + o, s.mel_in + (size_t)(p.min_off + p.left) * c.mel_bins,
                                                sizeof(float) * p.nf * c.mel_bins, cudaMemcpyDeviceToHost, st) != cudaSuccess)
                    break;
                o += (size_t)p.nf * c.mel_bins;
            }
        }
    };
    // rnnt_streaming_decode_chunk (eou.cpp:17-98) for all streams: the TDT decode kernel with carried state
    auto decode = [e, &s]() {
        TdtParams p{};   // (max_sym stays 0: pk_stream_open takes TDT models only)
        p.Bpad = e->Bpad; p.n_utt = s.S; p.max_steps = *std::max_element(s.nC.begin(), s.nC.end()) + e->cap + 2;
        p.row_off = s.meta_d(Meta::ROW_OFF); p.hbuf = s.hbuf;
        p.carry = 1; p.c_state = s.c_state; p.tok_state = s.tok_state; p.frame_base = s.meta_d(Meta::FRAME_BASE);
        p.boost_on = s.n_boosted > 0 ? 1 : 0; p.trie = s.boost.trie(); p.boost_bits = s.boost_bits; p.trie_active = s.trie_active; p.trie_nact = s.trie_nact;
        return e->tdt_decode(p);
    };
    // (the graph key depends on whether any stream is boosted: the lists themselves live in buffers that never move)
    if (pk_status ps = stream_step(e, "pk_stream_step", s.n_boosted > 0 ? 'b' : 's', n_mel, n_enc, nullptr, enc_out, chunk, upload, front, decode))
        return ps;
    if (!out) return PK_OK;
    if (s.act.empty()) {
        for (int i = 0; i < S; ++i) out->len[i] = 0;
        const cudaError_t ce = cudaStreamSynchronize(e->stream);
        return ce == cudaSuccess ? PK_OK : e->fail(PK_ERR_CUDA, std::string("pk_stream_step: ") + cudaGetErrorString(ce));
    }
    e->n_utt = S;                                   // the token rows cover all streams
    return e->fetch(out);
}

pk_status pk_stream_set_boost(pk_engine *e, int32_t stream, const int32_t *phrase_ids, const int32_t *phrase_off, int32_t n_phrases, float boost) {
    if (!e || n_phrases < 0 || (n_phrases > 0 && (!phrase_ids || !phrase_off))) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_stream_set_boost: a Sortformer engine has no decoder");
    if (!e->ss) return e->fail(PK_ERR_INVALID, "pk_stream_set_boost: no streams are open (pk_stream_open)");
    StreamSet &s = *e->ss;
    if (stream < 0 || stream >= s.S) return e->fail(PK_ERR_INVALID, "pk_stream_set_boost: bad stream index");
    const int32_t row_off[2] = {0, n_phrases};
    bool any = false;
    if (pk_status ps = e->boost_upload("pk_stream_set_boost", s.boost, stream, 1, 0, phrase_ids, phrase_off, row_off, &boost, &any)) return ps;
    s.n_boosted += (any ? 1 : 0) - (s.boosted[stream] ? 1 : 0);
    s.boosted[stream] = any ? 1 : 0;
    launch_boost_state_reset(s.boost.trie(), e->cfg.vocab, stream, 1, s.boost_bits, s.trie_active, s.trie_nact, e->stream);
    const cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_stream_set_boost: ") + cudaGetErrorString(ce));
    return PK_OK;
}

int32_t pk_stream_count(const pk_engine *e) { return (e && e->ss && !e->diar) ? e->ss->S : 0; }

// ===================================================================== Sortformer streams (sortformer.cpp:124-150)
// Sortformer::diarize_chunk for S streams in lock step.  Per stream and step: the chunk's own centred log-mel without
// normalisation (preprocess_audio(chunk, {n_mels = mel_bins, normalize = false}), no state across chunks), the NEST encoder's
// forward_chunk (leftover frames, K/V rings and conv caches of every layer), then projection_ -> transformer_ -> speaker head
// on THIS chunk's encoder rows only (each active stream is one utterance of the packed step), and the AOSC update on the host.

pk_status pk_diar_stream_open(pk_engine *e, int32_t n_streams, int32_t max_chunk_samples, int32_t att_context_left) {
    if (!e || n_streams < 1 || max_chunk_samples < 1 || att_context_left < 1) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (!e->diar) return e->fail(PK_ERR_INVALID, "pk_diar_stream_open: not a Sortformer engine (pk_sortformer_create)");
    const pk_config &c = e->cfg;
    auto s = std::make_unique<StreamSet>();
    s->diar = true;
    s->S = n_streams; s->L = att_context_left; s->R = 0; s->max_chunk = max_chunk_samples;
    s->nf_max = 1 + max_chunk_samples / 160;                   // centred STFT: 1 + n / 160 frames per chunk
    if (pk_status ps = stream_alloc(e, "pk_diar_stream_open", "diarization stream", *s)) return ps;
    const size_t mel_floats = (size_t)n_streams * s->nf_max * c.mel_bins;
    s->spk_seen.assign(n_streams, 0); s->arrival.assign(n_streams, {});
    s->mel_new = e->dalloc<float>(mel_floats);
    if (!s->mel_new) return e->fail(PK_ERR_CUDA, "cudaMalloc failed (diarization stream state)");
    if (cudaMallocHost(&s->h_mel, sizeof(float) * mel_floats) != cudaSuccess)
        return e->fail(PK_ERR_CUDA, "cudaMallocHost failed (diarization stream staging)");
    return stream_install(e, std::move(s), pk_diar_stream_reset);
}

// A fresh EncoderCache and AOSCCache::reset (sortformer.cpp:35-38) for one stream (or all: stream = -1)
pk_status pk_diar_stream_reset(pk_engine *e, int32_t stream) {
    if (!e) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (!e->diar || !e->ss) return e->fail(PK_ERR_INVALID, "pk_diar_stream_reset: no Sortformer streams open (pk_diar_stream_open)");
    StreamSet &s = *e->ss;
    return stream_reset(e, "pk_diar_stream_reset", stream, [&](int s0, int s1) {
        for (int i = s0; i < s1; ++i) {
            s.spk_seen[i] = 0;
            s.arrival[i].clear();
        }
        return cudaSuccess;
    });
}

namespace {

// One step from PCM (pcm / offsets) or from host features (feats / n_frames).
pk_status diar_stream_step(pk_engine *e, const float *pcm, const int64_t *offsets, const float *feats, const int32_t *n_frames,
                           float *probs_out, int32_t *n_out, int32_t *frame_base_out, float *enc_out) {
    const char *fn = feats ? "pk_diar_stream_step_feats" : "pk_diar_stream_step";
    if (!e) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (!e->diar || !e->ss) return e->fail(PK_ERR_INVALID, std::string(fn) + ": no Sortformer streams open (pk_diar_stream_open)");
    StreamSet &s = *e->ss;
    const pk_config &c = e->cfg;
    const int S = s.S, nm = c.mel_bins, SP = e->sf.max_speakers;
    // Stream i's new frames are rows [mel_off[i], mel_off[i+1]) of mel_new; its chunk starts at sample sig_off[i].
    int32_t *m_fo = s.meta_h(Meta::MEL_OFF);
    int64_t soff = 0;
    int moff = 0;
    auto chunk = [&](int i, StreamPlan &p) -> pk_status {
        if (feats) {
            p.nf = n_frames ? n_frames[i] : -1;
            if (p.nf < 0) return e->fail(PK_ERR_INVALID, std::string(fn) + ": n_frames missing or negative");
            if (p.nf > s.nf_max) return e->fail(PK_ERR_CAPACITY, std::string(fn) + ": more frames than a chunk of max_chunk_samples makes");
        } else {
            const int64_t n = offsets[i + 1] - offsets[i];
            if (n < 0 || n > s.max_chunk) return e->fail(PK_ERR_CAPACITY, std::string(fn) + ": chunk longer than max_chunk_samples");
            // axiom's reflect pad never terminates on a 1-sample signal (operations.cpp:2217-2227, DESIGN.md)
            if (n == 1) return e->fail(PK_ERR_INVALID, std::string(fn) + ": a 1-sample chunk cannot be reflect-padded (the reference does not return)");
            p.nf = n > 0 ? (int)(1 + n / 160) : 0;
            s.h_sig_off[i] = soff;
            if (n > 0) memcpy(s.h_chunk + soff, pcm + offsets[i], sizeof(float) * n);
            soff += n;
        }
        m_fo[i] = p.min_off = moff;
        moff += p.nf;
        m_fo[i + 1] = moff;
        return PK_OK;
    };
    auto upload = [&](cudaStream_t st) {
        cudaError_t ce = cudaSuccess;
        if (!feats) {
            s.h_sig_off[S] = soff;
            ce = cudaMemcpyAsync(s.d_sig_off, s.h_sig_off, sizeof(int64_t) * (S + 1), cudaMemcpyHostToDevice, st);
            if (ce == cudaSuccess && soff > 0) ce = cudaMemcpyAsync(s.d_chunk, s.h_chunk, sizeof(float) * soff, cudaMemcpyHostToDevice, st);
        } else if (moff > 0) {
            memcpy(s.h_mel, feats, sizeof(float) * (size_t)moff * nm);
            ce = cudaMemcpyAsync(s.mel_new, s.h_mel, sizeof(float) * (size_t)moff * nm, cudaMemcpyHostToDevice, st);
        }
        return ce;
    };
    // every chunk's centred log-mel in one launch (K1 of the offline front end), then the queue join
    auto front = [&](int max_nf) {
        cudaStream_t st = e->stream;
        if (!feats && max_nf > 0) {
            pk_engine::Scope sc(e, pk_engine::CAT_MEL);
            launch_mel(s.d_chunk, s.d_sig_off, s.meta_d(Meta::MEL_OFF), S, max_nf, nm, e->mel_tb, nullptr, s.mel_new, nullptr, st, false);
            ++e->launches;
        }
        launch_diar_stream_join(s.d_plan, s.mel_new, s.st.melq, S, nm, e->feats, st);
        ++e->launches;
    };
    // projection_, transformer_ and the speaker head on the encoder rows ('D': not an offline diarization key 'd' nor an
    // ASR stream key 's')
    if (pk_status ps = stream_step(e, fn, 'D', nullptr, n_out, frame_base_out, enc_out, chunk, upload, front, [e] { return e->run_diar_head(); }))
        return ps;
    cudaStream_t st = e->stream;
    if (s.act.empty()) {                           // CausalConvSubsampling returned nothing for every stream: no AOSC update
        const cudaError_t ce = cudaStreamSynchronize(st);
        return ce == cudaSuccess ? PK_OK : e->fail(PK_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(ce));
    }
    const size_t np = (size_t)e->M * SP;
    cudaError_t ce = cudaMemcpyAsync(e->h_probs, e->probs, np * sizeof(float), cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(ce));
    if (probs_out) memcpy(probs_out, e->h_probs, np * sizeof(float));
    // AOSCCache::update (sortformer.cpp:15-31): a speaker arrives the first time p > 0.5; within a frame in index order
    const int32_t *m_ro = s.meta_h(Meta::ROW_OFF);
    for (int i : s.act)
        for (int t = m_ro[i]; t < m_ro[i + 1]; ++t)
            for (int k = 0; k < SP; ++k)
                if (e->h_probs[(size_t)t * SP + k] > 0.5f && !(s.spk_seen[i] >> k & 1)) {
                    s.spk_seen[i] |= 1ull << k;
                    s.arrival[i].push_back(k);
                }
    return PK_OK;
}

}  // namespace

pk_status pk_diar_stream_step(pk_engine *e, const float *pcm, const int64_t *offsets, float *probs_out, int32_t *n_out,
                              int32_t *frame_base_out, float *enc_out) {
    if (!e || !offsets || (e->ss && !pcm && offsets[e->ss->S] > offsets[0])) return PK_ERR_INVALID;
    return diar_stream_step(e, pcm, offsets, nullptr, nullptr, probs_out, n_out, frame_base_out, enc_out);
}

pk_status pk_diar_stream_step_feats(pk_engine *e, const float *feats, const int32_t *n_frames, float *probs_out, int32_t *n_out,
                                    int32_t *frame_base_out, float *enc_out) {
    if (!e || !n_frames) return PK_ERR_INVALID;
    if (!feats && e->ss)
        for (int i = 0; i < e->ss->S; ++i)
            if (n_frames[i] > 0) return e->fail(PK_ERR_INVALID, "pk_diar_stream_step_feats: frames without features");
    static const float none = 0.f;
    return diar_stream_step(e, nullptr, nullptr, feats ? feats : &none, n_frames, probs_out, n_out, frame_base_out, enc_out);
}

int32_t pk_diar_stream_speakers(const pk_engine *e, int32_t stream, int32_t *order, int32_t cap) {
    if (!e || !e->diar || !e->ss || stream < 0 || stream >= e->ss->S || cap < 0 || (cap > 0 && !order)) return -1;
    const std::vector<int32_t> &a = e->ss->arrival[stream];
    for (size_t i = 0; i < a.size() && (int64_t)i < cap; ++i) order[i] = a[i];
    return (int32_t)a.size();
}

int32_t pk_diar_stream_count(const pk_engine *e) { return (e && e->diar && e->ss) ? e->ss->S : 0; }

}  // extern "C"

void pk_stream_free(pk_engine *e) {
    if (!e) return;
    delete e->ss;
    e->ss = nullptr;
}
