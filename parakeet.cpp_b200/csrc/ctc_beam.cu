// ctc_beam.cu -- CTC prefix beam search with word n-gram shallow fusion (PK_DECODER_CTC_BEAM; DESIGN.md section 14 is the
// definition this file implements, tests/ctc_beam_oracle.py its float64 restatement).
//
//   ctc_frame_topk_kernel : per frame, over every frame of the batch at once, the W best non-blank (id, log-prob) pairs
//                           (ties to the lower id) and lp[blank], read from the log-probs of ctc_frame_argmax_kernel.
//   ctc_beam_kernel       : one CTA per utterance walks its frames: W (1 + W) candidates, merged by token sequence,
//                           LM terms for word-starting extensions, block-wide top-W, one back-pointer row per frame; at the
//                           end the end-of-utterance LM terms, the best beam, and the backtrack into the greedy layout.
//
// Beam scores (ln probabilities and LM terms) are kept in double: the decode compares sums of hundreds of terms, and in
// double its decisions agree with the float64 oracle unless two candidates are within ~1e-12 of each other.
// Prefixes are identified by a 64-bit hash of their token sequence; a collision between two live prefixes is ignored
// (it would merge them).
#include "kernels.h"
#include "lm.h"

namespace pk {
namespace {

constexpr int BEAM_MAX = PK_CTC_BEAM_MAX;
constexpr int NWARP = CTC_BEAM_THREADS / 32;
constexpr int MAX_CAND = BEAM_MAX * (1 + BEAM_MAX);
constexpr int PER_LANE = (MAX_CAND / NWARP + 31) / 32;   // candidates a lane scans in the per-warp selection

__global__ void __launch_bounds__(256)
ctc_frame_topk_kernel(const float *__restrict__ logprobs, int M, int V, int W, int32_t *__restrict__ topk_id,
                      float *__restrict__ topk_lp, float *__restrict__ blank_lp) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    const float *l = logprobs + (size_t)row * V;
    const int blank = V - 1;
    // lane k < W holds the k-th best so far, in (value desc, id asc) order; absent entries are (-inf, -1)
    float lv = -INFINITY;
    int li = -1;
    for (int base = 0; base < blank; base += 32) {
        const int v = base + lane;
        const float x = v < blank ? l[v] : -INFINITY;
        unsigned cand = __ballot_sync(0xffffffffu, x > __shfl_sync(0xffffffffu, lv, W - 1));   // (NaN never enters)
        while (cand) {
            const int src = __ffs(cand) - 1;
            cand &= cand - 1;
            const float cx = __shfl_sync(0xffffffffu, x, src);
            if (!(cx > __shfl_sync(0xffffffffu, lv, W - 1))) continue;
            // entries of equal value have lower ids (the scan is in id order): the new one goes after them
            const int pos = __popc(__ballot_sync(0xffffffffu, lane < W && lv >= cx));
            const float uv = __shfl_up_sync(0xffffffffu, lv, 1);
            const int ui = __shfl_up_sync(0xffffffffu, li, 1);
            if (lane > pos) {
                lv = uv;
                li = ui;
            } else if (lane == pos) {
                lv = cx;
                li = base + src;
            }
        }
    }
    if (lane < W) {
        topk_id[(size_t)row * W + lane] = li;
        topk_lp[(size_t)row * W + lane] = lv;
    }
    if (lane == 0) blank_lp[row] = l[blank];
}

__device__ __forceinline__ double lse(double a, double b) {
    if (a == -INFINITY) return b;
    if (b == -INFINITY) return a;
    const double m = fmax(a, b);
    return m + log1p(exp(-fabs(a - b)));
}

__device__ __forceinline__ unsigned long long prefix_hash(unsigned long long h, int c) {
    unsigned long long z = h + 0x9e3779b97f4a7c15ull * (unsigned long long)(c + 1);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

__device__ int lm_word(const DeviceLM &lm, unsigned long long h) {
    if (h == 0) h = 1;
    for (uint32_t i = lm_slot(h, lm.word_mask);; i = (i + 1) & lm.word_mask) {
        const unsigned long long k = lm.word_key[i];
        if (k == h) return lm.word_id[i];
        if (k == 0) return lm.unk;
    }
}

// log10 p(wid | state) by ARPA back-off (pk_lm::score restated); moves the state on
__device__ double lm_score(const DeviceLM &lm, int &state, int wid) {
    double acc = 0.0;
    int ctx = state;
    while (ctx >= 0) {
        const unsigned long long key = lm_ngram_key(ctx, wid);
        for (uint32_t i = lm_slot(key, lm.ng_mask);; i = (i + 1) & lm.ng_mask) {
            const unsigned long long k = lm.ng_key[i];
            if (k == key) {
                const int e = lm.ng_val[i];
                state = lm.order[e] == lm.max_order ? lm.suffix[e] : e;
                return acc + lm.prob[e];
            }
            if (k == 0) break;
        }
        acc += lm.backoff[ctx];
        ctx = lm.suffix[ctx];
    }
    state = 0;            // (not reached: every word id is a 1-gram, found from the empty context)
    return acc;
}

struct BeamSet {          // W beams, structure of arrays
    double pb[BEAM_MAX], pnb[BEAM_MAX], lm[BEAM_MAX];
    unsigned long long h[BEAM_MAX], ph[BEAM_MAX], wh[BEAM_MAX];   // prefix hash, its parent prefix's hash, word hash
    int state[BEAM_MAX], last[BEAM_MAX], wlen[BEAM_MAX];
};

__global__ void __launch_bounds__(CTC_BEAM_THREADS)
ctc_beam_kernel(const float *__restrict__ logprobs, const int32_t *__restrict__ topk_id, const float *__restrict__ topk_lp,
                const float *__restrict__ blank_lp, const int32_t *__restrict__ row_off, int V, int W, int cap, DeviceLM lm,
                DevicePieces pc, int32_t *__restrict__ bp, int32_t *__restrict__ tok, int32_t *__restrict__ t_start,
                int32_t *__restrict__ t_end, float *__restrict__ t_conf) {
    __shared__ BeamSet bs[2];
    __shared__ double c_sc[MAX_CAND];                  // candidate scores: [blank/repeat of beam j][extension (i, r) at nb + i W + r]
    __shared__ double n_pb[BEAM_MAX], n_pnb[BEAM_MAX], w_sc[BEAM_MAX];
    __shared__ int n_bp[BEAM_MAX], w_state[BEAM_MAX], f_id[BEAM_MAX], sel[BEAM_MAX];
    __shared__ float f_lp[BEAM_MAX];
    __shared__ unsigned mmask[BEAM_MAX];               // extensions (i, r) merged into a blank/repeat candidate
    __shared__ double fin_sc[NWARP * BEAM_MAX];
    __shared__ int fin_pos[NWARP * BEAM_MAX];
    __shared__ float f_blank;
    __shared__ int s_nb;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    const bool use_lm = lm.word_key != nullptr;
    if (tid == 0) {
        bs[0].pb[0] = 0.0;
        bs[0].pnb[0] = -INFINITY;
        bs[0].lm[0] = 0.0;
        bs[0].h[0] = 0x243f6a8885a308d3ull;
        bs[0].ph[0] = 0;
        bs[0].wh[0] = kFnvBasis;
        bs[0].state[0] = lm.start;
        bs[0].last[0] = -1;
        bs[0].wlen[0] = 0;
        s_nb = T > 0 ? 1 : 0;
    }
    __syncthreads();
    int cur = 0;
    for (int t = 0; t < T; ++t) {
        const int nb = s_nb;
        if (nb == 0) break;
        const BeamSet &B = bs[cur];
        BeamSet &N = bs[cur ^ 1];
        const size_t row = (size_t)(r0 + t);
        // (a) the frame's top-W; each beam's unfinished word scored as a word-starting extension would complete it
        if (tid < W) {
            f_id[tid] = topk_id[row * W + tid];
            f_lp[tid] = topk_lp[row * W + tid];
        }
        if (tid == 0) f_blank = blank_lp[row];
        if (tid < nb) {
            mmask[tid] = 0u;
            if (use_lm && B.wlen[tid] > 0) {
                int st = B.state[tid];
                const double s = lm_score(lm, st, lm_word(lm, B.wh[tid]));
                w_sc[tid] = lm.alpha_ln10 * s + lm.beta;
                w_state[tid] = st;
            }
        }
        __syncthreads();
        // (b) blank/repeat candidate of beam j, and the one extension that has its token sequence merged into it
        if (tid < nb) {
            const int j = tid, lj = B.last[j];
            const double npb = lse(B.pb[j], B.pnb[j]) + (double)f_blank;
            double npnb = lj >= 0 ? B.pnb[j] + (double)logprobs[row * V + lj] : -INFINITY;
            const double own = lse(npb, npnb);
            int lineage = (j << 24);
            if (lj >= 0) {
                int i = -1;
                for (int k = 0; k < nb; ++k)
                    if (B.h[k] == B.ph[j]) { i = k; break; }
                int r = -1;
                if (i >= 0)
                    for (int k = 0; k < W; ++k)
                        if (f_id[k] == lj) { r = k; break; }
                if (r >= 0) {
                    const double ext = (lj == B.last[i] ? B.pb[i] : lse(B.pb[i], B.pnb[i])) + (double)f_lp[r];
                    atomicOr(&mmask[i], 1u << r);
                    if (ext > own) lineage = (i << 24) | (lj + 1);
                    npnb = lse(npnb, ext);
                }
            }
            n_pb[j] = npb;
            n_pnb[j] = npnb;
            n_bp[j] = lineage;
            c_sc[j] = lse(npb, npnb) + B.lm[j];
        }
        __syncthreads();
        // (c) the extensions that are new prefixes
        for (int p = tid; p < nb * W; p += blockDim.x) {
            const int i = p / W, r = p - i * W, c = f_id[r];
            double s = -INFINITY;
            if (c >= 0 && !((mmask[i] >> r) & 1u)) {
                s = (c == B.last[i] ? B.pb[i] : lse(B.pb[i], B.pnb[i])) + (double)f_lp[r] + B.lm[i];
                if (use_lm && B.wlen[i] > 0 && pc.starts[c]) s += w_sc[i];
            }
            c_sc[nb + p] = s;
        }
        __syncthreads();
        // (d) top-W: each warp extracts the W best of its slice, then the 8 W finalists are ranked
        const int n_cand = nb * (1 + W), chunk = (n_cand + NWARP - 1) / NWARP;
        const int lo = warp * chunk, hi = min(n_cand, lo + chunk);
        unsigned taken = 0u;
        int got = 0;
        for (; got < W; ++got) {
            double bv = -INFINITY;
            int bpos = 0x7fffffff, bk = -1;
            for (int k = 0; k < PER_LANE; ++k) {
                const int idx = lo + lane + 32 * k;
                if (idx < hi && !((taken >> k) & 1u) && c_sc[idx] > bv) {
                    bv = c_sc[idx];
                    bpos = idx;
                    bk = k;
                }
            }
            const int mine = bpos;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int op = __shfl_xor_sync(0xffffffffu, bpos, o);
                if (ov > bv || (ov == bv && op < bpos)) {
                    bv = ov;
                    bpos = op;
                }
            }
            if (bv == -INFINITY) break;
            if (bk >= 0 && mine == bpos) taken |= 1u << bk;
            if (lane == 0) {
                fin_sc[warp * W + got] = bv;
                fin_pos[warp * W + got] = bpos;
            }
        }
        if (lane == 0)
            for (int k = got; k < W; ++k) fin_sc[warp * W + k] = -INFINITY;
        if (tid == 0) s_nb = 0;
        __syncthreads();
        if (tid < NWARP * W && fin_sc[tid] != -INFINITY) {
            const double v = fin_sc[tid];
            const int pos = fin_pos[tid];
            int rank = 0;
            for (int k = 0; k < NWARP * W; ++k) {
                const double o = fin_sc[k];
                rank += o > v || (o == v && fin_pos[k] < pos);
            }
            if (rank < W) {
                sel[rank] = pos;
                atomicAdd(&s_nb, 1);
            }
        }
        __syncthreads();
        // (e) the new beams and this frame's back-pointer row
        const int nn = s_nb;
        if (tid < nn) {
            const int s = tid, pos = sel[s];
            int ptr;
            if (pos < nb) {
                const int j = pos;
                N.pb[s] = n_pb[j];
                N.pnb[s] = n_pnb[j];
                N.lm[s] = B.lm[j];
                N.h[s] = B.h[j];
                N.ph[s] = B.ph[j];
                N.wh[s] = B.wh[j];
                N.state[s] = B.state[j];
                N.last[s] = B.last[j];
                N.wlen[s] = B.wlen[j];
                ptr = n_bp[j];
            } else {
                const int p = pos - nb, i = p / W, r = p - i * W, c = f_id[r];
                N.pb[s] = -INFINITY;
                N.pnb[s] = (c == B.last[i] ? B.pb[i] : lse(B.pb[i], B.pnb[i])) + (double)f_lp[r];
                N.h[s] = prefix_hash(B.h[i], c);
                N.ph[s] = B.h[i];
                N.last[s] = c;
                double lmv = B.lm[i];
                int st = B.state[i];
                unsigned long long wh = B.wh[i];
                int wl = B.wlen[i];
                if (use_lm) {
                    const int n0 = pc.off[c], n1 = pc.off[c + 1];
                    if (pc.starts[c]) {
                        if (wl > 0) {
                            lmv += w_sc[i];
                            st = w_state[i];
                        }
                        wh = kFnvBasis;
                        wl = 0;
                    }
                    wh = fnv1a(wh, pc.bytes + n0, (size_t)(n1 - n0));
                    wl += n1 - n0;
                }
                N.lm[s] = lmv;
                N.state[s] = st;
                N.wh[s] = wh;
                N.wlen[s] = wl;
                ptr = (i << 24) | (c + 1);
            }
            bp[row * W + s] = ptr;
        }
        cur ^= 1;
        __syncthreads();
    }
    // end of the utterance: unfinished word and </s>, best beam (ties to the lower slot), backtrack
    if (tid == 0) {
        const BeamSet &B = bs[cur];
        const int nb = s_nb;
        int best = -1;
        double bv = -INFINITY;
        for (int s = 0; s < nb; ++s) {
            double v = lse(B.pb[s], B.pnb[s]) + B.lm[s];
            if (use_lm) {
                int st = B.state[s];
                double e = 0.0;
                if (B.wlen[s] > 0) {
                    e += lm_score(lm, st, lm_word(lm, B.wh[s]));
                    v += lm.beta;
                }
                e += lm_score(lm, st, lm.eos);
                v += lm.alpha_ln10 * e;
            }
            if (v > bv) {
                bv = v;
                best = s;
            }
        }
        int n = 0;
        if (best >= 0) {
            for (int t = T - 1, s = best; t >= 0; --t) {
                const int e = bp[(size_t)(r0 + t) * W + s];
                n += (e & 0xffffff) != 0;
                s = e >> 24;
            }
            int32_t *ids = tok + (size_t)b * (1 + cap) + 1;
            int32_t *stp = t_start + (size_t)b * cap, *enp = t_end + (size_t)b * cap;
            float *cf = t_conf + (size_t)b * cap;
            int k = n, next_start = T;
            for (int t = T - 1, s = best; t >= 0; --t) {
                const int e = bp[(size_t)(r0 + t) * W + s];
                const int c = (e & 0xffffff) - 1;
                if (c >= 0) {
                    --k;
                    if (k < cap) {
                        ids[k] = c;
                        stp[k] = t;
                        enp[k] = next_start - 1;
                        cf[k] = expf(logprobs[(size_t)(r0 + t) * V + c]);
                    }
                    next_start = t;
                }
                s = e >> 24;
            }
        }
        tok[(size_t)b * (1 + cap)] = n < cap ? n : cap;
    }
}

}  // namespace

uint64_t ctc_beam_tables_id(const pk_lm *lm, const pk_vocab *vocab, int V) {
    if (!lm) return 0;
    uint64_t h = fnv1a(kFnvBasis, reinterpret_cast<const uint8_t *>(&lm->serial), sizeof(lm->serial));
    const std::vector<std::string> *pieces = vocab_pieces(vocab);
    for (int v = 0; pieces && v < V - 1 && v < (int)pieces->size(); ++v) {
        const std::string &p = (*pieces)[v];
        h = fnv1a(h, reinterpret_cast<const uint8_t *>(p.data()), p.size() + 1);   // (with the terminating NUL as separator)
    }
    return h ? h : 1;
}

std::string ctc_beam_tables(const pk_lm *lm, const pk_vocab *vocab, int V, const std::function<void *(const void *, size_t)> &upload,
                            DeviceLM *lm_out, DevicePieces *pc_out) {
    *lm_out = DeviceLM{};
    *pc_out = DevicePieces{};
    if (!lm) return "";
    const std::vector<std::string> *pieces = vocab_pieces(vocab);
    if (!pieces) return "a language model needs the vocabulary (pk_vocab) of the model";
    if ((int)pieces->size() < V - 1)
        return "the vocabulary has " + std::to_string(pieces->size()) + " pieces, the model " + std::to_string(V - 1) + " non-blank tokens";
    std::vector<uint8_t> bytes, starts(V, 0);
    std::vector<int32_t> off(V + 1, 0);
    for (int v = 0; v < V - 1; ++v) {
        const std::string &p = (*pieces)[v];
        const bool mark = p.size() >= 3 && p.compare(0, 3, "\xe2\x96\x81") == 0;   // U+2581
        starts[v] = mark;
        bytes.insert(bytes.end(), p.begin() + (mark ? 3 : 0), p.end());
        off[v + 1] = (int32_t)bytes.size();
    }
    off[V] = (int32_t)bytes.size();                 // the blank: no bytes (never appended)
    bytes.push_back(0);
    const LmTables &t = lm->tables;
    void *p[11] = {upload(t.word_key.data(), t.word_key.size() * 8), upload(t.word_id.data(), t.word_id.size() * 4),
                   upload(t.ng_key.data(), t.ng_key.size() * 8), upload(t.ng_val.data(), t.ng_val.size() * 4),
                   upload(t.prob.data(), t.prob.size() * 8), upload(t.backoff.data(), t.backoff.size() * 8),
                   upload(t.suffix.data(), t.suffix.size() * 4), upload(t.order.data(), t.order.size() * 4),
                   upload(bytes.data(), bytes.size()), upload(off.data(), off.size() * 4), upload(starts.data(), starts.size())};
    for (void *q : p)
        if (!q) return "cudaMalloc failed (language-model tables)";
    lm_out->word_key = static_cast<const unsigned long long *>(p[0]);
    lm_out->word_id = static_cast<const int32_t *>(p[1]);
    lm_out->ng_key = static_cast<const unsigned long long *>(p[2]);
    lm_out->ng_val = static_cast<const int32_t *>(p[3]);
    lm_out->prob = static_cast<const double *>(p[4]);
    lm_out->backoff = static_cast<const double *>(p[5]);
    lm_out->suffix = static_cast<const int32_t *>(p[6]);
    lm_out->order = static_cast<const int32_t *>(p[7]);
    lm_out->word_mask = t.word_mask;
    lm_out->ng_mask = t.ng_mask;
    lm_out->max_order = lm->max_order;
    lm_out->start = lm->start;
    lm_out->unk = lm->unk;
    lm_out->eos = lm->eos;
    pc_out->bytes = static_cast<const uint8_t *>(p[8]);
    pc_out->off = static_cast<const int32_t *>(p[9]);
    pc_out->starts = static_cast<const uint8_t *>(p[10]);
    return "";
}

void launch_ctc_frame_topk(const float *logprobs, int M, int V, int width, int32_t *topk_id, float *topk_lp, float *blank_lp,
                           cudaStream_t st) {
    if (M <= 0) return;
    ctc_frame_topk_kernel<<<dim3((M + 7) / 8), dim3(256), 0, st>>>(logprobs, M, V, width, topk_id, topk_lp, blank_lp);
}

void launch_ctc_beam(const float *logprobs, const int32_t *topk_id, const float *topk_lp, const float *blank_lp,
                     const int32_t *row_off, int n_utt, int V, int width, int cap, const DeviceLM &lm, const DevicePieces &pieces,
                     int32_t *bp, int32_t *tok, int32_t *t_start, int32_t *t_end, float *t_conf, cudaStream_t st) {
    ctc_beam_kernel<<<dim3(n_utt), dim3(CTC_BEAM_THREADS), 0, st>>>(logprobs, topk_id, topk_lp, blank_lp, row_off, V, width,
               cap, lm, pieces, bp, tok, t_start, t_end, t_conf);
}

}  // namespace pk
