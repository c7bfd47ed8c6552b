// ctc.cu -- K9: CTC head reductions and greedy collapse.
//
// The head GEMM (CTCDecoder::forward's k=1 Conv1d, reference src/ctc.cpp:12-18) runs in the
// GEMM kernel; this file replaces log_softmax (:24) + the argmax scan + collapse of
// ctc_greedy_decode / ctc_greedy_decode_with_timestamps (src/ctc.cpp:40-127):
//   ctc_frame_argmax_kernel : per frame, first maximum (strict '>' scan order, :59-66) and
//                             exp(max log-prob) = 1 / sum exp(l - max)  (:110)
//   ctc_collapse_kernel     : per utterance, drop blanks/repeats (prev updates on every
//                             frame, :69-72), token spans: start = first frame of the run,
//                             end closed at t-1 when the argmax changes after a non-blank
//                             run, last token's end forced to T-1 (:104-121).
#include "kernels.h"

namespace pk {
namespace {

__global__ void __launch_bounds__(256)
ctc_frame_argmax_kernel(const float *__restrict__ logits, int M, int V, int ld, int32_t *__restrict__ best,
                        float *__restrict__ conf, float *__restrict__ logprobs) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    const float *l = logits + (size_t)row * ld;
    float mx = -INFINITY;
    int idx = 0x7fffffff;
    for (int v = lane; v < V; v += 32) {
        const float x = l[v];
        if (x > mx) {
            mx = x;
            idx = v;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, mx, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (om > mx || (om == mx && oi < idx)) {
            mx = om;
            idx = oi;
        }
    }
    float s = 0.f;
    for (int v = lane; v < V; v += 32) s += expf(l[v] - mx);
    s = warp_sum(s);
    if (lane == 0) {
        // no element > -inf (all -inf or NaN): the reference's scan starts at index 0 and keeps it
        best[row] = idx == 0x7fffffff ? 0 : idx;
        conf[row] = 1.0f / s;
    }
    if (logprobs) {
        const float lse = logf(s);
        for (int v = lane; v < V; v += 32) logprobs[(size_t)row * V + v] = (l[v] - mx) - lse;
    }
}

// greedy collapse of utterance b from the per-frame arg-max, by one thread
__device__ __forceinline__ void ctc_collapse_row(const int32_t *__restrict__ best, const float *__restrict__ conf,
                                                 const int32_t *__restrict__ row_off, int b, int blank, int cap,
                                                 int32_t *__restrict__ tok, int32_t *__restrict__ t_start,
                                                 int32_t *__restrict__ t_end, float *__restrict__ t_conf) {
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    int32_t *ids = tok + (size_t)b * (1 + cap) + 1;
    int32_t *st = t_start + (size_t)b * cap, *en = t_end + (size_t)b * cap;
    float *cf = t_conf + (size_t)b * cap;
    int prev = -1, n = 0;
    for (int t = 0; t < T; ++t) {
        const int cur = best[r0 + t];
        if (cur != prev) {
            if (prev != -1 && prev != blank && n > 0 && n <= cap) en[n - 1] = t - 1;
            if (cur != blank) {
                if (n < cap) {
                    ids[n] = cur;
                    st[n] = t;
                    en[n] = t;
                    cf[n] = conf[r0 + t];
                }
                ++n;
            }
        }
        prev = cur;
    }
    if (n > 0 && n <= cap) en[n - 1] = T - 1;
    tok[(size_t)b * (1 + cap)] = n < cap ? n : cap;
}

// one thread per utterance scans (T' <= a few hundred frames)
__global__ void ctc_collapse_kernel(const int32_t *__restrict__ best, const float *__restrict__ conf,
                                    const int32_t *__restrict__ row_off, int n_utt, int blank, int cap,
                                    int32_t *__restrict__ tok /* [n_utt][1+cap] */,
                                    int32_t *__restrict__ t_start, int32_t *__restrict__ t_end,
                                    float *__restrict__ t_conf) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n_utt) ctc_collapse_row(best, conf, row_off, b, blank, cap, tok, t_start, t_end, t_conf);
}

// ---- phrase-boosted CTC greedy decode (src/phrase_boost.cpp:70-176) ---------------------------------------------
// One block per utterance walks the frames in order (the boosted token set depends on the tokens emitted so far): per
// frame the block marks the children of the active trie states in a bitmap, takes argmax_v(logprob[v] + boost * [v
// marked]) with the first maximum winning (strict '>' scan, :94-102), and thread 0 applies the CTC collapse rules and
// advances the trie on an emission (:40-66: the root stays active, every state that continues with the token moves on).
// Confidence = exp of the UNboosted log-prob (:110).  Every utterance has its own trie and score (trie_row); one whose
// trie is empty takes the plain collapse of the raw arg-max (best, conf), so it decodes exactly as without boosting.
__global__ void __launch_bounds__(256)
ctc_boosted_decode_kernel(const float *__restrict__ logprobs, const int32_t *__restrict__ best, const float *__restrict__ conf,
                          const int32_t *__restrict__ row_off, int V, int blank, int cap,
                          DeviceTrie all_rows, int32_t *__restrict__ tok, int32_t *__restrict__ t_start,
                          int32_t *__restrict__ t_end, float *__restrict__ t_conf) {
    extern __shared__ uint32_t bsm[];
    const int W = (V + 31) >> 5;
    uint32_t *bits = bsm;                                   // [W]
    int *active = reinterpret_cast<int *>(bits + W);        // [BOOST_MAX_ACTIVE]
    int *next = active + BOOST_MAX_ACTIVE;
    __shared__ float red_v[8];
    __shared__ int red_i[8];
    __shared__ int s_nact, s_best;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const TrieRow trie = trie_row(all_rows, b);
    const float boost = trie.boost;
    if (trie.empty()) {
        if (tid == 0) ctc_collapse_row(best, conf, row_off, b, blank, cap, tok, t_start, t_end, t_conf);
        return;
    }
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    int32_t *ids = tok + (size_t)b * (1 + cap) + 1;
    int32_t *st = t_start + (size_t)b * cap, *en = t_end + (size_t)b * cap;
    float *cf = t_conf + (size_t)b * cap;
    if (tid == 0) {
        active[0] = 0;
        s_nact = 1;
    }
    int prev = -1, n = 0;                                   // (thread 0's decode state)
    __syncthreads();
    for (int t = 0; t < T; ++t) {
        const float *row = logprobs + (size_t)(r0 + t) * V;
        for (int w = tid; w < W; w += blockDim.x) bits[w] = 0u;
        __syncthreads();
        const int na = s_nact;
        for (int a = warp; a < na; a += 8) {                // a warp per active state, lanes over its edges
            const int node = active[a];
            for (int e = trie.first[node] + lane; e < trie.first[node + 1]; e += 32) {
                const int tk = trie.tok[e];
                if (tk >= 0 && tk < V) atomicOr(&bits[tk >> 5], 1u << (tk & 31));
            }
        }
        __syncthreads();
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int v = tid; v < V; v += blockDim.x) {
            const float val = row[v] + (((bits[v >> 5] >> (v & 31)) & 1u) ? boost : 0.0f);
            if (val > bv) {
                bv = val;
                bi = v;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) {
                bv = ov;
                bi = oi;
            }
        }
        if (lane == 0) {
            red_v[warp] = bv;
            red_i[warp] = bi;
        }
        __syncthreads();
        if (tid == 0) {
            float fv = red_v[0];
            int fi = red_i[0];
            for (int w2 = 1; w2 < 8; ++w2)
                if (red_v[w2] > fv || (red_v[w2] == fv && red_i[w2] < fi)) {
                    fv = red_v[w2];
                    fi = red_i[w2];
                }
            const int cur = fi;
            if (cur != prev) {
                if (prev != -1 && prev != blank && n > 0 && n <= cap) en[n - 1] = t - 1;
                if (cur != blank) {
                    if (n < cap) {
                        ids[n] = cur;
                        st[n] = t;
                        en[n] = t;
                        cf[n] = expf(row[cur]);
                    }
                    ++n;
                    int nn = 1;
                    next[0] = 0;
                    for (int a = 0; a < na; ++a) {
                        const int node = active[a];
                        for (int e = trie.first[node]; e < trie.first[node + 1]; ++e)
                            if (trie.tok[e] == cur) {
                                const int ch = trie.child[e];
                                bool dup = false;
                                for (int q = 0; q < nn; ++q) dup |= next[q] == ch;
                                if (!dup && nn < BOOST_MAX_ACTIVE) next[nn++] = ch;
                            }
                    }
                    for (int q = 0; q < nn; ++q) active[q] = next[q];
                    s_nact = nn;
                }
            }
            prev = cur;
            s_best = cur;
        }
        __syncthreads();
    }
    if (tid == 0) {
        if (n > 0 && n <= cap) en[n - 1] = T - 1;
        tok[(size_t)b * (1 + cap)] = n < cap ? n : cap;
    }
}

}  // namespace

void launch_ctc_boosted_decode(const float *logprobs, const int32_t *best, const float *conf, const int32_t *row_off, int n_utt, int V, int blank, int cap,
                               const DeviceTrie &trie, int32_t *tok, int32_t *t_start, int32_t *t_end, float *t_conf,
                               cudaStream_t st) {
    const size_t smem = sizeof(uint32_t) * ((V + 31) / 32) + sizeof(int) * 2 * BOOST_MAX_ACTIVE;
    ctc_boosted_decode_kernel<<<dim3(n_utt), dim3(256), smem, st>>>(logprobs, best, conf, row_off, V, blank, cap, trie, tok, t_start, t_end, t_conf);
}

void launch_ctc_frame_argmax(const float *logits, int M, int V, int ld, int32_t *best, float *conf,
                             float *logprobs, cudaStream_t st) {
    if (M <= 0) return;
    ctc_frame_argmax_kernel<<<dim3((M + 7) / 8), dim3(256), 0, st>>>(logits, M, V, ld, best, conf, logprobs);
}

void launch_ctc_collapse(const int32_t *best, const float *conf, const int32_t *row_off, int n_utt, int blank,
                         int cap, int32_t *tok, int32_t *t_start, int32_t *t_end, float *t_conf,
                         cudaStream_t st) {
    ctc_collapse_kernel<<<dim3((n_utt + 63) / 64), dim3(64), 0, st>>>(best, conf, row_off, n_utt, blank, cap, tok, t_start,
                                                        t_end, t_conf);
}

}  // namespace pk
