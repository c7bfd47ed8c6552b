// ctc_align.cu -- CTC forced alignment of a known token sequence (PK_DECODER_CTC_ALIGN; DESIGN.md section 15 is the
// definition this file implements, tests/ctc_align_oracle.py its float64 restatement).
//
//   ctc_align_kernel : one CTA per utterance walks its frames over the CTC trellis of the extended target sequence
//                      z = (blank, y_1, blank, ..., y_L, blank), S = 2L + 1 states, threads over the states.  Per frame it
//                      takes the Viterbi step (max over s, s-1, s-2; ties to s, then s-1) and the forward step
//                      (log-sum-exp), both in double, and writes one back-pointer byte per state.  One thread then traces
//                      the best path back and writes each frame's label and exp(log-prob) into best / conf, the layout
//                      of ctc_frame_argmax_kernel, so the unchanged greedy collapse (ctc.cu) turns the path into tokens.
//
// The Viterbi score adds the same fp32 log-probs in the same order as the float64 oracle, so it is bit-identical to it.
#include "../../include/parakeet_b200.h"
#include "kernels.h"

namespace pk {
namespace {

__device__ __forceinline__ double lse3(double a, double b, double c) {
    const double m = fmax(a, fmax(b, c));
    if (m == -INFINITY) return -INFINITY;
    return m + log(exp(a - m) + exp(b - m) + exp(c - m));
}

__global__ void __launch_bounds__(CTC_ALIGN_THREADS)
ctc_align_kernel(const float *__restrict__ logprobs, const int32_t *__restrict__ row_off, int V, const int32_t *__restrict__ tgt,
                 const int32_t *__restrict__ tgt_off, uint8_t *__restrict__ bp, int bp_stride, int32_t *__restrict__ best,
                 float *__restrict__ conf, double *__restrict__ score, double *__restrict__ loglik, int32_t *__restrict__ path) {
    extern __shared__ double dsm[];
    __shared__ int s_rep;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    const int t0 = tgt_off[b], L = tgt_off[b + 1] - t0, S = 2 * L + 1;
    const int blank = V - 1;
    double *dv = dsm, *al = dsm + 2 * S;                  // [2][S] each: frame t in half t & 1
    int *y = reinterpret_cast<int *>(dsm + 4 * S);
    if (tid == 0) s_rep = 0;
    __syncthreads();
    int rep = 0;
    for (int i = tid; i < L; i += blockDim.x) {
        y[i] = tgt[t0 + i];
        rep += i + 1 < L && tgt[t0 + i] == tgt[t0 + i + 1];
    }
    if (rep) atomicAdd(&s_rep, rep);
    __syncthreads();
    const float *lp = logprobs + (size_t)r0 * V;
    bool feasible = T >= L + s_rep;
    double vit = T == 0 && feasible ? 0.0 : -INFINITY, fwd = vit;
    int end = S - 1;
    if (feasible && T > 0) {
        for (int s = tid; s < S; s += blockDim.x) {
            const double x = s < 2 ? (double)lp[(s & 1) ? y[0] : blank] : -INFINITY;
            dv[s] = x;
            al[s] = x;
        }
        __syncthreads();
        for (int t = 1; t < T; ++t) {
            const size_t h = (size_t)(t & 1) * S, g = (size_t)S - h;   // this frame's half, the previous frame's
            const double *dp = dv + g, *ap = al + g;
            double *dc = dv + h, *ac = al + h;
            const float *row = lp + (size_t)t * V;
            uint8_t *bpr = bp + (size_t)(r0 + t) * bp_stride;
            for (int s = tid; s < S; s += blockDim.x) {
                const int k = s >> 1;
                const bool skip = (s & 1) && s >= 3 && y[k] != y[k - 1];   // z_s is a token unlike z_{s-2}
                const double x = (double)row[(s & 1) ? y[k] : blank];
                double m = dp[s];
                int arg = 0;
                if (s >= 1 && dp[s - 1] > m) { m = dp[s - 1]; arg = 1; }
                if (skip && dp[s - 2] > m) { m = dp[s - 2]; arg = 2; }
                dc[s] = x + m;
                bpr[s] = (uint8_t)arg;
                ac[s] = x + lse3(ap[s], s >= 1 ? ap[s - 1] : -INFINITY, skip ? ap[s - 2] : -INFINITY);
            }
            __syncthreads();
        }
        const double *dl = dv + (size_t)((T - 1) & 1) * S, *alast = al + (size_t)((T - 1) & 1) * S;
        vit = dl[S - 1];
        if (S >= 2 && dl[S - 2] > vit) {
            vit = dl[S - 2];
            end = S - 2;
        }
        fwd = S >= 2 ? lse3(alast[S - 1], alast[S - 2], -INFINITY) : alast[0];
        feasible = vit != -INFINITY;        // every path has probability 0: reported as an infeasible row
    }
    if (tid != 0) return;
    score[b] = feasible ? vit : -INFINITY;
    loglik[b] = feasible ? fwd : -INFINITY;
    for (int t = T - 1, s = end; t >= 0; --t) {
        const int lab = feasible ? ((s & 1) ? y[s >> 1] : blank) : blank;
        best[r0 + t] = lab;
        conf[r0 + t] = expf(lp[(size_t)t * V + lab]);
        if (path) path[r0 + t] = feasible ? s : -1;
        if (feasible && t > 0) s -= bp[(size_t)(r0 + t) * bp_stride + s];
    }
}

}  // namespace

size_t ctc_align_smem_bytes() {
    const size_t S = 2 * (size_t)PK_ALIGN_MAX_TOKENS + 1;
    return 4 * S * sizeof(double) + (size_t)PK_ALIGN_MAX_TOKENS * sizeof(int);
}

void launch_ctc_align(const float *logprobs, const int32_t *row_off, int n_utt, int V, const int32_t *tgt, const int32_t *tgt_off,
                      uint8_t *bp, int bp_stride, int32_t *best, float *conf, double *score, double *loglik, int32_t *path,
                      cudaStream_t st) {
    static PerDeviceFlag attr_flag;
    bool &attr_set = attr_flag.cur();
    const size_t smem = ctc_align_smem_bytes();
    if (!attr_set) {
        cudaFuncSetAttribute(ctc_align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr_set = true;
    }
    ctc_align_kernel<<<dim3(n_utt), dim3(CTC_ALIGN_THREADS), smem, st>>>(logprobs, row_off, V, tgt, tgt_off, bp, bp_stride,
               best, conf, score, loglik, path);
}

}  // namespace pk
