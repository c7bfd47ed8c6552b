// subsample.cu -- K3/K4: the convolutional front of ConvSubsampling::forward
// (reference src/encoder.cpp:219-241; conv2d semantics axiom operations.cpp:3133-3326:
// cross-correlation, zero padding, L_out = (L + 2p - k)/s + 1).
//
// Layout is channels-last and packed by utterance: a stage tensor is
// [(utterance, t, f), C] fp32 rows, so the 1x1 convolutions conv2_/conv3_ are plain
// GEMMs over those rows and the final permute(0,2,1,3)+reshape (encoder.cpp:236-238)
// is free (proj_ weight columns are permuted at load time instead).
//
// K3 subsample_conv1_dw1_kernel: conv1_ (1->C, 3x3, s2, p1) + ReLU + dw1_ (depthwise
//   3x3, s2, p1) fused; the (C, t1, f1) conv1 activation (20 MB per 10 s clip) never
//   touches HBM.  Feature rows are staged in shared memory once per tile (line
//   buffer); each thread owns one channel and slides a 3-column window along f.
// K4 subsample_dw_kernel: depthwise 3x3 s2 p1 on channels-last rows (dw2_).
#include "kernels.h"

namespace pk {
namespace {

constexpr int TT2 = 4;  // t2 rows per block

__global__ void __launch_bounds__(256)
subsample_conv1_dw1_kernel(const float *__restrict__ feats, const int32_t *__restrict__ frame_off,
                           const int32_t *__restrict__ s2_off, int mel, int C,
                           const float *__restrict__ w1, const float *__restrict__ b1,
                           const float *__restrict__ wd, const float *__restrict__ bd, ActBuf out) {
    extern __shared__ float S[];  // [(4*TT2+3)][mel + 4], column index = col + 2
    const int b = blockIdx.y;
    const int F = frame_off[b + 1] - frame_off[b];
    const int t1n = (F - 1) / 2 + 1, f1n = (mel - 1) / 2 + 1;
    const int t2n = (t1n - 1) / 2 + 1, f2n = (f1n - 1) / 2 + 1;
    const int r0 = blockIdx.x * TT2;
    if (r0 >= t2n) return;
    const int stride = mel + 4;
    constexpr int NROWS = 4 * TT2 + 3;      // feature rows 4*r0-3 .. 4*r0+4*TT2-1
    constexpr int NQ = 2 * TT2 + 1;         // conv1 rows 2*r0-1 .. 2*r0+2*TT2-1, shared by the TT2 outputs
    const int row_base = 4 * r0 - 3;        // feature row of S[0]
    const float *src = feats + (size_t)frame_off[b] * mel;
    for (int i = threadIdx.x; i < NROWS * stride; i += blockDim.x) {
        const int rr = i / stride, cc = i - rr * stride - 2;
        const int fr = row_base + rr;
        S[i] = (fr >= 0 && fr < F && cc >= 0 && cc < mel) ? src[(size_t)fr * mel + cc] : 0.f;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float W1[9], WD[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) {
            W1[i] = w1[c * 9 + i];
            WD[i] = wd[c * 9 + i];
        }
        const float B1 = b1[c], BD = bd[c];
        bool rv[NQ];  // conv1 row validity (zero padding of dw1's input)
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
            const int t1 = 2 * r0 - 1 + q;
            rv[q] = (t1 >= 0 && t1 < t1n);
        }
        // walk along the frequency axis; conv1 values of the NQ rows at column f1 are computed once and
        // feed every output row that needs them (a t2-outer loop computes each shared row twice)
        float colprev[NROWS];
#pragma unroll
        for (int r = 0; r < NROWS; ++r) colprev[r] = S[r * stride + 1];  // col -1 (zero pad)
        float p2[NQ], p1[NQ], cur[NQ];
#pragma unroll
        for (int q = 0; q < NQ; ++q) p2[q] = p1[q] = 0.f;
        for (int f1 = 0; f1 < 2 * f2n; ++f1) {
            float2 nw[NROWS];
#pragma unroll
            for (int r = 0; r < NROWS; ++r) nw[r] = *reinterpret_cast<const float2 *>(S + r * stride + 2 * f1 + 2);
            const bool fv = f1 < f1n;
#pragma unroll
            for (int q = 0; q < NQ; ++q) {
                float v = B1;
#pragma unroll
                for (int pp = 0; pp < 3; ++pp) {
                    v = fmaf(W1[pp * 3 + 0], colprev[2 * q + pp], v);
                    v = fmaf(W1[pp * 3 + 1], nw[2 * q + pp].x, v);
                    v = fmaf(W1[pp * 3 + 2], nw[2 * q + pp].y, v);
                }
                cur[q] = (rv[q] && fv) ? fmaxf(v, 0.f) : 0.f;
            }
            if (f1 & 1) {
#pragma unroll
                for (int tt = 0; tt < TT2; ++tt) {
                    const int t2 = r0 + tt;
                    if (t2 < t2n) {
                        float acc = BD;
#pragma unroll
                        for (int i = 0; i < 3; ++i) {
                            acc = fmaf(WD[i * 3 + 0], p2[2 * tt + i], acc);
                            acc = fmaf(WD[i * 3 + 1], p1[2 * tt + i], acc);
                            acc = fmaf(WD[i * 3 + 2], cur[2 * tt + i], acc);
                        }
                        store_act(out, (((size_t)s2_off[b] + (size_t)t2) * f2n + (f1 >> 1)) * C + c, acc);
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < NQ; ++q) {
                p2[q] = p1[q];
                p1[q] = cur[q];
            }
#pragma unroll
            for (int r = 0; r < NROWS; ++r) colprev[r] = nw[r].y;
        }
    }
}

// in: [(in_off[b] + t*fin + f), C] fp32; out: [(out_off[b] + t'*fout + f'), C]
__global__ void subsample_dw_kernel(const float *__restrict__ in, const int32_t *__restrict__ in_rows,
                                    const int32_t *__restrict__ in_off,
                                    const int32_t *__restrict__ out_off, int fin, int C,
                                    const float *__restrict__ wd /* tap-major [9][C] */,
                                    const float *__restrict__ bd, ActBuf out, int total_out_rows,
                                    int n_utt) {
    // one thread per (output row, 4 channels)
    const int c4n = C >> 2;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long orow = gid / c4n;
    if (orow >= total_out_rows) return;
    const int c = (int)(gid - orow * c4n) * 4;
    const int fout = (fin - 1) / 2 + 1;
    // locate the utterance (out_off is a prefix array in units of rows = t' * fout)
    int lo = 0, hi = n_utt - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if ((long long)out_off[mid] * fout <= orow) lo = mid; else hi = mid - 1;
    }
    const int b = lo;
    const int tin = in_rows[b];
    const long long local = orow - (long long)out_off[b] * fout;
    const int to = (int)(local / fout), fo = (int)(local - (long long)to * fout);
    float4 acc = *reinterpret_cast<const float4 *>(bd + c);
    const float *base = in + (size_t)in_off[b] * fin * C;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const int ti = 2 * to - 1 + i;
        if (ti < 0 || ti >= tin) continue;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int fi = 2 * fo - 1 + j;
            if (fi < 0 || fi >= fin) continue;
            const float4 x = *reinterpret_cast<const float4 *>(base + ((size_t)ti * fin + fi) * C + c);
            const float4 wk = __ldg(reinterpret_cast<const float4 *>(wd + (size_t)(i * 3 + j) * C + c));   // (was 4 scalar loads per tap)
            acc.x = fmaf(wk.x, x.x, acc.x);
            acc.y = fmaf(wk.y, x.y, acc.y);
            acc.z = fmaf(wk.z, x.z, acc.z);
            acc.w = fmaf(wk.w, x.w, acc.w);
        }
    }
    store_act4(out, (size_t)orow * C + c, acc);
}

}  // namespace

void launch_subsample_conv1_dw1(const float *feats, const int32_t *frame_off, const int32_t *s2_off,
                                int n_utt, int max_t2, int mel, int C, const float *w1, const float *b1,
                                const float *wd, const float *bd, ActBuf out, cudaStream_t st) {
    dim3 grid((max_t2 + TT2 - 1) / TT2, n_utt);
    int threads = ((C + 31) / 32) * 32;
    if (threads > 256) threads = 256;            // the kernel strides over channels
    size_t smem = sizeof(float) * (4 * TT2 + 3) * (mel + 4);
    subsample_conv1_dw1_kernel<<<dim3(grid), dim3(threads), smem, st>>>(feats, frame_off, s2_off, mel, C, w1, b1, wd, bd,
                                                            out);
}

void launch_subsample_dw(const float *in, const int32_t *in_rows, const int32_t *in_off,
                         const int32_t *out_off, int n_utt, int fin, int C, const float *wd,
                         const float *bd, ActBuf out, int total_out_rows, cudaStream_t st) {
    long long n = (long long)total_out_rows * (C / 4);
    int threads = 256;
    subsample_dw_kernel<<<dim3((unsigned)((n + threads - 1) / threads)), dim3(threads), 0, st>>>(
        in, in_rows, in_off, out_off, fin, C, wd, bd, out, total_out_rows, n_utt);
}

}  // namespace pk
