// norm_conv.cu -- K6 LayerNorm and K8 the Conformer depthwise convolution.
//
// K6 layernorm_kernel: nn::LayerNorm / ops::layer_norm (axiom operations.cpp:1796-1809:
//   biased variance, eps inside the sqrt).  One warp per row, the row lives in
//   registers, two passes (mean, then centred second moment) like the reference.
//   Optionally chains a second LayerNorm on the result (ConformerBlock's final_norm_
//   followed by the next block's ffn1_.norm_, src/encoder.cpp:196-204 / :40) so the
//   residual stream is read once.
// K8 dwconv_bn_silu_kernel: ConformerConvModule's depthwise Conv1d (k=9, pad 4, groups=d)
//   + BatchNorm1d(eval) + SiLU (src/encoder.cpp:67-69; BN axiom normalization.cpp:48-104).
//   BatchNorm is folded into the conv weights/bias at load time.  Rows are packed by
//   utterance; taps outside the utterance are zero padding.
#include "kernels.h"

namespace pk {
namespace {

constexpr int LN_MAXV = 8;  // float4 per lane: supports d <= 1024

// Lane `lane` holds float4 number lane + 32 i of the row for i < nv; when d is not a multiple of 128 (Sortformer's d 192:
// 48 float4), the last one exists only on the lanes with lane + 32 i < d / 4.
__device__ __forceinline__ bool ln_has(int i, int nv, int lane, int d) { return i < nv && lane + 32 * i < (d >> 2); }

__device__ __forceinline__ void ln_stats(const float4 *v, int nv, int d, float &mean, float &rstd, float eps) {
    const int lane = threadIdx.x & 31;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (ln_has(i, nv, lane, d)) s += v[i].x + v[i].y + v[i].z + v[i].w;
    mean = warp_sum(s) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (ln_has(i, nv, lane, d)) {
            float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
            q += a * a + b * b + c * c + e * e;
        }
    rstd = rsqrtf(warp_sum(q) / (float)d + eps);
}

__global__ void __launch_bounds__(256)
layernorm_kernel(const float *__restrict__ x, int M, int d, const float *__restrict__ w1,
                 const float *__restrict__ b1, float *out1_f32, ActBuf out1_act,
                 const float *__restrict__ w2, const float *__restrict__ b2, ActBuf out2_act, float eps) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    const int nv = (d + 127) >> 7;  // float4 per lane (the last one partial when d % 128 != 0)
    float4 v[LN_MAXV];
    const float4 *xr = reinterpret_cast<const float4 *>(x + (size_t)row * d);
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (ln_has(i, nv, lane, d)) v[i] = xr[lane + 32 * i];
    float mean, rstd;
    ln_stats(v, nv, d, mean, rstd, eps);
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (ln_has(i, nv, lane, d)) {
            const int c = (lane + 32 * i) * 4;
            const float4 g = *reinterpret_cast<const float4 *>(w1 + c);
            const float4 bb = *reinterpret_cast<const float4 *>(b1 + c);
            v[i].x = (v[i].x - mean) * rstd * g.x + bb.x;
            v[i].y = (v[i].y - mean) * rstd * g.y + bb.y;
            v[i].z = (v[i].z - mean) * rstd * g.z + bb.z;
            v[i].w = (v[i].w - mean) * rstd * g.w + bb.w;
            if (out1_f32) *reinterpret_cast<float4 *>(out1_f32 + (size_t)row * d + c) = v[i];
            store_act4(out1_act, (size_t)row * d + c, v[i]);
        }
    if (w2 == nullptr) return;
    ln_stats(v, nv, d, mean, rstd, eps);
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (ln_has(i, nv, lane, d)) {
            const int c = (lane + 32 * i) * 4;
            const float4 g = *reinterpret_cast<const float4 *>(w2 + c);
            const float4 bb = *reinterpret_cast<const float4 *>(b2 + c);
            float4 y;
            y.x = (v[i].x - mean) * rstd * g.x + bb.x;
            y.y = (v[i].y - mean) * rstd * g.y + bb.y;
            y.z = (v[i].z - mean) * rstd * g.z + bb.z;
            y.w = (v[i].w - mean) * rstd * g.w + bb.w;
            store_act4(out2_act, (size_t)row * d + c, y);
        }
}

// Depthwise conv over time (k = KS, "same" zero padding inside each utterance) + folded BatchNorm +
// SiLU (reference src/encoder.cpp:59-75).  A thread owns 4 channels and DW_TT consecutive frames and
// slides the KS-tap window down the column: DW_TT + KS - 1 float4 loads and one read of its 4 x KS
// taps for DW_TT x 4 outputs (the previous one-frame-per-thread version re-read both 9x).
constexpr int DW_TT = 4;
template <int KS>
__global__ void __launch_bounds__(128)
dwconv_bn_silu_kernel(const float *__restrict__ g, const int32_t *__restrict__ row_off, int d,
                      const float *__restrict__ w /* tap-major [KS][d], BatchNorm folded */, const float *__restrict__ bias /* [d] folded */,
                      ActBuf out) {
    const int b = blockIdx.z;
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    const int t0 = blockIdx.y * DW_TT;
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (t0 >= T || c >= d) return;
    float4 wr[KS];                       // one float4 per tap (4 channels)
#pragma unroll
    for (int j = 0; j < KS; ++j) wr[j] = __ldg(reinterpret_cast<const float4 *>(w + (size_t)j * d + c));
    const float4 bs = *reinterpret_cast<const float4 *>(bias + c);
    float4 win[KS];                      // win[j] = g[t - KS/2 + j]
#pragma unroll
    for (int j = 0; j < KS - 1; ++j) {
        const int tt = t0 - KS / 2 + j;
        win[j + 1] = (tt >= 0 && tt < T) ? *reinterpret_cast<const float4 *>(g + (size_t)(r0 + tt) * d + c)
                                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < DW_TT; ++i) {
        const int t = t0 + i;
        if (t >= T) break;
#pragma unroll
        for (int j = 0; j < KS - 1; ++j) win[j] = win[j + 1];
        const int tn = t + KS / 2;
        win[KS - 1] = (tn < T) ? *reinterpret_cast<const float4 *>(g + (size_t)(r0 + tn) * d + c)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 acc = bs;
#pragma unroll
        for (int j = 0; j < KS; ++j) {   // same tap order as the one-frame version (bit-identical sums)
            acc.x = fmaf(wr[j].x, win[j].x, acc.x);
            acc.y = fmaf(wr[j].y, win[j].y, acc.y);
            acc.z = fmaf(wr[j].z, win[j].z, acc.z);
            acc.w = fmaf(wr[j].w, win[j].w, acc.w);
        }
        store_act4(out, (size_t)(r0 + t) * d + c, make_float4(siluf_(acc.x), siluf_(acc.y), siluf_(acc.z), siluf_(acc.w)));
    }
}

__global__ void split_kernel(const float *__restrict__ x, size_t n4, ActBuf out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n4) store_act4(out, i * 4, reinterpret_cast<const float4 *>(x)[i]);
}

}  // namespace

void launch_split(const float *x, size_t n, ActBuf out, cudaStream_t st) {
    const size_t n4 = n / 4;
    if (n4 == 0) return;
    split_kernel<<<dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, st>>>(x, n4, out);
}

void launch_layernorm(const float *x, int M, int d, const float *w1, const float *b1, float *out1_f32,
                      ActBuf out1_act, const float *w2, const float *b2, ActBuf out2_act, cudaStream_t st) {
    if (M <= 0) return;
    const int warps = 8;
    layernorm_kernel<<<dim3((M + warps - 1) / warps), dim3(warps * 32), 0, st>>>(x, M, d, w1, b1, out1_f32, out1_act, w2, b2,
                                                                     out2_act, 1e-5f);
}

bool launch_dwconv_bn_silu(const float *g, const int32_t *row_off, int n_utt, int max_T, int d, int ks,
                           const float *w, const float *bias, ActBuf out, cudaStream_t st) {
    if (ks != 9) return false;
    dim3 block(128);
    dim3 grid((d / 4 + 127) / 128, (max_T + DW_TT - 1) / DW_TT, n_utt);
    dwconv_bn_silu_kernel<9><<<dim3(grid), dim3(block), 0, st>>>(g, row_off, d, w, bias, out);
    return true;
}

}  // namespace pk
