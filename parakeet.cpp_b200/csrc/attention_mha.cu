// attention_mha.cu -- plain multi-head self-attention of the Sortformer transformer (reference src/transformer.cpp:15-50):
//     ctx_i = softmax_j((q_i . k_j) / sqrt(hd)) v_j      per head, keys j of the query's own utterance only
// No position term, no mask (Sortformer::forward passes none).  The scale is applied to the dot product, as the reference
// scales the score matrix (transformer.cpp:38).
//
// Two forms, head_dim 24 (Sortformer: d 192, 8 heads) only:
//  * mha_tc_kernel (bf16x3 / bf16x1): mma.sync m16n8k16 on bf16 hi / lo operand splits (hi*hi + hi*lo + lo*hi with
//    split3, hi*hi alone otherwise), fp32 accumulation and an fp32 online softmax.  Input as the EPI_QKV_ACT epilogue lays
//    it out: q fp32 [M][d], k | v bf16 planes [M][2 d].  One CTA of 4 warps per (64-query tile, head, utterance), 16 query
//    rows per warp; head_dim is zero-padded to 32 in shared memory (two k-steps of 16) for S = Q K^T, and V is stored
//    transposed so that P V takes P straight from the S accumulators (flash-attention register reuse).
//  * mha_kernel (PK_MATH_FP32): fp32 CUDA cores.  Input fp32 q | k | v [M][3 d].
// fp32 form: one CTA per (query tile, head, utterance),
// one thread per query row holding q and the output accumulator in registers.  Key / value tiles of the utterance stream
// through shared memory (every thread reads the same key: broadcast loads); the softmax is online, rescaled once per chunk
// of MHA_CH keys.  Both write ctx [M][d] as the out_proj GEMM's operand (fp32 or bf16 hi / lo planes).
#include "kernels.h"

namespace pk {
namespace {

constexpr int MHA_BQ = 64;    // query rows per CTA (= threads)
constexpr int MHA_BK = 64;    // keys per shared-memory tile
constexpr int MHA_CH = 16;    // keys per softmax rescale

template <int HD>
__global__ void __launch_bounds__(MHA_BQ)
mha_kernel(const float *__restrict__ qkv, int ld_qkv, const int32_t *__restrict__ row_off, int d_model, float scale, ActBuf out) {
    static_assert(HD % 4 == 0, "float4 rows");
    constexpr int V4 = HD / 4;
    __shared__ __align__(16) float Ks[MHA_BK][HD];
    __shared__ __align__(16) float Vs[MHA_BK][HD];
    const int b = blockIdx.z, h = blockIdx.y;
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    const int i0 = blockIdx.x * MHA_BQ;
    if (i0 >= T) return;
    const int tid = threadIdx.x, i = i0 + tid;
    const bool live = i < T;

    float q[HD], o[HD];
#pragma unroll
    for (int c = 0; c < V4; ++c) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live) v = *reinterpret_cast<const float4 *>(qkv + (size_t)(r0 + i) * ld_qkv + h * HD + 4 * c);
        q[4 * c] = v.x; q[4 * c + 1] = v.y; q[4 * c + 2] = v.z; q[4 * c + 3] = v.w;
    }
#pragma unroll
    for (int c = 0; c < HD; ++c) o[c] = 0.f;
    float m = -INFINITY, l = 0.f;

    for (int j0 = 0; j0 < T; j0 += MHA_BK) {
        __syncthreads();   // previous tile consumed
        for (int idx = tid; idx < MHA_BK * V4; idx += MHA_BQ) {
            const int j = idx / V4, c = idx % V4;
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (j0 + j < T) {
                const float *row = qkv + (size_t)(r0 + j0 + j) * ld_qkv + h * HD + 4 * c;
                kv = *reinterpret_cast<const float4 *>(row + d_model);
                vv = *reinterpret_cast<const float4 *>(row + 2 * d_model);
            }
            *reinterpret_cast<float4 *>(&Ks[j][4 * c]) = kv;
            *reinterpret_cast<float4 *>(&Vs[j][4 * c]) = vv;
        }
        __syncthreads();
        const int nk = min(MHA_BK, T - j0);
        for (int jc = 0; jc < nk; jc += MHA_CH) {
            float s[MHA_CH];
            float cmax = -INFINITY;
#pragma unroll
            for (int u = 0; u < MHA_CH; ++u) {
                float dot = 0.f;
#pragma unroll
                for (int c = 0; c < HD; ++c) dot = fmaf(q[c], Ks[jc + u][c], dot);
                s[u] = (jc + u < nk) ? dot * scale : -INFINITY;
                cmax = fmaxf(cmax, s[u]);
            }
            const float m_new = fmaxf(m, cmax);    // finite: the chunk holds at least one key
            const float corr = expf(m - m_new);    // 0 on the first chunk (m = -inf)
            l *= corr;
#pragma unroll
            for (int c = 0; c < HD; ++c) o[c] *= corr;
#pragma unroll
            for (int u = 0; u < MHA_CH; ++u) {
                const float p = expf(s[u] - m_new);   // 0 for keys past the utterance (s = -inf)
                l += p;
#pragma unroll
                for (int c = 0; c < HD; ++c) o[c] = fmaf(p, Vs[jc + u][c], o[c]);
            }
            m = m_new;
        }
    }
    if (!live) return;
    const float inv = 1.0f / l;
#pragma unroll
    for (int c = 0; c < V4; ++c)
        store_act4(out, (size_t)(r0 + i) * d_model + h * HD + 4 * c,
                   make_float4(o[4 * c] * inv, o[4 * c + 1] * inv, o[4 * c + 2] * inv, o[4 * c + 3] * inv));
}

// ---------------------------------------------------------------- tensor-core form
constexpr int TC_BQ = 64, TC_BK = 64, TC_HDP = 32;       // query rows, keys per tile, padded head_dim
constexpr int TC_LD = TC_HDP + 8;                        // smem row stride (bf16) of Q / K: conflict-free fragment loads
constexpr int TC_LDV = TC_BK + 8;                        // smem row stride (bf16) of V^T

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&v);
}
__device__ __forceinline__ void split_pair(float a, float b, uint32_t &hi, uint32_t &lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    const float2 f = __bfloat1622float2(h);
    hi = *reinterpret_cast<uint32_t *>(&h);
    lo = pack_bf16(a - f.x, b - f.y);
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <bool SPLIT3>
__global__ void __launch_bounds__(128)
mha_tc_kernel(const float *__restrict__ q32, const bf16 *__restrict__ kv_hi, const bf16 *__restrict__ kv_lo, int ld_kv,
              const int32_t *__restrict__ row_off, int d_model, float scale, ActBuf out) {
    constexpr int HD = 24;
    __shared__ __align__(16) bf16 Qs[2][TC_BQ][TC_LD];    // [hi | lo][row][dim], dims 24..31 zero
    __shared__ __align__(16) bf16 Ks[2][TC_BK][TC_LD];    // [hi | lo][key][dim]
    __shared__ __align__(16) bf16 Vt[2][HD][TC_LDV];      // [hi | lo][dim][key]
    const int b = blockIdx.z, h = blockIdx.y;
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    const int i0 = blockIdx.x * TC_BQ;
    if (i0 >= T) return;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const bf16 z = __float2bfloat16(0.f);

    for (int idx = tid; idx < TC_BQ * TC_HDP; idx += 128) {
        const int i = idx / TC_HDP, c = idx % TC_HDP;
        float v = 0.f;
        if (c < HD && i0 + i < T) v = q32[(size_t)(r0 + i0 + i) * d_model + h * HD + c];
        const bf16 hv = __float2bfloat16_rn(v);
        Qs[0][i][c] = hv;
        Qs[1][i][c] = __float2bfloat16_rn(v - __bfloat162float(hv));
    }
    for (int idx = tid; idx < 2 * TC_BK * (TC_HDP - HD); idx += 128) {   // K's padding columns stay zero
        const int p = idx / (TC_BK * (TC_HDP - HD)), r = idx % (TC_BK * (TC_HDP - HD));
        Ks[p][r / (TC_HDP - HD)][HD + r % (TC_HDP - HD)] = z;
    }
    __syncthreads();
    uint32_t qa[2][2][4];                                 // [hi | lo][k-step][fragment]
    const int qr = warp * 16;
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const int c = ks * 16 + 2 * t4;
            qa[p][ks][0] = *reinterpret_cast<const uint32_t *>(&Qs[p][qr + g][c]);
            qa[p][ks][1] = *reinterpret_cast<const uint32_t *>(&Qs[p][qr + g + 8][c]);
            qa[p][ks][2] = *reinterpret_cast<const uint32_t *>(&Qs[p][qr + g][c + 8]);
            qa[p][ks][3] = *reinterpret_cast<const uint32_t *>(&Qs[p][qr + g + 8][c + 8]);
        }
    float o[3][4] = {};
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // rows g, g + 8 (l: this thread's partial)

    for (int j0 = 0; j0 < T; j0 += TC_BK) {
        __syncthreads();                                  // previous tile consumed
        for (int idx = tid; idx < TC_BK * HD; idx += 128) {
            const int j = idx / HD, c = idx % HD;
            bf16 kh = z, kl = z, vh = z, vl = z;
            if (j0 + j < T) {
                const size_t base = (size_t)(r0 + j0 + j) * ld_kv + h * HD + c;
                kh = kv_hi[base];
                vh = kv_hi[base + d_model];
                if (SPLIT3) { kl = kv_lo[base]; vl = kv_lo[base + d_model]; }
            }
            Ks[0][j][c] = kh; Ks[1][j][c] = kl;
            Vt[0][c][j] = vh; Vt[1][c][j] = vl;
        }
        __syncthreads();
        const int nk = min(TC_BK, T - j0);
        float s[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const int key = nt * 8 + g, c = ks * 16 + 2 * t4;
                const uint32_t bh0 = *reinterpret_cast<const uint32_t *>(&Ks[0][key][c]);
                const uint32_t bh1 = *reinterpret_cast<const uint32_t *>(&Ks[0][key][c + 8]);
                mma16816(s[nt], qa[0][ks], bh0, bh1);
                if (SPLIT3) {
                    const uint32_t bl0 = *reinterpret_cast<const uint32_t *>(&Ks[1][key][c]);
                    const uint32_t bl1 = *reinterpret_cast<const uint32_t *>(&Ks[1][key][c + 8]);
                    mma16816(s[nt], qa[0][ks], bl0, bl1);
                    mma16816(s[nt], qa[1][ks], bh0, bh1);
                }
            }
        }
        // online softmax per row: this thread holds keys nt*8 + 2 t4 + {0, 1} of rows g (s[.][0..1]) and g + 8 (s[.][2..3])
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = nt * 8 + 2 * t4 + (e & 1);
                s[nt][e] = key < nk ? s[nt][e] * scale : -INFINITY;
                mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
            }
        float corr[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float mn = fmaxf(m[r], mx[r]);         // finite: the tile holds at least one key
            corr[r] = expf(m[r] - mn);
            m[r] = mn;
            l[r] *= corr[r];
        }
#pragma unroll
        for (int nt = 0; nt < 3; ++nt) {
            o[nt][0] *= corr[0]; o[nt][1] *= corr[0]; o[nt][2] *= corr[1]; o[nt][3] *= corr[1];
        }
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                s[nt][e] = expf(s[nt][e] - m[e >> 1]);   // 0 for masked keys
                l[e >> 1] += s[nt][e];
            }
        // O += P V over the 4 key steps of 16
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            uint32_t ph[4], pl[4];
            split_pair(s[2 * kk][0], s[2 * kk][1], ph[0], pl[0]);
            split_pair(s[2 * kk][2], s[2 * kk][3], ph[1], pl[1]);
            split_pair(s[2 * kk + 1][0], s[2 * kk + 1][1], ph[2], pl[2]);
            split_pair(s[2 * kk + 1][2], s[2 * kk + 1][3], ph[3], pl[3]);
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                const int dim = nt * 8 + g, key = kk * 16 + 2 * t4;
                const uint32_t vh0 = *reinterpret_cast<const uint32_t *>(&Vt[0][dim][key]);
                const uint32_t vh1 = *reinterpret_cast<const uint32_t *>(&Vt[0][dim][key + 8]);
                mma16816(o[nt], ph, vh0, vh1);
                if (SPLIT3) {
                    const uint32_t vl0 = *reinterpret_cast<const uint32_t *>(&Vt[1][dim][key]);
                    const uint32_t vl1 = *reinterpret_cast<const uint32_t *>(&Vt[1][dim][key + 8]);
                    mma16816(o[nt], ph, vl0, vl1);
                    mma16816(o[nt], pl, vh0, vh1);
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int i = i0 + qr + g + 8 * r;
        if (i >= T) continue;
        const float inv = 1.0f / l[r];
#pragma unroll
        for (int nt = 0; nt < 3; ++nt) {
            const size_t idx = (size_t)(r0 + i) * d_model + h * HD + nt * 8 + 2 * t4;
            store_act(out, idx, o[nt][2 * r] * inv);
            store_act(out, idx + 1, o[nt][2 * r + 1] * inv);
        }
    }
}

}  // namespace

bool launch_mha_attention(const float *qkv, int ld_qkv, const int32_t *row_off, int n_utt, int max_T, int n_heads, int head_dim,
                          int d_model, ActBuf out, cudaStream_t st) {
    if (head_dim != 24 || n_heads * head_dim != d_model || ld_qkv < 3 * d_model || (ld_qkv & 3) || n_utt <= 0) return false;
    if (max_T <= 0) return true;
    const float scale = 1.0f / std::sqrt((float)head_dim);   // transformer.cpp:27
    dim3 grid((max_T + MHA_BQ - 1) / MHA_BQ, n_heads, n_utt);
    mha_kernel<24><<<grid, dim3(MHA_BQ), 0, st>>>(qkv, ld_qkv, row_off, d_model, scale, out);
    return cudaGetLastError() == cudaSuccess;
}

}  // namespace pk

namespace pk {

bool launch_mha_attention_tc(const float *q32, const bf16 *kv_hi, const bf16 *kv_lo, int ld_kv, const int32_t *row_off, int n_utt, int max_T,
                             int n_heads, int head_dim, int d_model, ActBuf out, cudaStream_t st) {
    if (head_dim != 24 || n_heads * head_dim != d_model || ld_kv < 2 * d_model || !kv_hi || n_utt <= 0) return false;
    if (max_T <= 0) return true;
    const float scale = 1.0f / std::sqrt((float)head_dim);   // transformer.cpp:27
    dim3 grid((max_T + TC_BQ - 1) / TC_BQ, n_heads, n_utt);
    if (kv_lo) mha_tc_kernel<true><<<grid, dim3(128), 0, st>>>(q32, kv_hi, kv_lo, ld_kv, row_off, d_model, scale, out);
    else mha_tc_kernel<false><<<grid, dim3(128), 0, st>>>(q32, kv_hi, kv_lo, ld_kv, row_off, d_model, scale, out);
    return cudaGetLastError() == cudaSuccess;
}

}  // namespace pk
