// attention.cu -- K7: relative-position multi-head self-attention core.
//
// Replaces ConformerAttention::rel_position_attention between the q/k/v and out
// projections (reference src/encoder.cpp:111-178) including rel_shift (:85-109):
//     AC[i,j] = (q_i + u_h) . k_j
//     BD[i,j] = rel_shift((q + v_h) P^T)[i,j] = (q_i + v_h) . PP[i - j]
//     ctx_i   = softmax_j((AC + BD) / sqrt(hd)) V
// rel_shift never wraps for 0 <= i,j < T (SURVEY.md section 7), so the shifted score is
// the dot product with the projected position embedding of RELATIVE POSITION i-j.
// PP[p] = pos_proj_(emb(p)) depends only on p (emb(p)[2k] = sin(p w_k), [2k+1] = cos(p w_k),
// encoder.cpp:9-30), not on T, so one table per layer covers every utterance length:
// `pp` is [(2*Tmax-1), d] with row (p + Tmax - 1).  Nothing of shape (T, 2T-1) is ever
// materialised.  No mask: Transcriber never passes one (transcribe.hpp:108); keys beyond
// the utterance's own length are excluded, which is what batch=1 in the reference means.
//
// Limited context (rel_pos_local_attn, DESIGN.md section 16): with a band (left, right) query i
// attends to key j only when -right <= i - j <= left; the softmax runs over the keys that remain.
// A query tile visits only the key tiles that meet [i0 - left, i0 + BQ - 1 + right], starting on
// multiples of BKV, and masks per element inside them.  The table then needs only the relative
// positions -W..W (W = max(left, right), tmax = W + 1); window rows outside it are zero-filled and
// every score that would read them is masked.  The launchers map the band (0, 0) to full attention.
//
// fp32 CUDA-core flash-style kernel: one CTA per (query tile, head, utterance); key tiles
// stream through shared memory with an online softmax; 4x4 register blocking; operands
// are stored transposed ([k][row]) so the inner loop uses float4 shared loads.
#include "kernels.h"

namespace pk {
namespace {

template <int HD, int BQ, int BKV>
struct AttnCfg {
    static constexpr int TX = BKV / 4, TY = BQ / 4, THREADS = TX * TY;
    static constexpr int LQ = BQ + 4, LK = BKV + 4;   // padded leading dims (floats)
    static constexpr int NP = BQ + BKV;               // relative positions per tile pair (+1 pad)
    static constexpr int LP = NP + 4;
    static constexpr int CPT = HD / TX;               // output columns per thread
    static constexpr size_t SMEM = sizeof(float) * (2 * HD * LQ + HD * LK + BKV * HD + HD * LP + BKV * LQ);
};

template <int HD, int BQ, int BKV>
__global__ void __launch_bounds__(AttnCfg<HD, BQ, BKV>::THREADS)
relpos_attention_kernel(const float *__restrict__ qkv, int ld_qkv, const int32_t *__restrict__ row_off,
                        const float *__restrict__ pp, int tmax, const float *__restrict__ bias_u,
                        const float *__restrict__ bias_v, int left, int right, int d_model, ActBuf out) {
    using C = AttnCfg<HD, BQ, BKV>;
    extern __shared__ __align__(16) float sm[];
    float *Qu_t = sm;                      // [HD][LQ]
    float *Qv_t = Qu_t + HD * C::LQ;       // [HD][LQ]
    float *K_t = Qv_t + HD * C::LQ;        // [HD][LK]
    float *V_s = K_t + HD * C::LK;         // [BKV][HD]
    float *PP_t = V_s + BKV * HD;          // [HD][LP], column = p - pmin
    float *P_t = PP_t + HD * C::LP;        // [BKV][LQ]  softmax numerators, transposed

    const int b = blockIdx.z, h = blockIdx.y;
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    const int i0 = blockIdx.x * BQ;
    if (i0 >= T) return;
    const int tid = threadIdx.x, tx = tid % C::TX, ty = tid / C::TX;
    const float scale = rsqrtf((float)HD);

    // ---- load the query tile once: Qu = q + u_h, Qv = q + v_h (transposed)
    for (int idx = tid; idx < BQ * HD; idx += C::THREADS) {
        const int i = idx / HD, k = idx % HD;
        float q = 0.f;
        if (i0 + i < T) q = qkv[(size_t)(r0 + i0 + i) * ld_qkv + h * HD + k];
        Qu_t[k * C::LQ + i] = q + bias_u[h * HD + k];
        Qv_t[k * C::LQ + i] = q + bias_v[h * HD + k];
    }

    float m_run[4], l_run[4], o[4][C::CPT];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        m_run[a] = -INFINITY;
        l_run[a] = 0.f;
#pragma unroll
        for (int c = 0; c < C::CPT; ++c) o[a][c] = 0.f;
    }

    const int j_lo = max(i0 - left, 0) / BKV * BKV, j_hi = min(T, i0 + BQ + right);
    for (int j0 = j_lo; j0 < j_hi; j0 += BKV) {
        __syncthreads();  // previous tile fully consumed (also orders the Q stores on first pass)
        // ---- K (transposed), V (natural), PP window (transposed)
        for (int idx = tid; idx < BKV * HD; idx += C::THREADS) {
            const int j = idx / HD, k = idx % HD;
            float kv = 0.f, vv = 0.f;
            if (j0 + j < T) {
                const float *row = qkv + (size_t)(r0 + j0 + j) * ld_qkv + h * HD + k;
                kv = row[d_model];
                vv = row[2 * d_model];
            }
            K_t[k * C::LK + j] = kv;
            V_s[j * HD + k] = vv;
        }
        const int pmin = i0 - (j0 + BKV - 1);  // smallest relative position in this tile pair
        for (int idx = tid; idx < C::NP * HD; idx += C::THREADS) {
            const int pi = idx / HD, k = idx % HD;
            const int prow = pmin + pi + tmax - 1;
            float v = 0.f;
            if (prow >= 0 && prow < 2 * tmax - 1) v = pp[(size_t)prow * d_model + h * HD + k];
            PP_t[k * C::LP + pi] = v;
        }
        __syncthreads();

        // ---- scores for the 4x4 block: rows ty*4+a, keys tx*4+bb
        float s[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int bb = 0; bb < 4; ++bb) s[a][bb] = 0.f;
        // p - pmin for (a, bb) = 4*(ty - tx) + (a - bb) + (BKV - 1); a-bb = -3 -> multiple of 4
        const int pbase = 4 * (ty - tx) + BKV - 4;
#pragma unroll 4
        for (int k = 0; k < HD; ++k) {
            const float4 qu = *reinterpret_cast<const float4 *>(Qu_t + k * C::LQ + ty * 4);
            const float4 qv = *reinterpret_cast<const float4 *>(Qv_t + k * C::LQ + ty * 4);
            const float4 kk = *reinterpret_cast<const float4 *>(K_t + k * C::LK + tx * 4);
            const float4 p0 = *reinterpret_cast<const float4 *>(PP_t + k * C::LP + pbase);
            const float4 p1 = *reinterpret_cast<const float4 *>(PP_t + k * C::LP + pbase + 4);
            const float qa[4] = {qu.x, qu.y, qu.z, qu.w};
            const float qb[4] = {qv.x, qv.y, qv.z, qv.w};
            const float kb[4] = {kk.x, kk.y, kk.z, kk.w};
            const float pv[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int bb = 0; bb < 4; ++bb) {
                    s[a][bb] = fmaf(qa[a], kb[bb], s[a][bb]);
                    s[a][bb] = fmaf(qb[a], pv[a - bb + 3], s[a][bb]);  // index = (p - pmin) - pbase
                }
        }
        // ---- online softmax (row statistics across the TX threads that share a row)
        float alpha[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            float mx = -INFINITY;
#pragma unroll
            for (int bb = 0; bb < 4; ++bb) {
                const int j = j0 + tx * 4 + bb, dij = i0 + ty * 4 + a - j;
                const bool valid = j < T && dij <= left && -dij <= right;
                s[a][bb] = valid ? s[a][bb] * scale : -INFINITY;
                mx = fmaxf(mx, s[a][bb]);
            }
#pragma unroll
            for (int off = C::TX / 2; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float m_new = fmaxf(m_run[a], mx);
            alpha[a] = (m_run[a] == -INFINITY) ? 0.f : expf(m_run[a] - m_new);
            float sum = 0.f;
#pragma unroll
            for (int bb = 0; bb < 4; ++bb) {
                const float e = (s[a][bb] == -INFINITY) ? 0.f : expf(s[a][bb] - m_new);
                s[a][bb] = e;
                sum += e;
            }
#pragma unroll
            for (int off = C::TX / 2; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
            l_run[a] = l_run[a] * alpha[a] + sum;
            m_run[a] = m_new;
        }
#pragma unroll
        for (int bb = 0; bb < 4; ++bb)
            *reinterpret_cast<float4 *>(P_t + (tx * 4 + bb) * C::LQ + ty * 4) =
                make_float4(s[0][bb], s[1][bb], s[2][bb], s[3][bb]);
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int c = 0; c < C::CPT; ++c) o[a][c] *= alpha[a];
        __syncthreads();
        // ---- O += P V : rows ty*4+a, columns tx*4 + BKV*m + cc
#pragma unroll 4
        for (int j = 0; j < BKV; ++j) {
            const float4 pj = *reinterpret_cast<const float4 *>(P_t + j * C::LQ + ty * 4);
            const float pa[4] = {pj.x, pj.y, pj.z, pj.w};
#pragma unroll
            for (int m = 0; m < C::CPT / 4; ++m) {
                const float4 vv = *reinterpret_cast<const float4 *>(V_s + j * HD + tx * 4 + BKV * m);
                const float vb[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int cc = 0; cc < 4; ++cc) o[a][m * 4 + cc] = fmaf(pa[a], vb[cc], o[a][m * 4 + cc]);
            }
        }
    }
    // ---- normalise and store ctx[(row), h*HD + col] (feeds the out_proj GEMM)
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int i = i0 + ty * 4 + a;
        if (i >= T) continue;
        const float inv = 1.0f / l_run[a];
#pragma unroll
        for (int m = 0; m < C::CPT / 4; ++m) {
            const size_t idx = (size_t)(r0 + i) * d_model + h * HD + tx * 4 + BKV * m;
            store_act4(out, idx,
                       make_float4(o[a][m * 4 + 0] * inv, o[a][m * 4 + 1] * inv, o[a][m * 4 + 2] * inv,
                                   o[a][m * 4 + 3] * inv));
        }
    }
}

template <int HD, int BQ, int BKV>
void launch_t(const float *qkv, int ld_qkv, const int32_t *row_off, int n_utt, int max_T, int n_heads,
              const float *pp, int tmax, const float *bu, const float *bv, int left, int right, int d_model, ActBuf out,
              cudaStream_t st) {
    using C = AttnCfg<HD, BQ, BKV>;
    static PerDeviceFlag attr_flag;
    bool &attr_set = attr_flag.cur();
    if (!attr_set) {
        cudaFuncSetAttribute(relpos_attention_kernel<HD, BQ, BKV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)C::SMEM);
        attr_set = true;
    }
    dim3 grid((max_T + BQ - 1) / BQ, n_heads, n_utt);
    relpos_attention_kernel<HD, BQ, BKV><<<dim3(grid), dim3(C::THREADS), C::SMEM, st>>>(qkv, ld_qkv, row_off, pp, tmax, bu,
                                                                           bv, left, right, d_model, out);
}

}  // namespace

bool launch_relpos_attention(const float *qkv, int ld_qkv, const int32_t *row_off, int n_utt, int max_T,
                             int n_heads, int head_dim, const float *pp, int tmax, int att_left, int att_right,
                             const float *bu, const float *bv, int d_model, ActBuf out, cudaStream_t st) {
    int left, right;
    if (!attention_band(att_left, att_right, &left, &right)) return false;
    if (head_dim == 64) {
        launch_t<64, 64, 64>(qkv, ld_qkv, row_off, n_utt, max_T, n_heads, pp, tmax, bu, bv, left, right, d_model, out, st);
    } else if (head_dim == 128) {
        launch_t<128, 64, 32>(qkv, ld_qkv, row_off, n_utt, max_T, n_heads, pp, tmax, bu, bv, left, right, d_model, out, st);
    } else {
        return false;
    }
    return true;
}

}  // namespace pk
