// attention_tc.cu -- K7 on tensor cores (head_dim 64 and 128): the relative-position attention of
// reference src/encoder.cpp:111-178 (rel_shift :85-109)
//     S[i,j] = ((q_i + u).k_j + (q_i + v).PP[i-j]) / sqrt(hd),  ctx_i = softmax_j(S[i,:]) V
// with every product on mma.sync.m16n8k16 (bf16 inputs, fp32 accumulate) using the same hi/lo
// operand split as the GEMMs (3 MMAs per product: hi.hi + hi.lo + lo.hi), i.e. ~16 mantissa bits,
// and an fp32 online softmax.  wgmma is not used here: per (utterance, head) the matrices are
// 126 x 126 x 64, far below a wgmma tile pipeline's break-even, and the rel_shift needs a per-row
// skew that is natural in registers/shared memory.
//
// Operands: the fused q/k/v projection (EPI_QKV_ACT epilogue of the wgmma GEMM) writes K | V as bf16 hi/lo
// planes [M, 2d] and q as fp32 [M, d]; PP = pos_emb . Wpos^T is split once at load.  K / V / PP-window tiles
// are cp.async'ed (16 B) into shared memory and read through ldmatrix (V through .trans).  The CTA forms
// Qu = q + pos_bias_u and Qv = q + pos_bias_v itself while it builds its Q fragments (one fp32 add and one hi/lo
// split per element, once per CTA) -- when the GEMM epilogue produced both as planes, a q tile cost it four plane
// stores and two passes of maths and the projection GEMM was epilogue-bound (profiles/r02_p_gemm_epilogue.txt).
//
// One CTA = (64-query tile, head, utterance), 4 warps x 16 query rows.  head_dim 64 (tdt-ctc-110m):
// Q fragments live in registers, 93 KB smem -> 2 CTAs per SM (one CTA's tile loads overlap the other's
// MMAs).  head_dim 128 (tdt-600m, config.hpp:98-116): the Qu / Qv tiles are staged in shared memory once
// and read through ldmatrix (128 fragment registers would spill), and the G patch aliases the K tile
// (dead after AC), 209 KB smem -> 1 CTA per SM.  Per 64-key tile a warp does
//   AC  = Qu . K^T                  16 x 64   (8 n-blocks x 4 k-steps x 3 MMAs)
//   G   = Qv . PPwin^T              16 x 80   window of relative positions i-j (10 x 4 x 3 MMAs)
//   S   = AC + skew(G)              G goes through a per-warp smem patch: S[r][jj] += G[r][r+63-jj]
//   online softmax (base 2), P -> bf16 hi/lo A-fragments (C-fragment layout == A-fragment layout)
//   O  += P . V                     16 x 64   (8 x 4 x 3 MMAs)
#include "kernels.h"

namespace pk {
namespace {

constexpr int BQ = 64, BKV = 64;
constexpr int NPW = 128;                               // relative-position window rows per (q-tile, k-tile)
constexpr int LDG_ = 84;                               // G patch row stride (floats)
constexpr int TCA_THREADS = 128;

// LDS_: smem row stride in bf16 (HD + 8: 144 B / 272 B rows, conflict-free ldmatrix)
template <int HD, bool QS>
struct __align__(16) AttnSmem {
    static constexpr int LDS_ = HD + 8;
    bf16 k_hi[BKV * LDS_], k_lo[BKV * LDS_];          // QS: the per-warp G patches alias this tile (dead after AC)
    bf16 v_hi[BKV * LDS_], v_lo[BKV * LDS_];          // [key][dim]; PV reads it through ldmatrix.trans
    bf16 pp_hi[NPW * LDS_], pp_lo[NPW * LDS_];
    float g[QS ? 1 : 4][QS ? 4 : 16 * LDG_];          // QS = false: own G patches
    bf16 q[QS ? 4 : 1][QS ? BQ * LDS_ : 8];           // QS = true: Qu_hi, Qu_lo, Qv_hi, Qv_lo tiles
};
static_assert(sizeof(float) * 4 * 16 * LDG_ <= sizeof(bf16) * 2 * BKV * (128 + 8), "G patches must fit in the K tile");

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// 16-byte async copy; src_bytes = 0 zero-fills the destination (rows outside the utterance / table)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void split2(float x, float y, uint32_t &hi, uint32_t &lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    float2 hf = __bfloat1622float2(h);
    __nv_bfloat162 l = __floats2bfloat162_rn(x - hf.x, y - hf.y);
    hi = *reinterpret_cast<uint32_t *>(&h);
    lo = *reinterpret_cast<uint32_t *>(&l);
}
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// B fragments of two adjacent 8-row n-blocks (rows n0..n0+15 of a row-major [n][LDS_] tile) for the
// 16-wide k-step at k0: r[0], r[1] = (b0, b1) of block n0; r[2], r[3] = (b0, b1) of block n0 + 8.
template <int LDS_>
__device__ __forceinline__ uint32_t bfrag_addr(const bf16 *base, int n0, int k0, int lane) {
    return smem_addr(base + (n0 + ((lane >> 4) << 3) + (lane & 7)) * LDS_ + k0 + (((lane >> 3) & 1) << 3));
}
// A fragment (a0..a3 of m16n8k16) of rows m0..m0+15, k-step at k0 of a row-major [m][LDS_] tile.
template <int LDS_>
__device__ __forceinline__ uint32_t afrag_addr(const bf16 *base, int m0, int k0, int lane) {
    return smem_addr(base + (m0 + (lane & 7) + (((lane >> 3) & 1) << 3)) * LDS_ + k0 + ((lane >> 4) << 3));
}
// Same for B[k][n] = src[k0 + k][n0 + n] (src row-major [k][LDS_]) through ldmatrix.trans:
// r[0], r[1] = (b0, b1) of columns n0..n0+7; r[2], r[3] of columns n0+8..n0+15.
template <int LDS_>
__device__ __forceinline__ uint32_t bfrag_t_addr(const bf16 *base, int k0, int n0, int lane) {
    return smem_addr(base + (k0 + (((lane >> 3) & 1) << 3) + (lane & 7)) * LDS_ + n0 + ((lane >> 4) << 3));
}

template <int HD, bool QS>
__global__ void __launch_bounds__(TCA_THREADS, QS ? 1 : 2)
relpos_attention_tc_kernel(const float *__restrict__ q32, const float *__restrict__ pos_u, const float *__restrict__ pos_v,
                           const bf16 *__restrict__ qkv_hi, const bf16 *__restrict__ qkv_lo, int ld_qkv,
                           const int32_t *__restrict__ row_off, const bf16 *__restrict__ pp_hi,
                           const bf16 *__restrict__ pp_lo, int tmax, int left, int right, int d_model, ActBuf out) {
    extern __shared__ __align__(16) uint8_t smraw[];
    using SM = AttnSmem<HD, QS>;
    constexpr int LDS_ = SM::LDS_, KS = HD / 16, NBO = HD / 8, CH = HD / 8;   // k-steps, output n-blocks, 16 B chunks per row
    SM &sm = *reinterpret_cast<SM *>(smraw);
    const int b = blockIdx.z, h = blockIdx.y;
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    const int i0 = blockIdx.x * BQ;
    if (i0 >= T) return;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const int wrow = warp * 16;          // this warp's first query row inside the tile

    // ---- Q fragments (A operand, rows wrow+g / wrow+g+8, KS k-steps): registers straight from the planes
    // (head_dim 64) or the Qu / Qv tiles staged in shared memory (head_dim 128)
    uint32_t qu_h[QS ? 1 : KS][4], qu_l[QS ? 1 : KS][4], qv_h[QS ? 1 : KS][4], qv_l[QS ? 1 : KS][4];
    constexpr int NQ = QS ? BQ * (HD / 4) / TCA_THREADS : 1;
    float4 qq[NQ];
    float2 qraw[QS ? 1 : KS][4];
    if (!QS) {
        const int ia = i0 + wrow + g, ib = ia + 8;
#pragma unroll
        for (int ks = 0; ks < (QS ? 1 : KS); ++ks)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = (e & 1) ? ib : ia;
                const int col = h * HD + ks * 16 + ((e >> 1) << 3) + 2 * c;
                qraw[ks][e] = make_float2(0.f, 0.f);
                if (row < T) qraw[ks][e] = *reinterpret_cast<const float2 *>(q32 + (size_t)(r0 + row) * d_model + col);
            }
    } else {
        // q rows of this tile: all loads in flight now, consumed after the first key tile's copies have been issued
#pragma unroll
        for (int it = 0; it < NQ; ++it) {
            const int idx = tid + it * TCA_THREADS, i = idx / (HD / 4), c4 = (idx % (HD / 4)) * 4;
            qq[it] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i0 + i < T) qq[it] = *reinterpret_cast<const float4 *>(q32 + (size_t)(r0 + i0 + i) * d_model + h * HD + c4);
        }
    }

    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float oacc[NBO][4];
#pragma unroll
    for (int nb = 0; nb < NBO; ++nb)
#pragma unroll
        for (int e = 0; e < 4; ++e) oacc[nb][e] = 0.f;
    float *gs = QS ? reinterpret_cast<float *>(sm.k_hi) + warp * 16 * LDG_ : sm.g[QS ? 0 : warp];
    const uint32_t sk_hi = smem_addr(sm.k_hi), sk_lo = smem_addr(sm.k_lo), sv_hi = smem_addr(sm.v_hi), sv_lo = smem_addr(sm.v_lo);
    const uint32_t sp_hi = smem_addr(sm.pp_hi), sp_lo = smem_addr(sm.pp_lo);

    // key tiles that meet [i0 - left, i0 + BQ - 1 + right] n [0, T), starting on multiples of BKV: a band that covers the
    // utterance visits the same tiles in the same order as full attention
    const int j_lo = max(i0 - left, 0) / BKV * BKV, j_hi = min(T, i0 + BQ + right);
    for (int j0 = j_lo; j0 < j_hi; j0 += BKV) {
        __syncthreads();                 // previous key tile fully consumed
        // ---- K, V rows j0..j0+63 and the PP window, 16 B per cp.async
        for (int idx = tid; idx < BKV * CH; idx += TCA_THREADS) {
            const int j = idx / CH, ch = idx % CH;
            const bool ok = (j0 + j < T);
            const size_t o = (size_t)(r0 + (ok ? j0 + j : 0)) * ld_qkv + h * HD + ch * 8;      // planes [k | v]
            const uint32_t so = (uint32_t)(j * LDS_ + ch * 8) * 2u;
            const int nb = ok ? 16 : 0;
            cp_async16(sk_hi + so, qkv_hi + o, nb);
            cp_async16(sk_lo + so, qkv_lo + o, nb);
            cp_async16(sv_hi + so, qkv_hi + o + d_model, nb);
            cp_async16(sv_lo + so, qkv_lo + o + d_model, nb);
        }
        const int pmin = i0 - (j0 + BKV - 1);
        for (int idx = tid; idx < NPW * CH; idx += TCA_THREADS) {
            const int w = idx / CH, ch = idx % CH;
            const int prow = pmin + w + tmax - 1;
            const bool ok = (prow >= 0 && prow < 2 * tmax - 1);
            const size_t o = (size_t)(ok ? prow : 0) * d_model + h * HD + ch * 8;
            const uint32_t so = (uint32_t)(w * LDS_ + ch * 8) * 2u;
            const int nb = ok ? 16 : 0;
            cp_async16(sp_hi + so, pp_hi + o, nb);
            cp_async16(sp_lo + so, pp_lo + o, nb);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        if (!QS && j0 == j_lo) {
            // Q fragments: Qu = q + pos_bias_u, Qv = q + pos_bias_v, split hi/lo (rows past T stay zero)
            const int ia = i0 + wrow + g, ib = ia + 8;
#pragma unroll
            for (int ks = 0; ks < (QS ? 1 : KS); ++ks)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int row = (e & 1) ? ib : ia;
                    const int col = h * HD + ks * 16 + ((e >> 1) << 3) + 2 * c;
                    const float2 bu = __ldg(reinterpret_cast<const float2 *>(pos_u + col)), bv = __ldg(reinterpret_cast<const float2 *>(pos_v + col));
                    const float2 qv2 = qraw[ks][e];
                    if (row < T) {
                        split2(qv2.x + bu.x, qv2.y + bu.y, qu_h[ks][e], qu_l[ks][e]);
                        split2(qv2.x + bv.x, qv2.y + bv.y, qv_h[ks][e], qv_l[ks][e]);
                    } else {
                        qu_h[ks][e] = qu_l[ks][e] = qv_h[ks][e] = qv_l[ks][e] = 0u;
                    }
                }
        }
        if (QS && j0 == j_lo) {
            // Qu / Qv tiles (hi, lo) -> shared memory while the first key tile is on its way; visible after the barrier below
#pragma unroll
            for (int it = 0; it < NQ; ++it) {
                const int idx = tid + it * TCA_THREADS, i = idx / (HD / 4), c4 = (idx % (HD / 4)) * 4;
                const bool ok = (i0 + i < T);
                const float4 bu = __ldg(reinterpret_cast<const float4 *>(pos_u + h * HD + c4)), bv = __ldg(reinterpret_cast<const float4 *>(pos_v + h * HD + c4));
                uint2 uh = make_uint2(0u, 0u), ul = uh, vh = uh, vl = uh;
                if (ok) {
                    split2(qq[it].x + bu.x, qq[it].y + bu.y, uh.x, ul.x);
                    split2(qq[it].z + bu.z, qq[it].w + bu.w, uh.y, ul.y);
                    split2(qq[it].x + bv.x, qq[it].y + bv.y, vh.x, vl.x);
                    split2(qq[it].z + bv.z, qq[it].w + bv.w, vh.y, vl.y);
                }
                const int so = i * LDS_ + c4;
                *reinterpret_cast<uint2 *>(sm.q[0] + so) = uh;
                *reinterpret_cast<uint2 *>(sm.q[QS ? 1 : 0] + so) = ul;
                *reinterpret_cast<uint2 *>(sm.q[QS ? 2 : 0] + so) = vh;
                *reinterpret_cast<uint2 *>(sm.q[QS ? 3 : 0] + so) = vl;
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();

        // ---- AC = Qu K^T (16 x 64 per warp)
        float sacc[8][4];
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
#pragma unroll
            for (int e = 0; e < 4; ++e) sacc[nb][e] = 0.f;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            uint32_t ah_[4], al_[4];
            if (QS) {
                ldsm_x4(ah_, afrag_addr<LDS_>(sm.q[0], wrow, ks * 16, lane));
                ldsm_x4(al_, afrag_addr<LDS_>(sm.q[QS ? 1 : 0], wrow, ks * 16, lane));
            }
            const uint32_t (&ah)[4] = QS ? ah_ : qu_h[QS ? 0 : ks];
            const uint32_t (&al)[4] = QS ? al_ : qu_l[QS ? 0 : ks];
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t bh[4], bl[4];
                ldsm_x4(bh, bfrag_addr<LDS_>(sm.k_hi, np * 16, ks * 16, lane));
                ldsm_x4(bl, bfrag_addr<LDS_>(sm.k_lo, np * 16, ks * 16, lane));
                mma_bf16(sacc[2 * np], ah, bh[0], bh[1]);
                mma_bf16(sacc[2 * np + 1], ah, bh[2], bh[3]);
                mma_bf16(sacc[2 * np], ah, bl[0], bl[1]);
                mma_bf16(sacc[2 * np + 1], ah, bl[2], bl[3]);
                mma_bf16(sacc[2 * np], al, bh[0], bh[1]);
                mma_bf16(sacc[2 * np + 1], al, bh[2], bh[3]);
            }
        }
        // ---- G = Qv PPwin^T (16 x 80: window rows wrow .. wrow+79), through the smem patch, skewed into S
        {
            float gacc[10][4];
#pragma unroll
            for (int nb = 0; nb < 10; ++nb)
#pragma unroll
                for (int e = 0; e < 4; ++e) gacc[nb][e] = 0.f;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
                uint32_t ah_[4], al_[4];
                if (QS) {
                    ldsm_x4(ah_, afrag_addr<LDS_>(sm.q[QS ? 2 : 0], wrow, ks * 16, lane));
                    ldsm_x4(al_, afrag_addr<LDS_>(sm.q[QS ? 3 : 0], wrow, ks * 16, lane));
                }
                const uint32_t (&ah)[4] = QS ? ah_ : qv_h[QS ? 0 : ks];
                const uint32_t (&al)[4] = QS ? al_ : qv_l[QS ? 0 : ks];
#pragma unroll
                for (int np = 0; np < 5; ++np) {
                    uint32_t bh[4], bl[4];
                    ldsm_x4(bh, bfrag_addr<LDS_>(sm.pp_hi, wrow + np * 16, ks * 16, lane));
                    ldsm_x4(bl, bfrag_addr<LDS_>(sm.pp_lo, wrow + np * 16, ks * 16, lane));
                    mma_bf16(gacc[2 * np], ah, bh[0], bh[1]);
                    mma_bf16(gacc[2 * np + 1], ah, bh[2], bh[3]);
                    mma_bf16(gacc[2 * np], ah, bl[0], bl[1]);
                    mma_bf16(gacc[2 * np + 1], ah, bl[2], bl[3]);
                    mma_bf16(gacc[2 * np], al, bh[0], bh[1]);
                    mma_bf16(gacc[2 * np + 1], al, bh[2], bh[3]);
                }
            }
            if (QS) __syncthreads();      // every warp has finished AC: the K tile may now hold the G patches
#pragma unroll
            for (int nb = 0; nb < 10; ++nb) {
                *reinterpret_cast<float2 *>(gs + g * LDG_ + nb * 8 + 2 * c) = make_float2(gacc[nb][0], gacc[nb][1]);
                *reinterpret_cast<float2 *>(gs + (g + 8) * LDG_ + nb * 8 + 2 * c) = make_float2(gacc[nb][2], gacc[nb][3]);
            }
            __syncwarp();
            // S[r][jj] += G[r][r + 63 - jj]   (relative position i - j, window column n = w - wrow)
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int jj = nb * 8 + 2 * c + e;
                    sacc[nb][e] += gs[g * LDG_ + g + (BKV - 1) - jj];
                    sacc[nb][2 + e] += gs[(g + 8) * LDG_ + g + 8 + (BKV - 1) - jj];
                }
            __syncwarp();
        }
        // ---- scale (1/sqrt(64), folded with log2 e), mask, online softmax in base 2 (rows g and g+8)
        constexpr float kScale = (HD == 64 ? 0.125f : 0.08838834764831845f) * 1.4426950408889634f;
        static_assert(HD == 64 || HD == 128, "head_dim");
        float alpha[2];
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int i = i0 + wrow + g + hrow * 8;
            float mx = -INFINITY;
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int jj = nb * 8 + 2 * c + e, dij = i - (j0 + jj);
                    float s = sacc[nb][hrow * 2 + e] * kScale;
                    s = (j0 + jj < T && dij <= left && -dij <= right) ? s : -INFINITY;
                    sacc[nb][hrow * 2 + e] = s;
                    mx = fmaxf(mx, s);
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            // Full attention: finite from the first tile on (key j0 is valid).  A band can mask every key a row has seen so
            // far; such a row keeps m = -inf and is shifted by 0 instead: p = ex2(-inf) = 0 and alpha scales l = 0, O = 0.
            const float m_new = fmaxf(m_run[hrow], mx);
            const float m_sh = m_new == -INFINITY ? 0.f : m_new;
            alpha[hrow] = ex2_approx(m_run[hrow] - m_sh);   // ex2(-inf) = 0 on the first tile
            float sum = 0.f;
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float pexp = ex2_approx(sacc[nb][hrow * 2 + e] - m_sh);
                    sacc[nb][hrow * 2 + e] = pexp;
                    sum += pexp;
                }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            l_run[hrow] = l_run[hrow] * alpha[hrow] + sum;
            m_run[hrow] = m_new;
        }
#pragma unroll
        for (int nb = 0; nb < NBO; ++nb) {
            oacc[nb][0] *= alpha[0];
            oacc[nb][1] *= alpha[0];
            oacc[nb][2] *= alpha[1];
            oacc[nb][3] *= alpha[1];
        }
        // ---- O += P V : P's C-fragments of n-blocks (2kk, 2kk+1) are the A-fragment of k-step kk
#pragma unroll
        for (int kk = 0; kk < BKV / 16; ++kk) {
            uint32_t ph[4], pl[4];
            split2(sacc[2 * kk][0], sacc[2 * kk][1], ph[0], pl[0]);
            split2(sacc[2 * kk][2], sacc[2 * kk][3], ph[1], pl[1]);
            split2(sacc[2 * kk + 1][0], sacc[2 * kk + 1][1], ph[2], pl[2]);
            split2(sacc[2 * kk + 1][2], sacc[2 * kk + 1][3], ph[3], pl[3]);
#pragma unroll
            for (int np = 0; np < HD / 16; ++np) {
                uint32_t bh[4], bl[4];
                ldsm_x4_t(bh, bfrag_t_addr<LDS_>(sm.v_hi, kk * 16, np * 16, lane));
                ldsm_x4_t(bl, bfrag_t_addr<LDS_>(sm.v_lo, kk * 16, np * 16, lane));
                mma_bf16(oacc[2 * np], ph, bh[0], bh[1]);
                mma_bf16(oacc[2 * np + 1], ph, bh[2], bh[3]);
                mma_bf16(oacc[2 * np], ph, bl[0], bl[1]);
                mma_bf16(oacc[2 * np + 1], ph, bl[2], bl[3]);
                mma_bf16(oacc[2 * np], pl, bh[0], bh[1]);
                mma_bf16(oacc[2 * np + 1], pl, bh[2], bh[3]);
            }
        }
    }
    // ---- normalise and store ctx[(row), h*HD + dim] (feeds the out_proj GEMM)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
        const int i = i0 + wrow + g + hrow * 8;
        if (i >= T) continue;
        const float inv = 1.0f / l_run[hrow];
#pragma unroll
        for (int nb = 0; nb < NBO; ++nb) {
            const size_t idx = (size_t)(r0 + i) * d_model + h * HD + nb * 8 + 2 * c;
            const float x = oacc[nb][hrow * 2] * inv, y = oacc[nb][hrow * 2 + 1] * inv;
            if (out.f32) *reinterpret_cast<float2 *>(out.f32 + idx) = make_float2(x, y);
            if (out.hi) {
                uint32_t hi, lo;
                split2(x, y, hi, lo);
                *reinterpret_cast<uint32_t *>(out.hi + idx) = hi;
                if (out.lo) *reinterpret_cast<uint32_t *>(out.lo + idx) = lo;
            }
        }
    }
}

}  // namespace

template <int HD, bool QS>
static bool launch_attn_t(const float *q32, const float *pos_u, const float *pos_v, const bf16 *qkv_hi, const bf16 *qkv_lo, int ld_qkv,
                          const int32_t *row_off, int n_utt, int max_T,
                          int n_heads, const bf16 *pp_hi, const bf16 *pp_lo, int tmax, int left, int right, int d_model, ActBuf out,
                          cudaStream_t st) {
    using SM = AttnSmem<HD, QS>;
    static PerDeviceFlag attr_flag;
    bool &attr = attr_flag.cur();
    if (!attr) {
        if (cudaFuncSetAttribute(relpos_attention_tc_kernel<HD, QS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sizeof(SM)) != cudaSuccess)
            return false;
        attr = true;
    }
    dim3 grid((max_T + BQ - 1) / BQ, n_heads, n_utt);
    relpos_attention_tc_kernel<HD, QS><<<dim3(grid), dim3(TCA_THREADS), sizeof(SM), st>>>(q32, pos_u, pos_v, qkv_hi, qkv_lo, ld_qkv, row_off, pp_hi, pp_lo,
                                                                              tmax, left, right, d_model, out);
    return true;
}

bool launch_relpos_attention_tc(const float *q32, const float *pos_u, const float *pos_v, const bf16 *qkv_hi, const bf16 *qkv_lo,
                                int ld_qkv, const int32_t *row_off, int n_utt, int max_T, int n_heads, int head_dim, const bf16 *pp_hi,
                                const bf16 *pp_lo, int tmax, int att_left, int att_right, int d_model, ActBuf out, cudaStream_t st) {
    if (!q32 || !pos_u || !pos_v || !qkv_hi || !qkv_lo || !pp_hi || !pp_lo) return false;
    int left, right;
    if (!attention_band(att_left, att_right, &left, &right)) return false;
    if (head_dim == 64)
        return launch_attn_t<64, false>(q32, pos_u, pos_v, qkv_hi, qkv_lo, ld_qkv, row_off, n_utt, max_T, n_heads, pp_hi, pp_lo, tmax, left, right,
                                        d_model, out, st);
    if (head_dim == 128)
        return launch_attn_t<128, true>(q32, pos_u, pos_v, qkv_hi, qkv_lo, ld_qkv, row_off, n_utt, max_T, n_heads, pp_hi, pp_lo, tmax, left, right,
                                        d_model, out, st);
    return false;
}

}  // namespace pk
