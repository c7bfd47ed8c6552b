// gemm_skinny.cu -- the GEMM for FEW ROWS (M <= 128): C = epi(A[M,K] . W[N,K]^T + bias) with the same bf16 hi/lo operand
// planes and the same 3-MMA split (hi.hi + hi.lo + lo.hi, fp32 accumulate) as the wgmma kernel (gemm_tc.cu), for the
// launches where that kernel cannot fill the machine: the streaming path (SURVEY.md section 8f row 2) advances S streams by
// 1-2 encoder frames per step, so every encoder GEMM has M = S .. 2S rows -- ONE 128-row tile -- and the persistent
// wgmma grid shrinks to N/128 CTAs (4 for the N = 512 layers) that walk K serially (32 k-blocks for fc2).  Such a
// GEMM is weight-streaming bound: 4 bytes per weight, each read once.
//
// Decomposition: CTA = (32 output columns, one slice of K); the grid is sized to ~2 CTAs per SM by splitting K, so all
// SMs pull disjoint pieces of the weight matrix at once.  Per 64-wide k chunk a CTA copies its 32 x 64 weight tile and
// the M x 64 activation tile (both planes) with 16-byte cp.async into a double-buffered shared-memory stage; 8 warps x
// 16 rows run mma.sync.m16n8k16 (ldmatrix fragments).  K slices meet in a fp32 workspace: the last CTA of a column
// tile to arrive (atomic ticket) adds the slices in slice order -- deterministic -- and applies the fused epilogue
// (pk_common.cuh epilogue4: every EpiKind, edge columns included).
#include "kernels.h"

namespace pk {
namespace {

constexpr int SK_BN = 32, SK_BK = 64, SK_BM = 128, SK_LDS = SK_BK + 8, SK_THREADS = 256;
constexpr int SK_A_ELEMS = SK_BM * SK_LDS, SK_W_ELEMS = SK_BN * SK_LDS;          // one plane of one stage
constexpr size_t SK_SMEM = (size_t)2 * 2 * (SK_A_ELEMS + SK_W_ELEMS) * sizeof(bf16);   // 2 stages x 2 planes = 92 160 B
constexpr int SK_CLD = SK_BN + 4;                                                  // fp32 tile staging stride (aliases the stages)

__device__ __forceinline__ uint32_t sk_smem(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sk_cp16(uint32_t dst, const void *src, int bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sk_ldsm4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void sk_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <bool SPLIT3>
__global__ void __launch_bounds__(SK_THREADS, 2)
gemm_skinny_kernel(const bf16 *__restrict__ Ahi, const bf16 *__restrict__ Alo, int lda, const bf16 *__restrict__ Whi,
                   const bf16 *__restrict__ Wlo, int M, int N, int K, int kc_chunks /* 64-wide chunks per K slice */,
                   float *__restrict__ ws, unsigned int *__restrict__ tickets, const __grid_constant__ EpiParams epi) {
    extern __shared__ __align__(16) uint8_t sk_raw[];
    bf16 *stage = reinterpret_cast<bf16 *>(sk_raw);            // [2 stages][A_hi | A_lo | W_hi | W_lo]
    constexpr int STAGE_ELEMS = 2 * (SK_A_ELEMS + SK_W_ELEMS);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n0 = blockIdx.x * SK_BN, ks = blockIdx.y, nsplit = gridDim.y;
    const int k0 = ks * kc_chunks * SK_BK;
    const int mrows = (M + 15) & ~15;                          // rows that carry data (whole MMA row blocks)

    auto load_chunk = [&](int c, int buf) {
        bf16 *st = stage + (size_t)buf * STAGE_ELEMS;
        const int kk = k0 + c * SK_BK;
        for (int i = tid; i < mrows * 8; i += SK_THREADS) {    // activation rows: 8 x 16 B per row and plane
            const int r = i >> 3, pc = i & 7;
            const bool ok = r < M;
            const size_t o = (size_t)(ok ? r : 0) * lda + kk + pc * 8;
            const uint32_t d = sk_smem(st + r * SK_LDS + pc * 8);
            sk_cp16(d, Ahi + o, ok ? 16 : 0);
            if (SPLIT3) sk_cp16(d + SK_A_ELEMS * 2, Alo + o, ok ? 16 : 0);
        }
        for (int i = tid; i < SK_BN * 8; i += SK_THREADS) {    // weight rows
            const int r = i >> 3, pc = i & 7;
            const bool ok = n0 + r < N;
            const size_t o = (size_t)(ok ? n0 + r : 0) * K + kk + pc * 8;
            const uint32_t d = sk_smem(st + 2 * SK_A_ELEMS + r * SK_LDS + pc * 8);
            sk_cp16(d, Whi + o, ok ? 16 : 0);
            if (SPLIT3) sk_cp16(d + SK_W_ELEMS * 2, Wlo + o, ok ? 16 : 0);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    float acc[4][4];
#pragma unroll
    for (int nb = 0; nb < 4; ++nb) acc[nb][0] = acc[nb][1] = acc[nb][2] = acc[nb][3] = 0.f;
    const bool active = warp * 16 < mrows;                     // warps past the last row block only help with the copies
    load_chunk(0, 0);
    for (int c = 0; c < kc_chunks; ++c) {
        if (c + 1 < kc_chunks) {
            load_chunk(c + 1, (c + 1) & 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        if (active) {
            const bf16 *st = stage + (size_t)(c & 1) * STAGE_ELEMS;
            const bf16 *a_hi = st, *a_lo = st + SK_A_ELEMS, *w_hi = st + 2 * SK_A_ELEMS, *w_lo = w_hi + SK_W_ELEMS;
#pragma unroll
            for (int kk = 0; kk < SK_BK / 16; ++kk) {
                uint32_t ah[4], al[4];
                const int arow = warp * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), acol = kk * 16 + ((lane >> 4) << 3);
                sk_ldsm4(ah, sk_smem(a_hi + arow * SK_LDS + acol));
                if (SPLIT3) sk_ldsm4(al, sk_smem(a_lo + arow * SK_LDS + acol));
#pragma unroll
                for (int np = 0; np < 2; ++np) {               // two n-blocks per ldmatrix.x4
                    uint32_t bh[4], bl[4];
                    const int brow = np * 16 + ((lane >> 4) << 3) + (lane & 7), bcol = kk * 16 + (((lane >> 3) & 1) << 3);
                    sk_ldsm4(bh, sk_smem(w_hi + brow * SK_LDS + bcol));
                    sk_mma(acc[2 * np], ah, bh[0], bh[1]);
                    sk_mma(acc[2 * np + 1], ah, bh[2], bh[3]);
                    if (SPLIT3) {
                        sk_ldsm4(bl, sk_smem(w_lo + brow * SK_LDS + bcol));
                        sk_mma(acc[2 * np], ah, bl[0], bl[1]);
                        sk_mma(acc[2 * np + 1], ah, bl[2], bl[3]);
                        sk_mma(acc[2 * np], al, bh[0], bh[1]);
                        sk_mma(acc[2 * np + 1], al, bh[2], bh[3]);
                    }
                }
            }
        }
        __syncthreads();                                        // the stage may be overwritten by the copy after next
    }

    // ---- this slice's M x 32 tile -> shared memory (fp32, aliases the stages: every copy has landed and been consumed)
    float *ct = reinterpret_cast<float *>(sk_raw);              // [128][SK_CLD]
    if (active) {
        const int g = lane >> 2, cq = lane & 3;
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
            const int r = warp * 16 + g, cidx = nb * 8 + 2 * cq;
            *reinterpret_cast<float2 *>(ct + r * SK_CLD + cidx) = make_float2(acc[nb][0], acc[nb][1]);
            *reinterpret_cast<float2 *>(ct + (r + 8) * SK_CLD + cidx) = make_float2(acc[nb][2], acc[nb][3]);
        }
    }
    __syncthreads();
    __shared__ unsigned int s_last;
    if (nsplit > 1) {
        // partial tile to the workspace [slice][M][N-tile columns], then take a ticket: the last slice to arrive reduces
        float *wp = ws + ((size_t)ks * gridDim.x + blockIdx.x) * (size_t)SK_BM * SK_BN;
        for (int i = tid; i < M * (SK_BN / 4); i += SK_THREADS) {
            const int r = i / (SK_BN / 4), c4 = (i % (SK_BN / 4)) * 4;
            *reinterpret_cast<float4 *>(wp + r * SK_BN + c4) = *reinterpret_cast<const float4 *>(ct + r * SK_CLD + c4);
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const unsigned int t = atomicAdd(&tickets[blockIdx.x], 1u);
            s_last = (t == (unsigned int)nsplit - 1) ? 1u : 0u;
            if (s_last) tickets[blockIdx.x] = 0u;               // ready for the next launch (stream-ordered)
        }
        __syncthreads();
        if (!s_last) return;
        __threadfence();
    }
    // ---- epilogue: 4 consecutive columns of one row per call (GLU pairs / vector stores stay in-thread)
    for (int i = tid; i < M * (SK_BN / 4); i += SK_THREADS) {
        const int r = i / (SK_BN / 4), c4 = (i % (SK_BN / 4)) * 4;
        float4 v;
        if (nsplit > 1) {
            v = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int s2 = 0; s2 < nsplit; ++s2) {               // fixed order: deterministic sums
                const float4 p = __ldcg(reinterpret_cast<const float4 *>(ws + ((size_t)s2 * gridDim.x + blockIdx.x) * (size_t)SK_BM * SK_BN + r * SK_BN + c4));
                v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
            }
        } else {
            v = *reinterpret_cast<const float4 *>(ct + r * SK_CLD + c4);
        }
        epilogue4(epi, r, n0 + c4, N, v);
    }
}

}  // namespace

// Workspace: [max slices][column tiles][128][32] fp32 + one ticket per column tile; allocated by the engine once.
size_t gemm_skinny_ws_floats(int max_n, int max_splits) { return (size_t)max_splits * ((max_n + SK_BN - 1) / SK_BN) * SK_BM * SK_BN; }

cudaError_t launch_gemm_skinny(const bf16 *Ahi, const bf16 *Alo, int lda, const bf16 *Whi, const bf16 *Wlo, int M, int N, int K, bool split3,
                               const EpiParams &epi, float *ws, size_t ws_floats, unsigned int *tickets, int n_tickets, int num_sms,
                               cudaStream_t st) {
    if (M <= 0 || N <= 0) return cudaSuccess;
    if (M > SK_BM || K % SK_BK != 0 || (lda & 7) || !Ahi || !Whi || (split3 && (!Alo || !Wlo))) return cudaErrorInvalidValue;
    const int ntiles = (N + SK_BN - 1) / SK_BN, chunks = K / SK_BK;
    if (ntiles > n_tickets) return cudaErrorInvalidValue;
    // K slices: ~2 CTAs per SM in total, whole chunks per slice, bounded by the workspace
    int nsplit = (2 * num_sms + ntiles - 1) / ntiles;
    if (nsplit > chunks) nsplit = chunks;
    if (nsplit < 1) nsplit = 1;
    while (chunks % nsplit != 0) --nsplit;
    while (nsplit > 1 && (size_t)nsplit * ntiles * SK_BM * SK_BN > ws_floats) {
        --nsplit;
        while (chunks % nsplit != 0) --nsplit;
    }
    static PerDeviceFlag attr_flag;
    bool &attr = attr_flag.cur();
    if (!attr) {
        cudaError_t e1 = cudaFuncSetAttribute(gemm_skinny_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SK_SMEM);
        cudaError_t e2 = cudaFuncSetAttribute(gemm_skinny_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SK_SMEM);
        if (e1 != cudaSuccess || e2 != cudaSuccess) return e1 != cudaSuccess ? e1 : e2;
        attr = true;
    }
    dim3 grid(ntiles, nsplit);
    if (split3)
        gemm_skinny_kernel<true><<<grid, dim3(SK_THREADS), SK_SMEM, st>>>(Ahi, Alo, lda, Whi, Wlo, M, N, K, chunks / nsplit, ws, tickets, epi);
    else
        gemm_skinny_kernel<false><<<grid, dim3(SK_THREADS), SK_SMEM, st>>>(Ahi, Alo, lda, Whi, Wlo, M, N, K, chunks / nsplit, ws, tickets, epi);
    return cudaGetLastError();
}

}  // namespace pk
