// gemm_tc.cu -- K5: the tensor-core GEMM of the encoder, hand-written for sm_90a:
//     C = epi(A[M,K] . W[N,K]^T + bias)
// TMA (cp.async.bulk.tensor, SWIZZLE_128B) -> shared-memory stages -> wgmma (m64 x BN x k16, bf16 operands straight
// from shared memory, fp32 accumulator in registers) -> fused epilogue from registers (pk_common.cuh: bias / ReLU /
// SiLU / GLU / residual, output either fp32 or the bf16 hi/lo operand planes of the next GEMM).
//
// Arithmetic (pk_math): operands are bf16 hi/lo SPLITS of the fp32 values
// (hi = rn_bf16(x), lo = rn_bf16(x - hi); weights split once at load, activations split by
// the producing kernel's epilogue).  PK_MATH_BF16X3 issues three MMAs per product,
//     A_hi.W_hi + A_hi.W_lo + A_lo.W_hi      (fp32 accumulate)
// which keeps ~16 mantissa bits -- the reference is an fp32 CPU build and parity is token-identical.
// PK_MATH_BF16X1 issues only A_hi.W_hi.
//
// Structure (persistent, one CTA per SM, 384 threads = three warpgroups, static round-robin tile schedule, n-tile
// fastest so that concurrently running CTAs share the same A rows through L2):
//   warpgroup 0     TMA producer : one elected thread waits empty[s], arms full[s] with the byte count and issues the
//                                  2 or 4 tile loads of k-block kb into stage s; it runs ahead across tiles
// The default kernel (gemm_tc_kernel) is PING-PONG: the producer hands most of its registers to the consumers
// (setmaxnreg), and each consumer warpgroup owns whole 128 x BN tiles, the CTA's tiles alternating between the two:
//   warpgroups 1-2  consumers    : wait for their turn (named barrier), then per k-block wait full[s], 4 x 2 x (1|3)
//                                  wgmma (rows 0-63 and 64-127, same B operand), commit; one wgmma group stays in flight
//                                  and the stage of the previous k-block is released (empty[s], one arrival per warp)
//                                  once it has retired; after the last k-block is issued the other warpgroup's turn
//                                  begins, and this one runs the epilogue under the other's wgmma
// The ping-pong epilogue is STAGED when the launcher can describe every output with a TMA map (N and ldo multiples of 4,
// 16-B aligned bases and pitches, qcols a multiple of 64): the warpgroup applies epi_math in the fragment layout, writes
// 64-row x 128-B chunks (SWIZZLE_128B) into its two chunk buffers and stores each with one TMA store of whole rows;
// RESID_F32 loads its residual chunk by TMA into the same buffer.  Otherwise it writes from registers (epilogue_regs).
// The cluster form (gemm_tc_cl_kernel) keeps the COOPERATIVE body (gemm_tc_body): both consumer warpgroups work on one
// tile (rows [64 (wg - 1), 64 wg)) and run its epilogue together, which their cluster-wide barriers need.
// Every spin-wait is bounded and traps, so a protocol bug is an error, not a hung GPU.
#include <cuda.h>

#include "kernels.h"
#include "tc_prims.cuh"

namespace pk {
namespace {

using namespace tc;

constexpr int TC_THREADS = 384;
constexpr int CONSUMER_WARPS = 8;

// The staged epilogue of the ping-pong kernel writes its output in chunks of 64 rows x 128 B (32 fp32 or 64 bf16 columns),
// each consumer warpgroup into its own two chunk buffers, and stores them with TMA.
constexpr int CHUNK_ROWS = 64, CHUNK_BYTES = CHUNK_ROWS * 128;

template <int BN, int NPASS, bool STAGED = false>
struct TcCfg {
    static constexpr int A_BYTES = BM * BK * 2;                 // one plane, 16 KB
    static constexpr int W_BYTES = BN * BK * 2;
    static constexpr int PLANES = (NPASS == 3) ? 2 : 1;
    static constexpr int STAGE_BYTES = PLANES * (A_BYTES + W_BYTES);
    static constexpr int EPI_BYTES = STAGED ? 2 * 2 * CHUNK_BYTES : 0;   // staged epilogue: 2 consumers x 2 chunk buffers
    static constexpr int AVAIL = 227 * 1024 - EPI_BYTES - 1024 - 256;
    static constexpr int STAGES = AVAIL / STAGE_BYTES > 8 ? 8 : AVAIL / STAGE_BYTES;
    static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + EPI_BYTES + 1024 /*align*/ + 256 /*barriers*/;
    static_assert(STAGES >= 2, "pipeline depth");
    static_assert(SMEM <= 227 * 1024, "shared memory per CTA");
    static_assert((2 * STAGES + (STAGED ? 4 : 0)) * 8 <= 256, "barrier space");
};

// Epilogue of one consumer warpgroup: its 64 x BN accumulator slab, rows row0.., columns n0...  Lanes t and t ^ 1 swap
// the row-(r + 8) pair of one and the row-r pair of the other, so every lane holds 4 consecutive columns of one row --
// the unit every epilogue kind works on (GLU pairs stay in-thread, vector stores).
template <int BN, int EK>
__device__ __forceinline__ void epilogue_regs(const float (&d)[BN / 2], const EpiParams &epi_param, int row0, int n0, int M, int N, int lane) {
    const EpiParams epi = epi_param;
    const int q = lane & 3;
    const int row = row0 + (lane >> 2) + ((q & 1) ? 8 : 0);
    const bool vec_ok = ((epi.ldo & 3) == 0) && ((N & 3) == 0);
    // The loads (bias, residual) of G column groups are issued before any of their stores: a load cannot be moved above
    // an earlier store by the compiler (out_f32 may alias resid), so one group at a time would wait out one memory
    // round trip per group.
    constexpr int G = 4;
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += G) {
        float4 b[G], r[G];
#pragma unroll
        for (int g = 0; g < G; ++g) {
            const int col = n0 + 8 * (j0 + g) + 4 * (q >> 1);
            b[g] = r[g] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (row < M && vec_ok && col + 4 <= N) {
                if (epi.bias) b[g] = __ldg(reinterpret_cast<const float4 *>(epi.bias + col));
                if (EK == EPI_RESID_F32) r[g] = *reinterpret_cast<const float4 *>(epi.resid + (size_t)row * epi.ldo + col);
            }
        }
#pragma unroll
        for (int g = 0; g < G; ++g) {
            const int j = j0 + g;
            // even lane: keeps its row-r pair, receives the partner's row-r pair; odd lane: the row-(r + 8) pairs
            const float s0 = (q & 1) ? d[4 * j] : d[4 * j + 2], s1 = (q & 1) ? d[4 * j + 1] : d[4 * j + 3];
            const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
            if (row >= M) continue;
            float4 v = (q & 1) ? make_float4(r0, r1, d[4 * j + 2], d[4 * j + 3]) : make_float4(d[4 * j], d[4 * j + 1], r0, r1);
            const int col = n0 + 8 * j + 4 * (q >> 1);
            if (vec_ok && col + 4 <= N) epi_store<EK>(epi, row, col, epi_math<EK>(v, b[g], r[g], epi.alpha));
            else epilogue4(epi_param, row, col, N, v);
        }
    }
}

// keeps the compiler from moving accesses of the accumulator registers across wgmma issue / wait
template <int N>
__device__ __forceinline__ void fence_operands(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---------------------------------------------------------------------------------------------- staged epilogue
// The ping-pong kernel's epilogue when every output of the launch can be written by TMA (launch_gemm_tc decides): each
// consumer warpgroup applies epi_math to its 64 x BN accumulator slabs in the wgmma fragment layout (thread t holds the
// column pairs 8 j + 2 (t % 4) of rows 16 (t / 32) + (t % 32) / 4 and + 8, and a GLU pair is such a column pair), writes
// the result chunk by chunk into shared memory and stores each chunk with one TMA store of whole rows.  Every element sees
// the same fp32 operations as in epilogue_regs, so the two write the same bytes.
//
// Tensor maps of the outputs: out = fp32 (out_f32, the act.f32 plane, or q [M, qcols] of QKV), hi / lo = the bf16 planes,
// resid = the residual input of RESID_F32 (loaded chunk by chunk by TMA into the chunk buffer it is then stored from).
struct EpiMaps {
    CUtensorMap out, hi, lo, resid;
};

constexpr uint32_t EPI_BAR = 3;         // named barrier EPI_BAR + cw: the 128 threads of consumer warpgroup cw

// Shared-memory stores and loads of the chunk buffers (32-bit shared addresses).
__device__ __forceinline__ void sts_f2(uint32_t a, float x, float y) { asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory"); }
__device__ __forceinline__ void sts_f1(uint32_t a, float x) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(x) : "memory"); }
__device__ __forceinline__ void sts_b2(uint32_t a, __nv_bfloat162 h) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(*reinterpret_cast<uint32_t *>(&h)) : "memory"); }
__device__ __forceinline__ float2 lds_f2(uint32_t a) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
    return v;
}

// One consumer warpgroup's chunk buffers.  Chunk c of the warpgroup goes to buffer c % 2.  Before the barrier of chunk c
// the leader waits until the store of chunk c - 1 has read its buffer, so after that barrier buffer (c + 1) % 2 is free.
//
// A chunk is a 64-row x 128-B box stored with SWIZZLE_128B: the 16-B unit u of row r sits at unit u ^ (r % 8), so the 8
// rows a warp writes at once fall in 8 different bank groups.  The thread of fragment rows rl, rl + 8 and column pair
// 8 j + 2 q writes fp32 pairs at byte 32 j + 8 q of its rows and bf16 pairs (or one GLU result) at byte 16 j + 4 q: the
// unit index of j enters by XOR, so an address is (buffer + b32) ^ 32 j, or (buffer + b16) ^ 16 j, and + 1024 for row rl + 8.
// The warpgroup's thread-dependent values are recomputed from threadIdx where they are used: the accumulators of two
// slabs leave the epilogue few registers to keep them in.
struct Stager {
    uint32_t buf;           // shared address of this warpgroup's 2 x CHUNK_BYTES, 1024-B aligned
    uint32_t cnt;           // chunks stored so far
    __device__ __forceinline__ static bool leader() { return (threadIdx.x & 127) == 0; }   // issues the TMA operations
    // this thread's byte offset of column pair 0 in row rl of a chunk: fp32 pairs (b32) and bf16 pairs / GLU results (b16)
    __device__ __forceinline__ static uint32_t b32() {
        const uint32_t t = threadIdx.x & 127, rl = ((t >> 5) << 4) + ((t & 31) >> 2), q = t & 3;
        return rl * 128u + ((((q >> 1) ^ rl) & 7u) << 4) + 8u * (q & 1u);
    }
    __device__ __forceinline__ static uint32_t b16() {
        const uint32_t t = threadIdx.x & 127, rl = ((t >> 5) << 4) + ((t & 31) >> 2), q = t & 3;
        return rl * 128u + ((rl & 7u) << 4) + 4u * q;
    }
    __device__ __forceinline__ uint32_t cur() const { return buf + (cnt & 1u) * CHUNK_BYTES; }
    // the mbarrier of the residual load into buffer b: the 4 of the CTA follow both warpgroups' buffers
    __device__ __forceinline__ uint32_t rbar(uint32_t b) const {
        const uint32_t cw = (threadIdx.x >> 7) - 1;
        return buf + (2u - cw) * 2u * CHUNK_BYTES + 16u * cw + 8u * b;
    }
    // loads the residual chunk at (c0, r0) into the buffer of chunk cnt + ahead (leader; that buffer is free)
    __device__ __forceinline__ void load(const CUtensorMap *tm, uint32_t ahead, int c0, int r0) const {
        const uint32_t b = (cnt + ahead) & 1u;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(rbar(b)), "r"(CHUNK_BYTES) : "memory");
        asm volatile(
            "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
            ::"r"(buf + b * CHUNK_BYTES), "l"(reinterpret_cast<uint64_t>(tm)), "r"(rbar(b)), "r"(c0), "r"(r0)
            : "memory");
    }
    __device__ __forceinline__ void wait_loaded() const { mbar_wait(rbar(cnt & 1u), (cnt >> 1) & 1u); }
    // after this thread's writes of chunk cnt: hand the chunk to TMA
    __device__ __forceinline__ void store(const CUtensorMap *tm, int c0, int r0) {
        fence_proxy_async_smem();
        if (leader()) bulk_wait_read<0>();
        __syncwarp();
        bar_sync(EPI_BAR + (threadIdx.x >> 7) - 1, 128);
        if (leader()) {
            tma_store_2d(tm, cur(), c0, r0);
            bulk_commit();
        }
        __syncwarp();
        ++cnt;
    }
    // Both buffers at once, for the hi and lo planes of the same columns (each value is read once, for both planes):
    // drain() waits until every store has read its buffer; store_pair() then stores the chunks written to cur() and
    // nxt().  A chunk that follows a pair starts with drain() again.
    __device__ __forceinline__ uint32_t nxt() const { return buf + ((cnt + 1u) & 1u) * CHUNK_BYTES; }
    __device__ __forceinline__ void drain() const {
        if (leader()) bulk_wait_read<0>();
        __syncwarp();
        bar_sync(EPI_BAR + (threadIdx.x >> 7) - 1, 128);
    }
    __device__ __forceinline__ void store_pair(const CUtensorMap *tm0, const CUtensorMap *tm1, int c0, int r0) {
        fence_proxy_async_smem();
        __syncwarp();
        bar_sync(EPI_BAR + (threadIdx.x >> 7) - 1, 128);
        if (leader()) {
            tma_store_2d(tm0, cur(), c0, r0);
            tma_store_2d(tm1, nxt(), c0, r0);
            bulk_commit();
        }
        __syncwarp();
        cnt += 2;
    }
};

// epi_math in place on the NJ column groups j0.. of a slab, in the fragment layout: (d[4 j], d[4 j + 1]) = row r,
// columns c, c + 1 and (d[4 j + 2], d[4 j + 3]) = row r + 8; for GLU the results of rows r and r + 8 land in d[4 j] and
// d[4 j + 1].  RESID_F32 gets its bias add here and the rest of epi_math in resid_chunk.  Applied chunk by chunk, just
// before the chunk is written, so that no more than one chunk's transient values sit beside the accumulators; the bias is
// read with a volatile load so that the compiler does not keep one slab's bias in registers for the other slab.
template <int BN, int EK, int NJ>
__device__ __forceinline__ void epi_chunk(float (&d)[BN / 2], int j0, const EpiParams &epi, int n0, int N) {
    constexpr int MK = EK == EPI_RESID_F32 ? EPI_BIAS_F32 : EK;
    const int q = threadIdx.x & 3;
#pragma unroll
    for (int jj = 0; jj < NJ; ++jj) {
        const int j = j0 + jj, col = n0 + 8 * j + 2 * q;
        float2 b = make_float2(0.f, 0.f);
        if (epi.bias && col < N)
            asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(b.x), "=f"(b.y) : "l"(epi.bias + col));
        const float4 v = epi_math<MK>(make_float4(d[4 * j], d[4 * j + 1], d[4 * j + 2], d[4 * j + 3]), make_float4(b.x, b.y, b.x, b.y),
                                      make_float4(0.f, 0.f, 0.f, 0.f), epi.alpha);
        d[4 * j] = v.x; d[4 * j + 1] = v.y; d[4 * j + 2] = v.z; d[4 * j + 3] = v.w;
    }
}

// chunk writers: slab columns 8 j0 .. 8 j0 + 31 (fp32) or + 63 (bf16, GLU) of the thread's rows
template <int BN>
__device__ __forceinline__ void put_f32(const Stager &sg, const float (&d)[BN / 2], int j0) {
    const uint32_t a = sg.cur() + Stager::b32();
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
        const int j = j0 + jj;
        sts_f2(a ^ (32u * jj), d[4 * j], d[4 * j + 1]);
        sts_f2((a ^ (32u * jj)) + 1024u, d[4 * j + 2], d[4 * j + 3]);
    }
}
// bf16 planes: hi into cur(), and with LO the lo plane (the split of store_act4: lo = rn(v - hi)) into nxt()
template <int BN, bool LO>
__device__ __forceinline__ void put_bf16(const Stager &sg, const float (&d)[BN / 2], int j0) {
    const uint32_t a = sg.cur() + Stager::b16(), al = sg.nxt() + Stager::b16();
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
        const int j = j0 + jj;
        const __nv_bfloat162 h0 = __floats2bfloat162_rn(d[4 * j], d[4 * j + 1]), h1 = __floats2bfloat162_rn(d[4 * j + 2], d[4 * j + 3]);
        sts_b2(a ^ (16u * jj), h0);
        sts_b2((a ^ (16u * jj)) + 1024u, h1);
        if (LO) {
            const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
            sts_b2(al ^ (16u * jj), __floats2bfloat162_rn(d[4 * j] - f0.x, d[4 * j + 1] - f0.y));
            sts_b2((al ^ (16u * jj)) + 1024u, __floats2bfloat162_rn(d[4 * j + 2] - f1.x, d[4 * j + 3] - f1.y));
        }
    }
}
template <int BN>
__device__ __forceinline__ void put_glu(const Stager &sg, const float (&d)[BN / 2], int j0) {
    const uint32_t a = sg.cur() + Stager::b16();
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {        // 64 interleaved columns -> 32 output columns
        const int j = j0 + jj;
        sts_f1(a ^ (16u * jj), d[4 * j]);
        sts_f1((a ^ (16u * jj)) + 1024u, d[4 * j + 1]);
    }
}

// RESID_F32 on one 32-column chunk whose residual the buffer holds, d = acc + bias: out = resid + alpha d (epi_math's
// expression), in place
template <int BN>
__device__ __forceinline__ void resid_chunk(const Stager &sg, const float (&d)[BN / 2], int j0, float alpha) {
    const uint32_t a = sg.cur() + Stager::b32();
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
        const int j = j0 + jj;
        const uint32_t p0 = a ^ (32u * jj), p1 = p0 + 1024u;
        const float2 r0 = lds_f2(p0), r1 = lds_f2(p1);
        sts_f2(p0, r0.x + alpha * d[4 * j], r0.y + alpha * d[4 * j + 1]);
        sts_f2(p1, r1.x + alpha * d[4 * j + 2], r1.y + alpha * d[4 * j + 3]);
    }
}

// The staged epilogue of one 64-row slab (rows row0.., columns n0..) of a consumer warpgroup.  For RESID_F32 the load of
// the slab's first chunk has been issued; each chunk issues the load of the next one (next_row >= 0: the next slab's
// first chunk follows this slab's last).
template <int BN, int EK>
__device__ __forceinline__ void epilogue_staged(float (&d)[BN / 2], const EpiParams &epi, const EpiMaps &om, Stager &sg, int row0,
                                                int n0, int N, int next_row) {
    constexpr int NCH = BN / 32, NG = BN / 64;      // 32-column fp32 chunks, 64-column groups
    // stores the chunk; the fence keeps the compiler from converting the values of later chunks ahead of this one, which
    // would hold them in registers next to the accumulators
    auto store = [&](const CUtensorMap *tm, int c0, int r0) {
        sg.store(tm, c0, r0);
        fence_operands(d);
    };
    if constexpr (EK == EPI_RESID_F32) {
#pragma unroll
        for (int s = 0; s < NCH; ++s) {
            const int c0 = n0 + 32 * s;
            if (c0 >= N) break;
            if (Stager::leader()) {
                bulk_wait_read<0>();        // chunk cnt - 1's store has read the buffer the next load goes to
                if (s + 1 < NCH && c0 + 32 < N) sg.load(&om.resid, 1, c0 + 32, row0);
                else if (next_row >= 0) sg.load(&om.resid, 1, n0, next_row);
            }
            __syncwarp();
            epi_chunk<BN, EK, 4>(d, 4 * s, epi, n0, N);
            sg.wait_loaded();
            resid_chunk<BN>(sg, d, 4 * s, epi.alpha);
            store(&om.out, c0, row0);
        }
    } else {
#pragma unroll
        for (int g = 0; g < NG; ++g) {
            const int c0 = n0 + 64 * g;
            if (c0 >= N) break;
            epi_chunk<BN, EK, 8>(d, 8 * g, epi, n0, N);
            if constexpr (EK == EPI_GLU_F32) {
                put_glu<BN>(sg, d, 8 * g);
                store(&om.out, c0 / 2, row0);
            } else if (EK == EPI_BIAS_F32 || EK == EPI_BIAS_RELU_F32) {
                put_f32<BN>(sg, d, 8 * g);
                store(&om.out, c0, row0);
                if (c0 + 32 < N) {
                    put_f32<BN>(sg, d, 8 * g + 4);
                    store(&om.out, c0 + 32, row0);
                }
            } else if (EK == EPI_QKV_ACT && c0 < epi.qcols) {     // q (qcols % 64 == 0): fp32 [M, qcols]
                sg.drain();
                put_f32<BN>(sg, d, 8 * g);
                store(&om.out, c0, row0);
                put_f32<BN>(sg, d, 8 * g + 4);
                store(&om.out, c0 + 32, row0);
            } else {                                                // act planes (k | v of QKV at column - qcols)
                const int pc = c0 - (EK == EPI_QKV_ACT ? epi.qcols : 0);
                sg.drain();
                if (EK != EPI_QKV_ACT && epi.act.f32) {
                    put_f32<BN>(sg, d, 8 * g);
                    store(&om.out, pc, row0);
                    if (pc + 32 < N) {
                        put_f32<BN>(sg, d, 8 * g + 4);
                        store(&om.out, pc + 32, row0);
                    }
                }
                if (epi.act.hi && epi.act.lo) {
                    if (EK != EPI_QKV_ACT && epi.act.f32) sg.drain();
                    put_bf16<BN, true>(sg, d, 8 * g);
                    sg.store_pair(&om.hi, &om.lo, pc, row0);
                    fence_operands(d);
                } else if (epi.act.hi) {
                    put_bf16<BN, false>(sg, d, 8 * g);
                    store(&om.hi, pc, row0);
                }
            }
        }
    }
}

// The cooperative kernel body of the cluster form below: thread-block clusters of CL CTAs along N.  The CL CTAs of a cluster
// work on the SAME 128-row block and on adjacent column tiles, so the A tile of a k-block is the same for all of them.  Each
// CTA fetches 128 / CL of its rows (tmA_* then have a 128 / CL-row box) and TMA-multicasts the slice into the stage of every
// CTA of the cluster; a stage is then written by all CTAs, so its "empty" barrier collects the arrivals of the consumer warps
// of all of them.
template <int BN, int NPASS, int EK, int CL>
__device__ __forceinline__ void gemm_tc_body(const CUtensorMap &tmA_hi, const CUtensorMap &tmA_lo, const CUtensorMap &tmW_hi,
                                             const CUtensorMap &tmW_lo, int M, int N, int K, const EpiParams &epi) {
    using C = TcCfg<BN, NPASS>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t *full = reinterpret_cast<uint64_t *>(tiles + (size_t)C::STAGES * C::STAGE_BYTES), *empty = full + C::STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int nkb = K / BK;
    const int tiles_n = (N + BN - 1) / BN, tiles_m = (M + BM - 1) / BM;
    // work units: the cluster walks (row block, group of CL column tiles); this CTA takes column tile `rank` of the group
    // (tiles_n % CL == 0, checked by the launcher)
    const uint32_t rank = cluster_ctarank();
    const int group_n = tiles_n / CL, num_units = group_n * tiles_m;
    const int first = (int)blockIdx.x / CL, step = (int)gridDim.x / CL;

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], CONSUMER_WARPS * CL);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    cluster_sync();      // every CTA's barriers exist before a peer multicasts into it / arrives on them

    if (wg == 0) {
        // ===================== TMA producer =====================
        if (warp == 0 && elect_one()) {
            uint32_t it = 0;   // global k-block counter across units
            for (int u = first; u < num_units; u += step) {
                const int m0 = (u / group_n) * BM, n0 = ((u % group_n) * CL + (int)rank) * BN;
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const int s = it % C::STAGES;
                    const uint32_t ph = (it / C::STAGES) & 1;
                    mbar_wait(&empty[s], ph ^ 1);
                    uint8_t *st = tiles + (size_t)s * C::STAGE_BYTES;
                    mbar_expect_tx(&full[s], C::STAGE_BYTES);
                    // this CTA's slice of the A rows, into the stage of every CTA of the cluster
                    constexpr int SL = BM / CL, SLB = SL * BK * 2;
                    constexpr uint16_t mask = (uint16_t)((1u << CL) - 1u);
                    tma_load_2d_mcast(st + rank * SLB, &tmA_hi, &full[s], kb * BK, m0 + (int)rank * SL, mask);
                    if (NPASS == 3) tma_load_2d_mcast(st + C::A_BYTES + C::W_BYTES + rank * SLB, &tmA_lo, &full[s], kb * BK, m0 + (int)rank * SL, mask);
                    tma_load_2d(st + C::A_BYTES, &tmW_hi, &full[s], kb * BK, n0);
                    if (NPASS == 3) tma_load_2d(st + 2 * C::A_BYTES + C::W_BYTES, &tmW_lo, &full[s], kb * BK, n0);
                }
            }
        }
        __syncwarp();                // the elected lane rejoins its warp before the .aligned cluster barrier at the end
    } else {
        // ===================== consumers: wgmma + epilogue =====================
        const int cw = wg - 1;                              // row half of the tile
        const uint32_t a_off = (uint32_t)cw * 64u * 128u;   // 64 rows of 128 B
        auto release = [&](int s) {                         // this warp has finished reading stage s
            __syncwarp();
            if (lane == 0) {
                const uint32_t a = smem_u32(&empty[s]);
#pragma unroll
                for (uint32_t r = 0; r < (uint32_t)CL; ++r) mbar_arrive_cluster(mapa_rank(a, r));
            }
        };
        uint32_t it = 0;
        for (int u = first; u < num_units; u += step) {
            const int m0 = (u / group_n) * BM, n0 = ((u % group_n) * CL + (int)rank) * BN;
            float d[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
            fence_operands(d);
            int prev_s = -1;
            for (int kb = 0; kb < nkb; ++kb, ++it) {
                const int s = it % C::STAGES;
                const uint32_t ph = (it / C::STAGES) & 1;
                mbar_wait(&full[s], ph);
                const uint32_t st = smem_u32(tiles + (size_t)s * C::STAGE_BYTES);
                const uint64_t a_hi = wgmma_desc_sw128(st + a_off), w_hi = wgmma_desc_sw128(st + C::A_BYTES);
                const uint64_t a_lo = wgmma_desc_sw128(st + C::A_BYTES + C::W_BYTES + a_off);
                const uint64_t w_lo = wgmma_desc_sw128(st + 2 * C::A_BYTES + C::W_BYTES);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / WGMMA_K; ++k) {
                    const uint64_t koff = (uint64_t)((k * WGMMA_K * 2) >> 4);   // 32 B per K step, encoded >> 4
                    wgmma_bf16<BN>(d, a_hi + koff, w_hi + koff);
                    if (NPASS == 3) {
                        wgmma_bf16<BN>(d, a_hi + koff, w_lo + koff);
                        wgmma_bf16<BN>(d, a_lo + koff, w_hi + koff);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();                            // the group of the previous k-block has retired
                if (prev_s >= 0) release(prev_s);
                prev_s = s;
            }
            wgmma_wait<0>();
            fence_operands(d);
            if (prev_s >= 0) release(prev_s);
            const int lrow0 = cw * 64 + (warp & 3) * 16;
            epilogue_regs<BN, EK>(d, epi, m0 + lrow0, n0, M, N, lane);
        }
    }
    cluster_sync();      // nobody leaves while a peer may still multicast into it / arrive on its barriers
}

// The default GEMM, in the ping-pong form: each consumer warpgroup owns whole 128 x BN tiles (the CTA's units alternate
// between them) and the two take turns in the mainloop, so one warpgroup's epilogue runs while the other issues wgmma.
// Named barriers ORDER_BAR + cw say "warpgroup cw may start its next mainloop"; the other warpgroup arrives on it once it
// has issued (not retired) the last wgmma of its own unit.  An arrival is made only if the waiting warpgroup has a unit
// left, so no barrier is left half-arrived when the CTA exits.
constexpr uint32_t ORDER_BAR = 1;
constexpr uint32_t PRODUCER_REGS = 40, CONSUMER_REGS = 232;    // 128 x 40 + 256 x 232 <= 64 K registers of the SM

template <int BN, int NPASS, int EK, bool STAGED>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo, int M, int N,
               int K, const __grid_constant__ EpiParams epi, const __grid_constant__ EpiMaps om) {
    using C = TcCfg<BN, NPASS, STAGED>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *chunks = tiles + (size_t)C::STAGES * C::STAGE_BYTES;
    uint64_t *rbar = reinterpret_cast<uint64_t *>(chunks + C::EPI_BYTES);     // STAGED: the residual loads, 2 per consumer
    uint64_t *full = rbar + (STAGED ? 4 : 0), *empty = full + C::STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int nkb = K / BK;
    const int tiles_n = (N + BN - 1) / BN, num_units = tiles_n * ((M + BM - 1) / BM);

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 4);       // the 4 warps of the warpgroup that consumed the stage
        }
        if (STAGED)
            for (int i = 0; i < 4; ++i) mbar_init(&rbar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<PRODUCER_REGS>();
        if (warp == 0 && elect_one()) {
            uint32_t it = 0;   // global k-block counter across units
            for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
                const int m0 = (u / tiles_n) * BM, n0 = (u % tiles_n) * BN;
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const int s = it % C::STAGES;
                    const uint32_t ph = (it / C::STAGES) & 1;
                    mbar_wait(&empty[s], ph ^ 1);
                    uint8_t *st = tiles + (size_t)s * C::STAGE_BYTES;
                    mbar_expect_tx(&full[s], C::STAGE_BYTES);
                    tma_load_2d(st, &tmA_hi, &full[s], kb * BK, m0);
                    if (NPASS == 3) tma_load_2d(st + C::A_BYTES + C::W_BYTES, &tmA_lo, &full[s], kb * BK, m0);
                    tma_load_2d(st + C::A_BYTES, &tmW_hi, &full[s], kb * BK, n0);
                    if (NPASS == 3) tma_load_2d(st + 2 * C::A_BYTES + C::W_BYTES, &tmW_lo, &full[s], kb * BK, n0);
                }
            }
        }
    } else {
        // ===================== consumers: wgmma + epilogue, one whole tile each =====================
        setmaxnreg_inc<CONSUMER_REGS>();
        const int cw = wg - 1;       // this warpgroup takes units cw, cw + 2, cw + 4, ... of the CTA
        auto release = [&](int s) {  // this warp has finished reading stage s
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        };
        Stager sg{smem_u32(chunks) + (uint32_t)cw * 2u * CHUNK_BYTES, 0u};
        constexpr uint32_t HALF = 64u * 128u;    // rows 64..127 of the A tile: 64 rows of 128 B further on
        uint32_t it = (uint32_t)(cw * nkb);      // the producer's k-block counter; the other warpgroup's units are skipped
        for (int j = cw;; j += 2) {
            const int u = (int)blockIdx.x + j * (int)gridDim.x;
            if (u >= num_units) break;
            const int m0 = (u / tiles_n) * BM, n0 = (u % tiles_n) * BN;
            float d0[BN / 2], d1[BN / 2];        // rows 0..63 and 64..127 of the tile
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) d0[i] = d1[i] = 0.f;
            fence_operands(d0);
            fence_operands(d1);
            if (j > 0) bar_sync(ORDER_BAR + cw, 256);     // the other warpgroup has issued its mainloop of unit j - 1
            int prev_s = -1;
            for (int kb = 0; kb < nkb; ++kb, ++it) {
                const int s = it % C::STAGES;
                const uint32_t ph = (it / C::STAGES) & 1;
                mbar_wait(&full[s], ph);
                const uint32_t st = smem_u32(tiles + (size_t)s * C::STAGE_BYTES);
                const uint64_t a_hi = wgmma_desc_sw128(st), w_hi = wgmma_desc_sw128(st + C::A_BYTES);
                const uint64_t a_lo = wgmma_desc_sw128(st + C::A_BYTES + C::W_BYTES);
                const uint64_t w_lo = wgmma_desc_sw128(st + 2 * C::A_BYTES + C::W_BYTES);
                const uint64_t a_hi1 = wgmma_desc_sw128(st + HALF), a_lo1 = wgmma_desc_sw128(st + C::A_BYTES + C::W_BYTES + HALF);
                wgmma_fence();
                // per accumulator the same MMA sequence as the cooperative body: k steps in order, hi.hi, hi.lo, lo.hi
#pragma unroll
                for (int k = 0; k < BK / WGMMA_K; ++k) {
                    const uint64_t koff = (uint64_t)((k * WGMMA_K * 2) >> 4);   // 32 B per K step, encoded >> 4
                    wgmma_bf16<BN>(d0, a_hi + koff, w_hi + koff);
                    wgmma_bf16<BN>(d1, a_hi1 + koff, w_hi + koff);
                    if (NPASS == 3) {
                        wgmma_bf16<BN>(d0, a_hi + koff, w_lo + koff);
                        wgmma_bf16<BN>(d1, a_hi1 + koff, w_lo + koff);
                        wgmma_bf16<BN>(d0, a_lo + koff, w_hi + koff);
                        wgmma_bf16<BN>(d1, a_lo1 + koff, w_hi + koff);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();                            // the group of the previous k-block has retired
                if (prev_s >= 0) release(prev_s);
                prev_s = s;
            }
            it += (uint32_t)nkb;
            if ((int)blockIdx.x + (j + 1) * (int)gridDim.x < num_units) bar_arrive(ORDER_BAR + (1 - cw), 256);
            if (EK == EPI_RESID_F32 && STAGED) {     // the tile's first residual chunk loads during the last k-block
                if (Stager::leader()) {
                    bulk_wait_read<0>();
                    sg.load(&om.resid, 0, n0, m0);
                }
                __syncwarp();
            }
            wgmma_wait<0>();
            fence_operands(d0);
            fence_operands(d1);
            if (prev_s >= 0) release(prev_s);
            const int lrow0 = (warp & 3) * 16;
            if constexpr (STAGED) {
                const bool two = m0 + 64 < M;        // rows 64..127 of the tile exist
                epilogue_staged<BN, EK>(d0, epi, om, sg, m0, n0, N, two ? m0 + 64 : -1);
                fence_operands(d1);
                if (two) epilogue_staged<BN, EK>(d1, epi, om, sg, m0 + 64, n0, N, -1);
            } else {
                epilogue_regs<BN, EK>(d0, epi, m0 + lrow0, n0, M, N, lane);
                epilogue_regs<BN, EK>(d1, epi, m0 + 64 + lrow0, n0, M, N, lane);
            }
        }
        // the stores must have written global memory before the CTA exits: the next grid may read them as soon as this one
        // has completed
        if constexpr (STAGED)
            if (Stager::leader()) bulk_wait<0>();
    }
}

// clusters of CL CTAs along N with the A tile multicast; 128-column tiles only
template <int NPASS, int EK, int CL>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(TC_THREADS, 1)
gemm_tc_cl_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                  const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo, int M, int N,
                  int K, const __grid_constant__ EpiParams epi) {
    gemm_tc_body<128, NPASS, EK, CL>(tmA_hi, tmA_lo, tmW_hi, tmW_lo, M, N, K, epi);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
            qr == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

int num_sms_cur() {
    int dev = 0;
    cudaGetDevice(&dev);
    static int sms_of[64] = {};
    if (!sms_of[dev & 63]) cudaDeviceGetAttribute(&sms_of[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    return sms_of[dev & 63];
}

// Tensor map of one [rows, width] output (leading dimension ld elements) in chunk boxes of 64 rows x 128 B, SWIZZLE_128B.
// TMA needs a 16-B aligned base and row pitch; TMA stores clip the rows >= rows and the columns >= width.
bool encode_out(CUtensorMap *m, const void *p, bool f32, uint64_t width, uint64_t rows, uint64_t ld) {
    EncodeTiledFn fn = encode_fn();
    const uint64_t esz = f32 ? 4 : 2;
    if (!fn || !p || (reinterpret_cast<uintptr_t>(p) & 15) || (ld * esz) % 16 || width == 0) return false;
    const cuuint64_t gdim[2] = {width, rows};
    const cuuint64_t gstr[1] = {ld * esz};
    const cuuint32_t box[2] = {(cuuint32_t)(128 / esz), (cuuint32_t)CHUNK_ROWS};
    const cuuint32_t estr[2] = {1, 1};
    return fn(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(p), gdim, gstr, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// The output maps of the staged epilogue, or false when a launch's outputs cannot all be written by TMA: it then keeps the
// register epilogue, whose fast path it would also take (N and ldo multiples of 4; otherwise epilogue4 serves every
// column, with its own sigmoid).
bool staged_maps(EpiMaps *om, const EpiParams &e, int M, int N) {
    if (N % 4 || e.ldo % 4) return false;
    switch (e.kind) {
    case EPI_BIAS_F32:
    case EPI_BIAS_RELU_F32: return encode_out(&om->out, e.out_f32, true, N, M, e.ldo);
    case EPI_RESID_F32: return encode_out(&om->out, e.out_f32, true, N, M, e.ldo) && encode_out(&om->resid, e.resid, true, N, M, e.ldo);
    case EPI_GLU_F32: return encode_out(&om->out, e.out_f32, true, N / 2, M, e.ldo);
    case EPI_QKV_ACT:
        if (e.qcols <= 0 || e.qcols % 64 || e.qcols >= N || e.act.f32 || !e.act.hi) return false;
        return encode_out(&om->out, e.out_f32, true, e.qcols, M, e.qcols) && encode_out(&om->hi, e.act.hi, false, N - e.qcols, M, e.ldo) &&
               (!e.act.lo || encode_out(&om->lo, e.act.lo, false, N - e.qcols, M, e.ldo));
    case EPI_BIAS_RELU_ACT:
    case EPI_BIAS_SILU_ACT:
    case EPI_BIAS_ACT:
        if (!e.act.f32 && !e.act.hi) return false;
        return (!e.act.f32 || encode_out(&om->out, e.act.f32, true, N, M, e.ldo)) && (!e.act.hi || encode_out(&om->hi, e.act.hi, false, N, M, e.ldo)) &&
               (!e.act.lo || encode_out(&om->lo, e.act.lo, false, N, M, e.ldo));
    default: return false;
    }
}

template <int BN, int NPASS, int EK, bool STAGED>
cudaError_t launch_k(const TcOperand &A, const TcOperand &W, int M, int N, int K, const EpiParams &epi, const EpiMaps &om, cudaStream_t st) {
    using C = TcCfg<BN, NPASS, STAGED>;
    static PerDeviceFlag attr_flag;
    bool &attr = attr_flag.cur();
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<BN, NPASS, EK, STAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
        if (e != cudaSuccess) return e;
        attr = true;
    }
    const int num_sms = num_sms_cur();
    const int num_tiles = ((N + BN - 1) / BN) * ((M + BM - 1) / BM);
    dim3 grid(num_tiles < num_sms ? num_tiles : num_sms);
    const CUtensorMap &alo = (NPASS == 3) ? A.lo : A.hi, &wlo = (NPASS == 3) ? W.lo : W.hi;
    gemm_tc_kernel<BN, NPASS, EK, STAGED><<<grid, dim3(TC_THREADS), C::SMEM, st>>>(A.hi, alo, W.hi, wlo, M, N, K, epi, om);
    return cudaGetLastError();
}

template <int BN, int NPASS, int EK>
cudaError_t launch_e(const TcOperand &A, const TcOperand &W, int M, int N, int K, const EpiParams &epi, cudaStream_t st) {
    EpiMaps om = {};
    if (staged_maps(&om, epi, M, N)) return launch_k<BN, NPASS, EK, true>(A, W, M, N, K, epi, om, st);
    return launch_k<BN, NPASS, EK, false>(A, W, M, N, K, epi, om, st);
}

template <int BN, int NPASS>
cudaError_t launch_t(const TcOperand &A, const TcOperand &W, int M, int N, int K, const EpiParams &epi, cudaStream_t st) {
    switch (epi.kind) {
    case EPI_BIAS_F32: return launch_e<BN, NPASS, EPI_BIAS_F32>(A, W, M, N, K, epi, st);
    case EPI_BIAS_RELU_F32: return launch_e<BN, NPASS, EPI_BIAS_RELU_F32>(A, W, M, N, K, epi, st);
    case EPI_BIAS_RELU_ACT: return launch_e<BN, NPASS, EPI_BIAS_RELU_ACT>(A, W, M, N, K, epi, st);
    case EPI_BIAS_SILU_ACT: return launch_e<BN, NPASS, EPI_BIAS_SILU_ACT>(A, W, M, N, K, epi, st);
    case EPI_RESID_F32: return launch_e<BN, NPASS, EPI_RESID_F32>(A, W, M, N, K, epi, st);
    case EPI_GLU_F32: return launch_e<BN, NPASS, EPI_GLU_F32>(A, W, M, N, K, epi, st);
    case EPI_BIAS_ACT: return launch_e<BN, NPASS, EPI_BIAS_ACT>(A, W, M, N, K, epi, st);
    case EPI_QKV_ACT: return launch_e<BN, NPASS, EPI_QKV_ACT>(A, W, M, N, K, epi, st);
    default: return cudaErrorInvalidValue;
    }
}

// cluster / multicast variant: A_sl = the A operand with a 128 / CL-row box
template <int NPASS, int EK, int CL>
cudaError_t launch_kcl(const TcOperand &A_sl, const TcOperand &W, int M, int N, int K, const EpiParams &epi, cudaStream_t st) {
    using C = TcCfg<128, NPASS>;
    static PerDeviceFlag attr_flag;
    static int max_clusters[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    const int num_sms = num_sms_cur();
    if (!attr_flag.cur()) {
        cudaError_t e = cudaFuncSetAttribute(gemm_tc_cl_kernel<NPASS, EK, CL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
        if (e != cudaSuccess) return e;
        cudaLaunchConfig_t q = {};
        q.gridDim = dim3((unsigned)(num_sms / CL * CL));
        q.blockDim = dim3(TC_THREADS);
        q.dynamicSmemBytes = C::SMEM;
        int mc = 0;
        if (cudaOccupancyMaxActiveClusters(&mc, gemm_tc_cl_kernel<NPASS, EK, CL>, &q) != cudaSuccess || mc < 1) {
            cudaGetLastError();
            mc = num_sms / CL;
        }
        max_clusters[dev & 63] = mc;
        attr_flag.cur() = true;
    }
    const int units = ((N / 128) / CL) * ((M + BM - 1) / BM);
    int ncl = max_clusters[dev & 63];
    if (ncl > num_sms / CL) ncl = num_sms / CL;
    if (ncl > units) ncl = units;
    const CUtensorMap &alo = (NPASS == 3) ? A_sl.lo : A_sl.hi, &wlo = (NPASS == 3) ? W.lo : W.hi;
    gemm_tc_cl_kernel<NPASS, EK, CL><<<dim3((unsigned)(ncl * CL)), dim3(TC_THREADS), C::SMEM, st>>>(A_sl.hi, alo, W.hi, wlo, M, N, K, epi);
    return cudaGetLastError();
}

}  // namespace

bool make_tc_operand(TcOperand *out, const bf16 *hi, const bf16 *lo, uint64_t rows, uint64_t K, uint32_t box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn || !hi || (K % 8) != 0) return false;
    const cuuint64_t gdim[2] = {K, rows};
    const cuuint64_t gstr[1] = {K * sizeof(bf16)};
    const cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    if (fn(&out->hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<bf16 *>(hi), gdim, gstr, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return false;
    out->has_lo = lo != nullptr;
    if (lo && fn(&out->lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<bf16 *>(lo), gdim, gstr, box, estr,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return false;
    out->box_rows = box_rows;
    return true;
}

int tc_tile_n(int N) { return N <= 64 ? 64 : 128; }

bool gemm_tc_cluster_supported(int N, int epi_kind, int cl) {
    return (cl == 2 || cl == 4) && N % (128 * cl) == 0 && (epi_kind == EPI_BIAS_SILU_ACT || epi_kind == EPI_GLU_F32 || epi_kind == EPI_QKV_ACT);
}

cudaError_t launch_gemm_tc(const TcOperand &A, const TcOperand &W, int M, int N, int K, bool split3, const EpiParams &epi, cudaStream_t st,
                           int cl, const TcOperand *A_slice) {
    if (M <= 0 || N <= 0) return cudaSuccess;
    if (K % BK != 0 || A.box_rows != BM) return cudaErrorInvalidValue;
    if (split3 && !(A.has_lo && W.has_lo)) return cudaErrorInvalidValue;
    if (cl > 1 && split3 && A_slice && A_slice->has_lo && (int)A_slice->box_rows * cl == BM && W.box_rows == 128 && gemm_tc_cluster_supported(N, epi.kind, cl)) {
        // clusters of `cl` CTAs along N, A tile multicast (gemm_tc_body)
        switch (epi.kind) {
        case EPI_BIAS_SILU_ACT: return cl == 2 ? launch_kcl<3, EPI_BIAS_SILU_ACT, 2>(*A_slice, W, M, N, K, epi, st) : launch_kcl<3, EPI_BIAS_SILU_ACT, 4>(*A_slice, W, M, N, K, epi, st);
        case EPI_GLU_F32: return cl == 2 ? launch_kcl<3, EPI_GLU_F32, 2>(*A_slice, W, M, N, K, epi, st) : launch_kcl<3, EPI_GLU_F32, 4>(*A_slice, W, M, N, K, epi, st);
        default: return cl == 2 ? launch_kcl<3, EPI_QKV_ACT, 2>(*A_slice, W, M, N, K, epi, st) : launch_kcl<3, EPI_QKV_ACT, 4>(*A_slice, W, M, N, K, epi, st);
        }
    }
    if (W.box_rows == 128) return split3 ? launch_t<128, 3>(A, W, M, N, K, epi, st) : launch_t<128, 1>(A, W, M, N, K, epi, st);
    if (W.box_rows == 64) return split3 ? launch_t<64, 3>(A, W, M, N, K, epi, st) : launch_t<64, 1>(A, W, M, N, K, epi, st);
    return cudaErrorInvalidValue;
}

}  // namespace pk
