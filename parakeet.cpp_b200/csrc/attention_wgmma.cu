// attention_wgmma.cu -- K7 for head_dim 64 and utterances of <= 128 frames (every tdt-ctc-110m 10 s clip) on Hopper
// wgmma: the relative-position attention of reference src/encoder.cpp:111-178 (rel_shift :85-109)
//     S[i,j] = ((q_i + u).k_j + (q_i + v).PP[i-j]) / sqrt(64),  ctx_i = softmax_j(S[i,:]) V
// with the same bf16 hi/lo operand split as the GEMMs (3 MMAs per product: hi.hi + hi.lo + lo.hi, fp32 accumulate).
//
// One CTA = (utterance, head), 256 threads = two warpgroups; warpgroup w owns query rows [64 w, 64 w + 64).
//   1. The CTA stages every operand in shared memory once, as SWIZZLE_128B K-major tiles (the layout wgmma reads):
//      Qu = q + u and Qv = q + v (fp32 add, hi/lo split), K, V transposed (V^T: the B operand of P.V is K-major), and
//      the window of the position table that the tile's relative positions i - j in [-127, 127] touch (255 rows).
//   2. G = Qv . PPwin^T (wgmma m64 n192: the 191 positions of this warpgroup's rows) -> shared memory, where the
//      rel_shift is a skewed read: S[r][j] += G[r][r - j + 127].  G overlays the Qv / PP tiles, dead by then.
//   3. S = Qu . K^T (wgmma m64 n128), scale, mask keys j >= T, softmax over the whole row in registers.
//   4. O = P . V (wgmma m64 n64 with P as the register A operand: the accumulator layout of S is the A-fragment
//      layout), normalise, store ctx as fp32 and / or bf16 hi/lo planes.
#include "kernels.h"
#include "tc_prims.cuh"

namespace pk {
namespace {

using namespace tc;

constexpr int AW_THREADS = 256;
constexpr int AW_T = 128, AW_HD = 64, AW_NPOS = 256;  // max frames, head_dim, position window rows (255 used)
constexpr int GLD = 192;                               // G staging row stride (floats)

// shared-memory map (bytes); every tile 1024-byte aligned
constexpr int OFF_QU = 0;                              // Qu hi | lo: 2 x 128 rows x 128 B
constexpr int OFF_K = OFF_QU + 2 * AW_T * 128;         // K hi | lo
constexpr int OFF_VT = OFF_K + 2 * AW_T * 128;         // V^T hi | lo: per plane 2 key blocks x 64 rows x 128 B
constexpr int OFF_QV = OFF_VT + 2 * AW_T * 128;        // Qv hi | lo
constexpr int OFF_PP = OFF_QV + 2 * AW_T * 128;        // PP window hi | lo: 2 x 256 rows x 128 B
constexpr int OFF_END = OFF_PP + 2 * AW_NPOS * 128;
constexpr int OFF_G = OFF_QV;                          // G staging (overlays Qv and PP): 2 warpgroups x 64 rows x GLD floats
static_assert(OFF_G + 2 * 64 * GLD * 4 <= OFF_END, "G staging fits over Qv / PP");
constexpr size_t AW_SMEM = OFF_END + 1024;

// byte offset of 16-byte chunk `c` of row `r` in a SWIZZLE_128B K-major tile
__device__ __forceinline__ uint32_t sw128(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

__device__ __forceinline__ void wgmma_ss_n192(float (&d)[96], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
        : "l"(adesc), "l"(bdesc));
}

__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc));
}

template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ uint32_t pack_bf16(float x, float y) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    return *reinterpret_cast<const uint32_t *>(&h);
}
__device__ __forceinline__ void split2(float x, float y, uint32_t &hi, uint32_t &lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    const float2 hf = __bfloat1622float2(h);
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = pack_bf16(x - hf.x, y - hf.y);
}

__global__ void __launch_bounds__(AW_THREADS, 1)
relpos_attention_wgmma_kernel(const float *__restrict__ q32, const float *__restrict__ pos_u, const float *__restrict__ pos_v,
                              const bf16 *__restrict__ kv_hi, const bf16 *__restrict__ kv_lo, int ld_kv, const int32_t *__restrict__ row_off,
                              const bf16 *__restrict__ pp_hi, const bf16 *__restrict__ pp_lo, int tmax, int d_model, ActBuf out) {
    pdl_wait();
    pdl_trigger();
    extern __shared__ uint8_t smraw[];
    uint8_t *sm = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smraw) + 1023) & ~(uintptr_t)1023);
    const int b = blockIdx.y, h = blockIdx.x;
    const int r0 = row_off[b], T = row_off[b + 1] - r0;
    if (T <= 0) return;
    const int tid = threadIdx.x;

    // ---- 1. operands -> swizzled tiles (rows past T and positions outside the table are zeros)
    for (int e = tid; e < AW_T * 8; e += AW_THREADS) {           // K: row j, chunk c (8 bf16)
        const int j = e >> 3, c = e & 7;
        uint4 kh = make_uint4(0u, 0u, 0u, 0u), kl = kh;
        if (j < T) {
            const size_t g = (size_t)(r0 + j) * ld_kv + h * AW_HD + c * 8;
            kh = *reinterpret_cast<const uint4 *>(kv_hi + g);
            kl = *reinterpret_cast<const uint4 *>(kv_lo + g);
        }
        *reinterpret_cast<uint4 *>(sm + OFF_K + sw128(j, c)) = kh;
        *reinterpret_cast<uint4 *>(sm + OFF_K + AW_T * 128 + sw128(j, c)) = kl;
    }
    for (int e = tid; e < AW_T * 32; e += AW_THREADS) {          // V^T: key j, dims 2 p, 2 p + 1 -> rows 2 p, 2 p + 1 of key block j / 64
        const int j = e >> 5, p = e & 31;
        uint32_t vh = 0u, vl = 0u;
        if (j < T) {
            const size_t g = (size_t)(r0 + j) * ld_kv + d_model + h * AW_HD + 2 * p;
            vh = *reinterpret_cast<const uint32_t *>(kv_hi + g);
            vl = *reinterpret_cast<const uint32_t *>(kv_lo + g);
        }
        const int kb = j >> 6, k = j & 63;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int row = 2 * p + t;
            const uint32_t off = kb * 64 * 128 + sw128(row, k >> 3) + (k & 7) * 2;
            *reinterpret_cast<uint16_t *>(sm + OFF_VT + off) = (uint16_t)(t ? vh >> 16 : vh & 0xffffu);
            *reinterpret_cast<uint16_t *>(sm + OFF_VT + AW_T * 128 + off) = (uint16_t)(t ? vl >> 16 : vl & 0xffffu);
        }
    }
    for (int e = tid; e < AW_NPOS * 8; e += AW_THREADS) {        // PP window: smem row pr <-> relative position pr - 127
        const int pr = e >> 3, c = e & 7;
        const int prow = pr - (AW_T - 1) + tmax - 1;
        uint4 ph = make_uint4(0u, 0u, 0u, 0u), pl = ph;
        if (pr < 2 * AW_T - 1 && prow >= 0 && prow < 2 * tmax - 1) {
            const size_t g = (size_t)prow * d_model + h * AW_HD + c * 8;
            ph = *reinterpret_cast<const uint4 *>(pp_hi + g);
            pl = *reinterpret_cast<const uint4 *>(pp_lo + g);
        }
        *reinterpret_cast<uint4 *>(sm + OFF_PP + sw128(pr, c)) = ph;
        *reinterpret_cast<uint4 *>(sm + OFF_PP + AW_NPOS * 128 + sw128(pr, c)) = pl;
    }
    for (int e = tid; e < AW_T * 16; e += AW_THREADS) {          // Qu / Qv: row i, 4 columns 4 c4 .. (fp32 q + bias, then split)
        const int i = e >> 4, c4 = e & 15;
        float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < T) q = *reinterpret_cast<const float4 *>(q32 + (size_t)(r0 + i) * d_model + h * AW_HD + 4 * c4);
        const float4 u = __ldg(reinterpret_cast<const float4 *>(pos_u + h * AW_HD + 4 * c4));
        const float4 v = __ldg(reinterpret_cast<const float4 *>(pos_v + h * AW_HD + 4 * c4));
        uint32_t uh0, ul0, uh1, ul1, vh0, vl0, vh1, vl1;
        split2(q.x + u.x, q.y + u.y, uh0, ul0);
        split2(q.z + u.z, q.w + u.w, uh1, ul1);
        split2(q.x + v.x, q.y + v.y, vh0, vl0);
        split2(q.z + v.z, q.w + v.w, vh1, vl1);
        const uint32_t off = sw128(i, c4 >> 1) + (c4 & 1) * 8;
        *reinterpret_cast<uint2 *>(sm + OFF_QU + off) = make_uint2(uh0, uh1);
        *reinterpret_cast<uint2 *>(sm + OFF_QU + AW_T * 128 + off) = make_uint2(ul0, ul1);
        *reinterpret_cast<uint2 *>(sm + OFF_QV + off) = make_uint2(vh0, vh1);
        *reinterpret_cast<uint2 *>(sm + OFF_QV + AW_T * 128 + off) = make_uint2(vl0, vl1);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
    __syncthreads();

    const int wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const uint32_t base = smem_u32(sm);
    const uint32_t qrow = (uint32_t)wg * 64u * 128u;             // this warpgroup's 64 query rows
    constexpr uint32_t PL = AW_T * 128;                           // plane stride of the 128-row tiles

    // ---- 2. G = Qv . PPwin^T over window rows [64 wg, 64 wg + 192)
    {
        float gacc[96];
#pragma unroll
        for (int i = 0; i < 96; ++i) gacc[i] = 0.f;
        fence_regs(gacc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t ko = (uint32_t)k * 32u;
            const uint32_t pw = base + OFF_PP + (uint32_t)wg * 64u * 128u + ko;
            const uint64_t ah = wgmma_desc_sw128(base + OFF_QV + qrow + ko), al = wgmma_desc_sw128(base + OFF_QV + PL + qrow + ko);
            const uint64_t bh = wgmma_desc_sw128(pw), bl = wgmma_desc_sw128(pw + AW_NPOS * 128);
            wgmma_ss_n192(gacc, ah, bh);
            wgmma_ss_n192(gacc, ah, bl);
            wgmma_ss_n192(gacc, al, bh);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(gacc);
        __syncthreads();                                          // both warpgroups are done with Qv / PP
        float *gs = reinterpret_cast<float *>(sm + OFF_G) + wg * 64 * GLD;
#pragma unroll
        for (int jj = 0; jj < 24; ++jj) {
            const int col = 8 * jj + 2 * c, ra = warp * 16 + g;
            *reinterpret_cast<float2 *>(gs + ra * GLD + col) = make_float2(gacc[4 * jj], gacc[4 * jj + 1]);
            *reinterpret_cast<float2 *>(gs + (ra + 8) * GLD + col) = make_float2(gacc[4 * jj + 2], gacc[4 * jj + 3]);
        }
    }

    // ---- 3. S = Qu . K^T, + skewed G, scale, mask, softmax
    float s[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
    fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t ko = (uint32_t)k * 32u;
        const uint64_t ah = wgmma_desc_sw128(base + OFF_QU + qrow + ko), al = wgmma_desc_sw128(base + OFF_QU + PL + qrow + ko);
        const uint64_t bh = wgmma_desc_sw128(base + OFF_K + ko), bl = wgmma_desc_sw128(base + OFF_K + PL + ko);
        wgmma_bf16<128>(s, ah, bh);
        wgmma_bf16<128>(s, ah, bl);
        wgmma_bf16<128>(s, al, bh);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    __syncthreads();                                              // G staging complete
    const float *gs = reinterpret_cast<const float *>(sm + OFF_G) + wg * 64 * GLD;
    constexpr float kScale = 0.125f * 1.4426950408889634f;       // 1 / sqrt(64), folded with log2 e
    float l_row[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int r = warp * 16 + g + 8 * hr;                     // row inside the warpgroup
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int j = 8 * jj + 2 * c + e;
                float v = (s[4 * jj + 2 * hr + e] + gs[r * GLD + r - j + (AW_T - 1)]) * kScale;
                v = j < T ? v : -INFINITY;
                s[4 * jj + 2 * hr + e] = v;
                mx = fmaxf(mx, v);
            }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float sum = 0.f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float p = exp2f(s[4 * jj + 2 * hr + e] - mx);
                s[4 * jj + 2 * hr + e] = p;
                sum += p;
            }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        l_row[hr] = sum;
    }

    // ---- 4. O = P . V: P of key k-step kk = accumulator columns 16 kk .. 16 kk + 15 as the register A fragment
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
        uint32_t ph[4], pl[4];
        split2(s[8 * kk], s[8 * kk + 1], ph[0], pl[0]);
        split2(s[8 * kk + 2], s[8 * kk + 3], ph[1], pl[1]);
        split2(s[8 * kk + 4], s[8 * kk + 5], ph[2], pl[2]);
        split2(s[8 * kk + 6], s[8 * kk + 7], ph[3], pl[3]);
        const uint32_t vt = base + OFF_VT + (uint32_t)(kk >> 2) * 64u * 128u + (uint32_t)(kk & 3) * 32u;
        const uint64_t bh = wgmma_desc_sw128(vt), bl = wgmma_desc_sw128(vt + PL);
        wgmma_rs_n64(o, ph, bh);
        wgmma_rs_n64(o, ph, bl);
        wgmma_rs_n64(o, pl, bh);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);

#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int i = wg * 64 + warp * 16 + g + 8 * hr;
        if (i >= T) continue;
        const float inv = 1.0f / l_row[hr];
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) {
            const size_t idx = (size_t)(r0 + i) * d_model + h * AW_HD + nb * 8 + 2 * c;
            const float x = o[4 * nb + 2 * hr] * inv, y = o[4 * nb + 2 * hr + 1] * inv;
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

bool relpos_attention_wgmma_supported(int head_dim, int max_T) { return head_dim == AW_HD && max_T >= 1 && max_T <= AW_T; }

bool launch_relpos_attention_wgmma(const float *q32, const float *pos_u, const float *pos_v, const bf16 *kv_hi, const bf16 *kv_lo, int ld_kv,
                                   const int32_t *row_off, int n_utt, int max_T, int n_heads, int head_dim, const bf16 *pp_hi, const bf16 *pp_lo,
                                   int tmax, int d_model, ActBuf out, cudaStream_t st) {
    if (!q32 || !pos_u || !pos_v || !kv_hi || !kv_lo || !pp_hi || !pp_lo || !relpos_attention_wgmma_supported(head_dim, max_T)) return false;
    if (n_utt <= 0) return true;
    static PerDeviceFlag attr_flag;
    if (!attr_flag.cur()) {
        if (cudaFuncSetAttribute(relpos_attention_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AW_SMEM) != cudaSuccess) return false;
        attr_flag.cur() = true;
    }
    return launch_pdl(relpos_attention_wgmma_kernel, dim3(n_heads, n_utt), dim3(AW_THREADS), AW_SMEM, st, q32, pos_u, pos_v, kv_hi, kv_lo, ld_kv, row_off,
                      pp_hi, pp_lo, tmax, d_model, out) == cudaSuccess;
}

}  // namespace pk
