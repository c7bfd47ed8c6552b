// pk_common.cuh -- shared declarations for the sm_90a kernels of the hot path.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pk {

typedef __nv_bfloat16 bf16;

// cudaFuncSetAttribute is per DEVICE: a process that drives several GPUs (one pk_engine per device, e.g.
// examples/sharded_transcribe.cpp) must set a kernel's attributes once on each of them.  Returns the flag of the
// current device inside a caller-owned per-kernel table.
struct PerDeviceFlag {
    bool done[64] = {};
    size_t size[64] = {};
    bool &cur() {
        int dev = 0;
        cudaGetDevice(&dev);
        return done[dev & 63];
    }
    size_t &cur_size() {
        int dev = 0;
        cudaGetDevice(&dev);
        return size[dev & 63];
    }
};

// An activation that feeds a GEMM as the A operand.  In PK_MATH_FP32 mode only
// `f32` is set; in the tensor-core modes the producer kernel writes the bf16 hi/lo
// split planes (hi = rn(x), lo = rn(x - hi)), which cost the same bytes as fp32.
struct ActBuf {
    float *f32 = nullptr;
    bf16 *hi = nullptr;
    bf16 *lo = nullptr;
};

__device__ __forceinline__ void store_act(const ActBuf &o, size_t idx, float v) {
    if (o.f32) o.f32[idx] = v;
    if (o.hi) {
        bf16 h = __float2bfloat16_rn(v);
        o.hi[idx] = h;
        if (o.lo) o.lo[idx] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
}

// 4 consecutive elements (idx multiple of 4): vectorised stores.
__device__ __forceinline__ void store_act4(const ActBuf &o, size_t idx, float4 v) {
    if (o.f32) *reinterpret_cast<float4 *>(o.f32 + idx) = v;
    if (o.hi) {
        __nv_bfloat162 h01 = __floats2bfloat162_rn(v.x, v.y), h23 = __floats2bfloat162_rn(v.z, v.w);
        uint2 hp;
        hp.x = *reinterpret_cast<uint32_t *>(&h01);
        hp.y = *reinterpret_cast<uint32_t *>(&h23);
        *reinterpret_cast<uint2 *>(o.hi + idx) = hp;
        if (o.lo) {
            float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
            __nv_bfloat162 l01 = __floats2bfloat162_rn(v.x - f01.x, v.y - f01.y);
            __nv_bfloat162 l23 = __floats2bfloat162_rn(v.z - f23.x, v.w - f23.y);
            uint2 lp;
            lp.x = *reinterpret_cast<uint32_t *>(&l01);
            lp.y = *reinterpret_cast<uint32_t *>(&l23);
            *reinterpret_cast<uint2 *>(o.lo + idx) = lp;
        }
    }
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float siluf_(float x) { return x * sigmoidf_(x); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---------------------------------------------------------------- GEMM epilogues
// out = epi(A[M,K] . W[N,K]^T + bias).  All epilogues see 4 consecutive columns
// of one row (col0 % 4 == 0) so GLU pairs and vector stores stay in-thread.
enum EpiKind : int {
    EPI_BIAS_F32 = 0,      // out_f32[row, col] = acc + bias
    EPI_BIAS_RELU_F32 = 1, // relu -> out_f32
    EPI_BIAS_RELU_ACT = 2, // relu -> act (feeds the next GEMM)
    EPI_BIAS_SILU_ACT = 3, // silu -> act
    EPI_RESID_F32 = 4,     // out_f32[row, col] = resid[row, col] + alpha * (acc + bias)
    EPI_GLU_F32 = 5,       // columns interleaved (a0,b0,a1,b1..): out_f32[row, col/2] = a * sigmoid(b)
    EPI_BIAS_ACT = 6,      // acc + bias -> act
    EPI_QKV_ACT = 7,       // fused q/k/v projection for the tensor-core attention (encoder.cpp:129-140): columns < qcols (q)
                           // -> out_f32[M, qcols] (fp32: the attention kernel adds pos_bias_u / pos_bias_v and splits, so a q
                           // tile costs the epilogue ONE fp32 tile instead of four bf16 planes); the rest (k | v) -> act planes
                           // [M, N - qcols]
};

struct EpiParams {
    int kind = EPI_BIAS_F32;
    const float *bias = nullptr;  // [N] (interleaved order for GLU)
    float *out_f32 = nullptr;
    int ldo = 0;                  // leading dimension of out_f32 / act / resid (elements)
    ActBuf act;
    const float *resid = nullptr;
    float alpha = 1.0f;
    int qcols = 0;                // EPI_QKV_ACT: leading q columns (also the leading dimension of out_f32)
};

// Generic (edge-tile / run-time-kind) path; out of line so that it does not bloat the hot loops.
static __device__ __noinline__ void epilogue4(const EpiParams &p, int row, int col0, int N, float4 acc) {
    if (col0 >= N) return;
    float v[4] = {acc.x, acc.y, acc.z, acc.w};
    const bool full = (col0 + 3 < N);
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if (p.bias && col0 + i < N) v[i] += p.bias[col0 + i];
    switch (p.kind) {
    case EPI_BIAS_RELU_F32:
    case EPI_BIAS_RELU_ACT:
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = fmaxf(v[i], 0.f);
        break;
    case EPI_BIAS_SILU_ACT:
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = siluf_(v[i]);
        break;
    default:
        break;
    }
    const size_t base = (size_t)row * p.ldo + col0;
    switch (p.kind) {
    case EPI_BIAS_F32:
    case EPI_BIAS_RELU_F32:
        if (full && (p.ldo & 3) == 0) {
            *reinterpret_cast<float4 *>(p.out_f32 + base) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
            for (int i = 0; i < 4 && col0 + i < N; ++i) p.out_f32[base + i] = v[i];
        }
        break;
    case EPI_BIAS_RELU_ACT:
    case EPI_BIAS_SILU_ACT:
    case EPI_BIAS_ACT:
        if (full && (p.ldo & 3) == 0) {
            store_act4(p.act, base, make_float4(v[0], v[1], v[2], v[3]));
        } else {
            for (int i = 0; i < 4 && col0 + i < N; ++i) store_act(p.act, base + i, v[i]);
        }
        break;
    case EPI_RESID_F32:
        if (full && (p.ldo & 3) == 0) {
            float4 r = *reinterpret_cast<const float4 *>(p.resid + base);
            *reinterpret_cast<float4 *>(p.out_f32 + base) =
                make_float4(r.x + p.alpha * v[0], r.y + p.alpha * v[1], r.z + p.alpha * v[2],
                            r.w + p.alpha * v[3]);
        } else {
            for (int i = 0; i < 4 && col0 + i < N; ++i)
                p.out_f32[base + i] = p.resid[base + i] + p.alpha * v[i];
        }
        break;
    case EPI_QKV_ACT:
        for (int i = 0; i < 4 && col0 + i < N; ++i) {
            const int cidx = col0 + i;
            if (cidx < p.qcols) p.out_f32[(size_t)row * p.qcols + cidx] = v[i];
            else store_act(p.act, (size_t)row * p.ldo + cidx - p.qcols, v[i]);
        }
        break;
    case EPI_GLU_F32: {
        // N is even and col0 % 4 == 0, so both pairs are in range together.
        const size_t ob = (size_t)row * p.ldo + (col0 >> 1);
        p.out_f32[ob] = v[0] * sigmoidf_(v[1]);
        if (col0 + 2 < N) p.out_f32[ob + 1] = v[2] * sigmoidf_(v[3]);
        break;
    }
    }
}

// Compile-time-specialised fast path for interior tiles (all 4 columns < N, ldo % 4 == 0).
// (ex2.approx + rcp.approx: two MUFU ops, branch-free.  __frcp_rn is an IEEE-rounded reciprocal with
// a per-element slow-path branch, which serialises the whole epilogue.)
__device__ __forceinline__ float fast_sigmoid(float x) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return r;
}

// Split form used by the tensor-core kernels: all global LOADS of a 16-column chunk (bias, residual)
// are issued before the accumulator is read, then pure math, then all STORES -- otherwise every
// epilogue4 call waits for its own L2 round trip (loads cannot be hoisted above the previous
// call's stores: out_f32 may alias resid).
template <int KIND>
__device__ __forceinline__ float4 epi_math(float4 v, const float4 &b, const float4 &r, float alpha) {
    v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
    if (KIND == EPI_BIAS_RELU_F32 || KIND == EPI_BIAS_RELU_ACT) {
        v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    } else if (KIND == EPI_BIAS_SILU_ACT) {
        v.x *= fast_sigmoid(v.x); v.y *= fast_sigmoid(v.y); v.z *= fast_sigmoid(v.z); v.w *= fast_sigmoid(v.w);
    } else if (KIND == EPI_RESID_F32) {
        v = make_float4(r.x + alpha * v.x, r.y + alpha * v.y, r.z + alpha * v.z, r.w + alpha * v.w);
    } else if (KIND == EPI_GLU_F32) {
        v = make_float4(v.x * fast_sigmoid(v.y), v.z * fast_sigmoid(v.w), 0.f, 0.f);
    }
    return v;
}
template <int KIND>
__device__ __forceinline__ void epi_store(const EpiParams &p, int row, int col0, const float4 &v) {
    const size_t base = (size_t)row * p.ldo + col0;
    if (KIND == EPI_QKV_ACT) {
        if (col0 < p.qcols) *reinterpret_cast<float4 *>(p.out_f32 + (size_t)row * p.qcols + col0) = v;
        else store_act4(p.act, base - p.qcols, v);
    } else if (KIND == EPI_BIAS_F32 || KIND == EPI_BIAS_RELU_F32 || KIND == EPI_RESID_F32) {
        *reinterpret_cast<float4 *>(p.out_f32 + base) = v;
    } else if (KIND == EPI_GLU_F32) {
        *reinterpret_cast<float2 *>(p.out_f32 + (size_t)row * p.ldo + (col0 >> 1)) = make_float2(v.x, v.y);
    } else {
        store_act4(p.act, base, v);
    }
}

}  // namespace pk
