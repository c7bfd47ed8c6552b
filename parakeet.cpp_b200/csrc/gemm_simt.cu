// gemm_simt.cu -- fp32 CUDA-core GEMM  C = epi(A[M,K] . W[N,K]^T + bias)
//
// This is the PK_MATH_FP32 arithmetic: exact fp32 products and fp32 accumulation,
// used for bring-up, as the on-device checker of the wgmma kernel (gemm_tc.cu), and
// for the small load-time GEMMs (pos_proj of the position table, the LSTM input table).
// It computes what nn::Linear (axiom linear.cpp:15-27) and the k=1 / 1x1 convolutions
// (operations.cpp:2960, :3133) compute, with the activation/residual that follows
// fused into the epilogue (pk_common.cuh).
//
// 128x128x16 tiles, 256 threads, 8x8 outputs per thread, register-prefetched double
// buffer; both operands are K-contiguous so global loads are float4 along K.
#include "kernels.h"

namespace pk {
namespace {

constexpr int BM = 128, BN = 128, BK = 16;

__global__ void __launch_bounds__(256)
gemm_simt_kernel(const float *__restrict__ A, int lda, const float *__restrict__ W, int ldw, int M, int N,
                 int K, EpiParams epi) {
    __shared__ __align__(16) float As[2][BK][BM + 4];
    __shared__ __align__(16) float Bs[2][BK][BN + 4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;     // row tiles on x: M may exceed 65535 tiles (long front ends)
    const int tx = tid & 15, ty = tid >> 4;
    // loader mapping: 512 float4 per operand tile, 2 per thread: row = idx / 4, kq = idx % 4
    float4 ra[2], rb[2];
    auto gload = [&](int k0) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int idx = tid + i * 256;
            const int row = idx >> 2, kq = (idx & 3) * 4;
            const int gm = m0 + row, gn = n0 + row, gk = k0 + kq;
            ra[i] = (gm < M && gk < K) ? *reinterpret_cast<const float4 *>(A + (size_t)gm * lda + gk)
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
            rb[i] = (gn < N && gk < K) ? *reinterpret_cast<const float4 *>(W + (size_t)gn * ldw + gk)
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int idx = tid + i * 256;
            const int row = idx >> 2, kq = (idx & 3) * 4;
            As[buf][kq + 0][row] = ra[i].x;
            As[buf][kq + 1][row] = ra[i].y;
            As[buf][kq + 2][row] = ra[i].z;
            As[buf][kq + 3][row] = ra[i].w;
            Bs[buf][kq + 0][row] = rb[i].x;
            Bs[buf][kq + 1][row] = rb[i].y;
            Bs[buf][kq + 2][row] = rb[i].z;
            Bs[buf][kq + 3][row] = rb[i].w;
        }
    };
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    const int nk = (K + BK - 1) / BK;
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kb = 0; kb < nk; ++kb) {
        const int buf = kb & 1;
        if (kb + 1 < nk) gload((kb + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4 *>(&Bs[buf][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4 *>(&Bs[buf][k][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kb + 1 < nk) {
            sstore(buf ^ 1);
            __syncthreads();
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int row = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (row >= M) continue;
        epilogue4(epi, row, n0 + tx * 4, N, make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]));
        epilogue4(epi, row, n0 + 64 + tx * 4, N, make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]));
    }
}

}  // namespace

void launch_gemm_simt(const float *A, int lda, const float *W, int ldw, int M, int N, int K,
                      const EpiParams &epi, cudaStream_t st) {
    if (M <= 0 || N <= 0) return;
    dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN);
    gemm_simt_kernel<<<dim3(grid), dim3(256), 0, st>>>(A, lda, W, ldw, M, N, K, epi);
}

}  // namespace pk
