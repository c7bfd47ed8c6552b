// speaker_head.cu -- Sortformer's speaker head (reference src/sortformer.cpp:59-67), fused into one kernel:
//     probs = sigmoid(output_proj_(ReLU(first_hidden_(ReLU(x)))))      x [M][D] -> probs [M][S]
// in fp32 on CUDA cores.  It replaces two GEMM launches (one of them N = S = 4 wide, which no tensor-core tile fits) and the
// element-wise ReLU / sigmoid passes.  Each CTA stages first_hidden_'s weight transposed ([k][n], D x D fp32) and
// output_proj_'s weight in shared memory once and walks row tiles of HEAD_R rows: thread n computes hidden column n of the
// tile, then S x HEAD_R threads reduce the logits.  hidden_to_spks_ is not used by the reference's forward.
#include "kernels.h"

namespace pk {
namespace {

constexpr int HEAD_R = 16;   // rows per tile

__global__ void __launch_bounds__(256)
speaker_head_kernel(const float *__restrict__ x, int M, int D, int S, const float *__restrict__ w1t /* [D][D] = W1^T */,
                    const float *__restrict__ b1, const float *__restrict__ w2 /* [S][D] */, const float *__restrict__ b2,
                    float *__restrict__ probs) {
    extern __shared__ __align__(16) float sm[];
    float *W1 = sm;                    // [D][D]
    float *W2 = W1 + (size_t)D * D;    // [S][D]
    float *xs = W2 + (size_t)S * D;    // [HEAD_R][D]  ReLU(x)
    float *hs = xs + HEAD_R * D;       // [HEAD_R][D]  ReLU(first_hidden_(.))
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < D * D; i += nt) W1[i] = w1t[i];
    for (int i = tid; i < S * D; i += nt) W2[i] = w2[i];
    const float bn = tid < D ? b1[tid] : 0.f;
    for (int r0 = blockIdx.x * HEAD_R; r0 < M; r0 += gridDim.x * HEAD_R) {
        const int nr = min(HEAD_R, M - r0);
        __syncthreads();               // weights staged / previous tile consumed
        for (int i = tid; i < HEAD_R * D; i += nt) {
            const int r = i / D;
            xs[i] = r < nr ? fmaxf(x[(size_t)r0 * D + i], 0.f) : 0.f;
        }
        __syncthreads();
        if (tid < D) {
            float acc[HEAD_R];
#pragma unroll
            for (int r = 0; r < HEAD_R; ++r) acc[r] = 0.f;
            for (int k = 0; k < D; ++k) {
                const float w = W1[k * D + tid];
#pragma unroll
                for (int r = 0; r < HEAD_R; ++r) acc[r] = fmaf(xs[r * D + k], w, acc[r]);
            }
#pragma unroll
            for (int r = 0; r < HEAD_R; ++r) hs[r * D + tid] = fmaxf(acc[r] + bn, 0.f);
        }
        __syncthreads();
        for (int o = tid; o < nr * S; o += nt) {
            const int r = o / S, s = o % S;
            float acc = 0.f;
            for (int k = 0; k < D; ++k) acc = fmaf(hs[r * D + k], W2[s * D + k], acc);
            probs[(size_t)(r0 + r) * S + s] = 1.0f / (1.0f + expf(-(acc + b2[s])));
        }
    }
}

}  // namespace

size_t speaker_head_smem(int D, int S) { return sizeof(float) * ((size_t)D * D + (size_t)S * D + 2 * HEAD_R * D); }

bool launch_speaker_head(const float *x, int M, int D, int S, const float *w1t, const float *b1, const float *w2, const float *b2,
                         float *probs, int num_sms, cudaStream_t st) {
    const size_t smem = speaker_head_smem(D, S);
    if (D < 1 || D > 256 || D % 32 || S < 1 || S > 64 || smem > 227 * 1024) return false;
    if (M <= 0) return true;
    static PerDeviceFlag attr_flag;
    bool &attr_set = attr_flag.cur();
    if (!attr_set) {
        if (cudaFuncSetAttribute(speaker_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess) return false;
        attr_set = true;
    }
    const int tiles = (M + HEAD_R - 1) / HEAD_R;
    const int grid = std::max(1, std::min(tiles, num_sms));
    speaker_head_kernel<<<dim3(grid), dim3(D), smem, st>>>(x, M, D, S, w1t, b1, w2, b2, probs);
    return cudaGetLastError() == cudaSuccess;
}

}  // namespace pk
