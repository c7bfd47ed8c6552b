// mel.cu -- K1/K2: 16 kHz PCM -> per-utterance normalised log-mel features.
//
// Replaces preprocess_audio (reference src/audio.cpp:100-158) and the pieces of
// axiom it calls (fft::hann_window fft.cpp:1117-1142, fft::stft fft.cpp:1478-1605,
// ops::matmul with the Slaney filterbank audio.cpp:40-94, ops::log, mean / unbiased
// std normalisation audio.cpp:139-152).
//
// K1 mel_logpower_kernel: one warp per STFT frame.
//   pre-emphasis + reflect padding + centred 400-tap Hann -> 512 real samples ->
//   256-point complex FFT done in registers (8-point DFT per lane, twiddle,
//   32-point DFT across the warp with shuffles: the "four-step" split 256 = 8 x 32)
//   -> real-FFT untangling -> |X|^2 for 257 bins -> sparse Slaney filterbank -> log.
//   HBM traffic: each PCM sample is read ~3.2x from L2 (512/160 frame overlap),
//   once from DRAM; 4*n_mels bytes written per frame.
// K2 mel_normalize_kernel: per utterance, per mel bin: mean, unbiased variance,
//   (x - mean) / (sqrt(var) + 1e-5), two-pass like the reference.
#include <cmath>

#include "kernels.h"

namespace pk {

namespace {

constexpr int N_FFT = 512;
constexpr int WIN = 400;
constexpr int HOP = 160;
constexpr int WIN_PAD = (N_FFT - WIN) / 2;  // 56, axiom fft.cpp:1539-1547
constexpr int WARPS = 4;

struct cplx {
    float re, im;
};
__device__ __forceinline__ cplx cadd(cplx a, cplx b) { return {a.re + b.re, a.im + b.im}; }
__device__ __forceinline__ cplx csub(cplx a, cplx b) { return {a.re - b.re, a.im - b.im}; }
__device__ __forceinline__ cplx cmul(cplx a, cplx b) {
    return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re};
}
__device__ __forceinline__ cplx cmul_negi(cplx a) { return {a.im, -a.re}; }  // a * (-i)
__device__ __forceinline__ cplx cshfl_xor(cplx a, int m) {
    return {__shfl_xor_sync(0xffffffffu, a.re, m), __shfl_xor_sync(0xffffffffu, a.im, m)};
}

__device__ __forceinline__ void dft4(cplx x0, cplx x1, cplx x2, cplx x3, cplx &q0, cplx &q1, cplx &q2,
                                     cplx &q3) {
    cplx c0 = cadd(x0, x2), c2 = csub(x0, x2), c1 = cadd(x1, x3), c3 = cmul_negi(csub(x1, x3));
    q0 = cadd(c0, c1);
    q1 = cadd(c2, c3);
    q2 = csub(c0, c1);
    q3 = csub(c2, c3);
}

// sample of the pre-emphasised signal y[i] = x[i] - 0.97 x[i-1] (y[0] = x[0]),
// audio.cpp:104-114, with reflect padding (axiom ops::pad "reflect") for i outside [0, n).  axiom reflects repeatedly
// (operations.cpp:2217-2227), which matters for signals of 2..200 samples (Sortformer stream chunks); from 201 samples
// on one reflection reaches every index a frame reads.  n >= 2 (n = 1 never terminates in the reference).
__device__ __forceinline__ float preemph_reflect(const float *__restrict__ x, int64_t i, int64_t n) {
    while (i < 0 || i >= n) {
        if (i < 0) i = -i;
        if (i >= n) i = 2 * n - 2 - i;
    }
    float v = x[i];
    if (i > 0) v -= 0.97f * x[i - 1];
    return v;
}

// STREAM = true: the streaming preprocessor's frames (audio.cpp:195-259): `pcm` is the pre-emphasised signal
// [overlap | chunk] of stream b, frame f = window . sig[f*160 + j], j in [0, 512) (center = False: no reflection, no
// half-window shift), n_frames from `n_frames_arr`, output row = frame_off[b] + f.
template <bool STREAM>
__global__ void __launch_bounds__(WARPS * 32)
mel_logpower_kernel(const float *__restrict__ pcm, const int64_t *__restrict__ pcm_off,
                    const int32_t *__restrict__ frame_off, const int32_t *__restrict__ n_frames_arr, int n_mels, MelTables tb,
                    float *__restrict__ logmel) {
    extern __shared__ float smem[];
    // layout: [window 400][tw256 512][tw512 514][fb weights nnz][per-warp: frame 512 | Z 512 | P 260]
    float *s_win = smem;
    float2 *s_tw256 = reinterpret_cast<float2 *>(s_win + WIN);
    float2 *s_tw512 = s_tw256 + 256;
    float *s_fbw = reinterpret_cast<float *>(s_tw512 + 257);
    float *s_warp = s_fbw + ((tb.fb_nnz + 3) & ~3);

    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_frames = STREAM ? n_frames_arr[b] : frame_off[b + 1] - frame_off[b];
    const int f0 = blockIdx.x * (WARPS * 4);
    if (f0 >= n_frames) return;

    for (int i = threadIdx.x; i < WIN; i += blockDim.x) s_win[i] = tb.window[i];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_tw256[i] = tb.tw256[i];
    for (int i = threadIdx.x; i < 257; i += blockDim.x) s_tw512[i] = tb.tw512[i];
    for (int i = threadIdx.x; i < tb.fb_nnz; i += blockDim.x) s_fbw[i] = tb.fb_w[i];
    __syncthreads();

    float *s_frame = s_warp + warp * (512 + 512 + 260);
    float2 *s_Z = reinterpret_cast<float2 *>(s_frame + 512);
    float *s_P = s_frame + 1024;

    const float *x = pcm + pcm_off[b];
    const int64_t n = pcm_off[b + 1] - pcm_off[b];

    // each warp handles 4 consecutive frames of this block's 16
    for (int fi = 0; fi < 4; ++fi) {
        const int f = f0 + warp * 4 + fi;
        if (f >= n_frames) break;  // warp-uniform
        // frame j in [0,512) <-> sample index f*HOP - 256 + j; window is zero outside [56, 456)
        const int64_t s0 = (int64_t)f * HOP - (STREAM ? 0 : N_FFT / 2);
        const bool interior = (s0 + WIN_PAD - 1 >= 0) && (s0 + WIN_PAD + WIN <= n);
        for (int j = lane; j < N_FFT; j += 32) {
            float v = 0.f;
            if (j >= WIN_PAD && j < WIN_PAD + WIN) {
                const int64_t i = s0 + j;
                float y;
                if (STREAM) {
                    y = x[i];
                } else if (interior) {
                    y = x[i] - 0.97f * x[i - 1];  // coalesced; x[i-1] hits the same lines
                } else {
                    y = preemph_reflect(x, i, n);
                }
                v = y * s_win[j - WIN_PAD];
            }
            s_frame[j] = v;
        }
        __syncwarp();

        // ---- 256-point complex FFT of z[m] = frame[2m] + i frame[2m+1], m = 32*n1 + lane
        cplx a[8];
#pragma unroll
        for (int n1 = 0; n1 < 8; ++n1) {
            float2 v = *reinterpret_cast<const float2 *>(s_frame + 2 * (32 * n1 + lane));
            a[n1] = {v.x, v.y};
        }
        // 8-point DFT over n1 (decimation in frequency)
        cplx b0 = cadd(a[0], a[4]), b4 = csub(a[0], a[4]);
        cplx b1 = cadd(a[1], a[5]), b5 = csub(a[1], a[5]);
        cplx b2 = cadd(a[2], a[6]), b6 = csub(a[2], a[6]);
        cplx b3 = cadd(a[3], a[7]), b7 = csub(a[3], a[7]);
        const float r = 0.70710678118654752440f;
        b5 = cmul(b5, cplx{r, -r});   // W8^1
        b6 = cmul_negi(b6);           // W8^2
        b7 = cmul(b7, cplx{-r, -r});  // W8^3
        cplx Y[8];
        dft4(b0, b1, b2, b3, Y[0], Y[2], Y[4], Y[6]);
        dft4(b4, b5, b6, b7, Y[1], Y[3], Y[5], Y[7]);
        // twiddle W256^(lane*k1)
#pragma unroll
        for (int k1 = 1; k1 < 8; ++k1) {
            float2 w = s_tw256[lane * k1];
            Y[k1] = cmul(Y[k1], cplx{w.x, w.y});
        }
        // 32-point DFT across lanes (radix-2 DIF, output lane = bitrev5(k2))
#pragma unroll
        for (int h = 16; h >= 1; h >>= 1) {
            float2 w = s_tw256[(lane & (h - 1)) * (128 / h)];  // W_{2h}^(lane mod h) = W256^(.. * 128/h)
            const bool upper = (lane & h) != 0;
#pragma unroll
            for (int k1 = 0; k1 < 8; ++k1) {
                cplx o = cshfl_xor(Y[k1], h);
                Y[k1] = upper ? cmul(csub(o, Y[k1]), cplx{w.x, w.y}) : cadd(Y[k1], o);
            }
        }
        const int k2 = __brev((unsigned)lane) >> 27;
#pragma unroll
        for (int k1 = 0; k1 < 8; ++k1) s_Z[k1 + 8 * k2] = make_float2(Y[k1].re, Y[k1].im);
        __syncwarp();

        // ---- untangle to the 257-bin real spectrum, power = |X|^2 (audio.cpp:123-124)
        for (int k = lane; k <= 256; k += 32) {
            float2 zk = s_Z[k & 255], zm = s_Z[(256 - k) & 255];
            cplx Zk = {zk.x, zk.y}, Zm = {zm.x, -zm.y};
            cplx E = {0.5f * (Zk.re + Zm.re), 0.5f * (Zk.im + Zm.im)};
            cplx D = csub(Zk, Zm);
            cplx O = {0.5f * D.im, -0.5f * D.re};  // -0.5 i D
            float2 w = s_tw512[k];
            cplx X = cadd(E, cmul(cplx{w.x, w.y}, O));
            s_P[k] = X.re * X.re + X.im * X.im;
        }
        __syncwarp();

        // ---- sparse Slaney filterbank + log (audio.cpp:126-136)
        float *out = logmel + ((size_t)frame_off[b] + f) * n_mels;
        for (int m = lane; m < n_mels; m += 32) {
            const int st = tb.fb_start[m], len = tb.fb_len[m], off = tb.fb_off[m];
            float acc = 0.f;
            for (int i = 0; i < len; ++i) acc = fmaf(s_fbw[off + i], s_P[st + i], acc);
            out[m] = logf(acc + 5.96046448e-8f);
        }
        __syncwarp();
    }
}

// K2: per-utterance, per-bin normalisation (audio.cpp:138-150: mean over the frames, UNBIASED variance, eps outside the root).
// One block per utterance would leave most SMs idle (64 blocks) and sweep the frames three times serially.  Instead every
// utterance is cut into MEL_CH frame chunks: mel_stats_kernel reduces a chunk to (mean_c, M2_c = sum (x - mean_c)^2) per bin with
// two sweeps over its own frames, mel_apply_kernel combines the MEL_CH partials of an utterance in a fixed order with Chan's
// formula (mean = sum n_c mean_c / F, M2 = sum M2_c + n_c (mean_c - mean)^2: the accuracy of the two-pass form, deterministic,
// independent of the batch) and normalises its chunk.  threads = (groups x n_mels).  Both work on x - x0, x0 = the bin's value in
// the utterance's first frame: a constant bin (digital silence) then has chunk means and M2 of exactly 0 and comes out as 0,
// where rounded means of the raw values would leave an offset of an ulp that 1 / (0 + 1e-5) scales up to O(1).
constexpr int MEL_CH = 16;

__device__ __forceinline__ void mel_chunk(int c, int F, int &f0, int &f1) {
    f0 = (int)((long long)c * F / MEL_CH);
    f1 = (int)((long long)(c + 1) * F / MEL_CH);
}

__global__ void mel_stats_kernel(const float *__restrict__ logmel, const int32_t *__restrict__ frame_off, int n_mels,
                                 float *__restrict__ part /* [utterance][MEL_CH][2][n_mels] */) {
    extern __shared__ float red[];  // [groups][n_mels]
    const int b = blockIdx.y, c = blockIdx.x;
    const int groups = blockDim.x / n_mels;
    const int m = threadIdx.x % n_mels, g = threadIdx.x / n_mels;
    const int F0 = frame_off[b], F = frame_off[b + 1] - F0;
    int f0, f1;
    mel_chunk(c, F, f0, f1);
    const int nc = f1 - f0;
    const bool active = g < groups;
    const float *src = logmel + (size_t)F0 * n_mels;
    const float x0 = src[m];

    float s = 0.f;
    if (active)
        for (int f = f0 + g; f < f1; f += groups) s += src[(size_t)f * n_mels + m] - x0;
    if (active) red[g * n_mels + m] = s;
    __syncthreads();
    float mean = 0.f;
    for (int i = 0; i < groups; ++i) mean += red[i * n_mels + m];
    mean = nc > 0 ? mean / (float)nc : 0.f;
    __syncthreads();
    float q = 0.f;
    if (active)
        for (int f = f0 + g; f < f1; f += groups) {
            float d = (src[(size_t)f * n_mels + m] - x0) - mean;
            q = fmaf(d, d, q);
        }
    if (active) red[g * n_mels + m] = q;
    __syncthreads();
    if (g == 0) {
        float m2 = 0.f;
        for (int i = 0; i < groups; ++i) m2 += red[i * n_mels + m];
        float *p = part + ((size_t)(b * MEL_CH + c) * 2) * n_mels;
        p[m] = mean;
        p[n_mels + m] = m2;
    }
}

__global__ void mel_apply_kernel(const float *__restrict__ logmel, const int32_t *__restrict__ frame_off, int n_mels,
                                 const float *__restrict__ part, float *__restrict__ feats) {
    const int b = blockIdx.y, c = blockIdx.x;
    const int groups = blockDim.x / n_mels;
    const int m = threadIdx.x % n_mels, g = threadIdx.x / n_mels;
    const int F0 = frame_off[b], F = frame_off[b + 1] - F0;
    if (g >= groups) return;
    const float *pb = part + ((size_t)b * MEL_CH * 2) * n_mels;
    float tot = 0.f;
    for (int k = 0; k < MEL_CH; ++k) {
        int a0, a1;
        mel_chunk(k, F, a0, a1);
        tot = fmaf((float)(a1 - a0), pb[(size_t)(2 * k) * n_mels + m], tot);
    }
    const float mean = tot / (float)F;
    float m2 = 0.f;
    for (int k = 0; k < MEL_CH; ++k) {
        int a0, a1;
        mel_chunk(k, F, a0, a1);
        const float d = pb[(size_t)(2 * k) * n_mels + m] - mean;
        m2 += pb[(size_t)(2 * k + 1) * n_mels + m] + (float)(a1 - a0) * d * d;
    }
    const float var = m2 / (float)(F - 1);          // unbiased, audio.cpp:146-147
    const float inv = 1.0f / (sqrtf(var) + 1e-5f);  // eps outside the sqrt, :148
    int f0, f1;
    mel_chunk(c, F, f0, f1);
    const float *src = logmel + (size_t)F0 * n_mels;
    const float x0 = src[m];
    float *dst = feats + (size_t)F0 * n_mels;
    for (int f = f0 + g; f < f1; f += groups) dst[(size_t)f * n_mels + m] = ((src[(size_t)f * n_mels + m] - x0) - mean) * inv;
}

}  // namespace

MelTables build_mel_tables(int n_mels, const std::function<void *(const void *, size_t)> &upload) {
    // host, double precision where the reference uses it
    std::vector<float> win(400);
    for (int i = 0; i < 400; ++i) win[i] = (float)(0.5 - 0.5 * std::cos(2.0 * M_PI * i / 399.0));  // fft.cpp:1117-1142
    std::vector<float2> tw256(256), tw512(257);
    for (int m = 0; m < 256; ++m) tw256[m] = make_float2((float)std::cos(2.0 * M_PI * m / 256.0), (float)-std::sin(2.0 * M_PI * m / 256.0));
    for (int k = 0; k <= 256; ++k) tw512[k] = make_float2((float)std::cos(2.0 * M_PI * k / 512.0), (float)-std::sin(2.0 * M_PI * k / 512.0));
    // Slaney filterbank, audio.cpp:18-94
    auto hz2mel = [](double f) { return f < 1000.0 ? f / (200.0 / 3.0) : 15.0 + std::log(f / 1000.0) / 0.06875177742094912; };
    auto mel2hz = [](double m) { return m < 15.0 ? m * (200.0 / 3.0) : 1000.0 * std::exp((m - 15.0) * 0.06875177742094912); };
    const int nm = n_mels, nf = 257;
    const double mmin = hz2mel(0.0), mmax = hz2mel(8000.0);
    std::vector<double> hz(nm + 2);
    for (int i = 0; i < nm + 2; ++i) hz[i] = mel2hz(mmin + (double)i * (mmax - mmin) / (double)(nm + 1));
    std::vector<float> fbw;
    std::vector<int32_t> fstart(nm), flen(nm), foff(nm);
    for (int m = 0; m < nm; ++m) {
        const double left = hz[m], center = hz[m + 1], right = hz[m + 2], enorm = 2.0 / (right - left);
        int first = -1, last = -1;
        std::vector<float> col(nf);
        for (int f = 0; f < nf; ++f) {
            const double fr = (double)f * 16000.0 / (2.0 * (nf - 1));
            double v = 0.0;
            if (fr >= left && fr <= center && center > left) v = (fr - left) / (center - left);
            else if (fr > center && fr <= right && right > center) v = (right - fr) / (right - center);
            col[f] = (float)(v * enorm);
            if (col[f] != 0.f) {
                if (first < 0) first = f;
                last = f;
            }
        }
        fstart[m] = first < 0 ? 0 : first;
        flen[m] = first < 0 ? 0 : last - first + 1;
        foff[m] = (int32_t)fbw.size();
        for (int f = fstart[m]; f < fstart[m] + flen[m]; ++f) fbw.push_back(col[f]);
    }
    auto up = [&](const auto &v) { return upload(v.data(), v.size() * sizeof(v[0])); };
    MelTables tb;
    tb.window = static_cast<const float *>(up(win));
    tb.tw256 = static_cast<const float2 *>(up(tw256));
    tb.tw512 = static_cast<const float2 *>(up(tw512));
    tb.fb_w = static_cast<const float *>(up(fbw));
    tb.fb_start = static_cast<const int32_t *>(up(fstart));
    tb.fb_len = static_cast<const int32_t *>(up(flen));
    tb.fb_off = static_cast<const int32_t *>(up(foff));
    tb.fb_nnz = (int)fbw.size();
    return tb;
}

size_t mel_smem_bytes(const MelTables &tb) {
    return sizeof(float) * (WIN + 512 + 514 + ((tb.fb_nnz + 3) & ~3) + WARPS * (512 + 512 + 260));
}

size_t mel_part_floats(int n_utt, int n_mels) { return (size_t)n_utt * MEL_CH * 2 * n_mels; }

void launch_mel(const float *pcm, const int64_t *pcm_off, const int32_t *frame_off, int n_utt,
                int max_frames, int n_mels, const MelTables &tb, float *logmel, float *feats, float *part,
                cudaStream_t st, bool normalize) {
    dim3 grid((max_frames + WARPS * 4 - 1) / (WARPS * 4), n_utt);
    mel_logpower_kernel<false><<<dim3(grid), dim3(WARPS * 32), mel_smem_bytes(tb), st>>>(pcm, pcm_off, frame_off, nullptr, n_mels, tb,
                                                                             normalize ? logmel : feats);
    if (!normalize) return;
    int groups = MEL_NORM_THREADS / n_mels;  // 8 for 80 bins, 5 for 128
    mel_stats_kernel<<<dim3(MEL_CH, n_utt), dim3(groups * n_mels), sizeof(float) * groups * n_mels, st>>>(logmel, frame_off, n_mels, part);
    mel_apply_kernel<<<dim3(MEL_CH, n_utt), dim3(groups * n_mels), 0, st>>>(logmel, frame_off, n_mels, part, feats);
}

void launch_mel_stream(const float *sig, const int64_t *sig_off, const int32_t *n_frames, const int32_t *out_row, int n_streams,
                       int max_frames, int n_mels, const MelTables &tb, float *logmel, cudaStream_t st) {
    if (max_frames <= 0) return;
    dim3 grid((max_frames + WARPS * 4 - 1) / (WARPS * 4), n_streams);
    mel_logpower_kernel<true><<<dim3(grid), dim3(WARPS * 32), mel_smem_bytes(tb), st>>>(sig, sig_off, out_row, n_frames, n_mels, tb, logmel);
}

}  // namespace pk
