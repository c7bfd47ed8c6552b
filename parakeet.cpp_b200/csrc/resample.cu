// resample.cu -- front-of-path sample-rate conversion (SURVEY.md section 8f row 4) as a POLYPHASE filter, on the device
// for batches that enter the path (pk_stage_pcm_rate, pk_resample_batch) and on the host for engine-less callers
// (pk_resample: parakeet::resample of the C++ shim).  It replaces sinc_resample / parakeet::resample of the reference
// (src/audio_io.cpp:123-195, :238-251), whose definition is: output i sits at source position i * src/dst; it is the
// weighted mean of the 32 input samples around floor(position) with weights
//     sinc(pi * cutoff * dist) * kaiser(dist / widen; beta 7.857, half-width 16) * cutoff,
// cutoff = min(1, dst/src), widen = max(1, src/dst), taps outside the input or outside the window dropped from both the
// sum and the normalising weight sum, all in double.
//
// The reference re-evaluates the window (a Bessel series) and the sinc for every tap of every output.  Here the
// structure of the problem is used instead: with src/dst = down/up in lowest terms, output i has the exact rational
// position (i * down) / up, so its 32 weights depend only on the PHASE r = (i * down) mod up.  The host builds the
// up x 32 weight table once per rate pair (double precision); converting a sample is then 32 multiply-adds in double
// (explicitly un-fused, accumulated in the reference's tap order), a table row read from L1/L2 and 32 coalesced input
// reads.  Results equal the reference's to the last float bit except where its per-output rounding of i / (dst/src)
// differs from the exact rational (measured in tests/: >= 99.9 % identical floats, rest 1 ulp).
#include <cmath>
#include <map>
#include <mutex>
#include <numeric>
#include <vector>

#include "../../include/parakeet_b200.h"
#include "kernels.h"

namespace pk {
namespace {

constexpr int RS_TAPS = 32, RS_HALF = 16;
constexpr double RS_BETA = 7.857;

// I0 by its power series: sum_k ((x/2)^k / k!)^2
double i0_series(double x) {
    const double q = 0.25 * x * x;
    double term = 1.0, sum = 1.0;
    for (int k = 1; k < 30; ++k) {
        term *= q / ((double)k * (double)k);
        sum += term;
        if (term < 1e-12 * sum) break;
    }
    return sum;
}

struct RateTable {
    int up = 1, down = 1;
    std::vector<double> w;      // [up][32]; 0.0 marks a tap outside the window
};

// weights of phase r: tap k sits at source index floor(pos) - 15 + k, i.e. at distance frac + 15 - k from the output
RateTable build_table(int src_rate, int dst_rate) {
    RateTable t;
    const int g = std::gcd(src_rate, dst_rate);
    t.up = dst_rate / g;
    t.down = src_rate / g;
    const double ratio = (double)src_rate / (double)dst_rate;
    const double cutoff = ratio > 1.0 ? 1.0 / ratio : 1.0, widen = ratio > 1.0 ? ratio : 1.0;
    const double i0_beta = i0_series(RS_BETA);
    t.w.assign((size_t)t.up * RS_TAPS, 0.0);
    for (int r = 0; r < t.up; ++r) {
        const double frac = (double)r / (double)t.up;
        for (int k = 0; k < RS_TAPS; ++k) {
            const double dist = frac + (double)(RS_HALF - 1 - k);
            const double wpos = dist / widen;
            if (std::fabs(wpos) > (double)RS_HALF) continue;
            const double a = 2.0 * (wpos + RS_HALF) / (2.0 * RS_HALF) - 1.0;      // window argument in [-1, 1]
            double inside = 1.0 - a * a;
            if (inside < 0.0) inside = 0.0;
            const double win = i0_series(RS_BETA * std::sqrt(inside)) / i0_beta;
            const double x = dist * cutoff * M_PI;
            const double sinc = std::fabs(x) < 1e-10 ? 1.0 : std::sin(x) / x;
            t.w[(size_t)r * RS_TAPS + k] = sinc * win * cutoff;
        }
    }
    return t;
}

const RateTable &table_for(int src_rate, int dst_rate) {
    static std::mutex mu;
    static std::map<std::pair<int, int>, RateTable> cache;
    std::lock_guard<std::mutex> lk(mu);
    auto key = std::make_pair(src_rate, dst_rate);
    auto it = cache.find(key);
    if (it == cache.end()) it = cache.emplace(key, build_table(src_rate, dst_rate)).first;
    return it->second;
}

// one thread per output sample; utterance = blockIdx.y
__global__ void polyphase_resample_kernel(const float *__restrict__ in, const int64_t *__restrict__ in_off,
                                          const int64_t *__restrict__ out_off, const double *__restrict__ table, int up, int down,
                                          float *__restrict__ out) {
    const int b = blockIdx.y;
    const float *x = in + in_off[b];
    const int64_t n = in_off[b + 1] - in_off[b], m = out_off[b + 1] - out_off[b];
    float *y = out + out_off[b];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t num = i * down;
        const int64_t center = num / up;
        const double *w = table + (size_t)(num - center * up) * RS_TAPS;
        double sum = 0.0, wsum = 0.0;
#pragma unroll 8
        for (int k = 0; k < RS_TAPS; ++k) {
            const int64_t j = center - (RS_HALF - 1) + k;
            if (j < 0 || j >= n) continue;
            const double wk = w[k];
            sum = __dadd_rn(sum, __dmul_rn((double)x[j], wk));      // un-fused, tap order of the reference
            wsum = __dadd_rn(wsum, wk);
        }
        y[i] = wsum > 1e-10 ? (float)(sum / wsum) : 0.0f;
    }
}

}  // namespace

// device table cache (per process and device): returns a device pointer to the [up][32] doubles
const double *resample_device_table(int src_rate, int dst_rate, int *up, int *down, cudaStream_t st) {
    static std::mutex mu;
    static std::map<std::tuple<int, int, int>, double *> cache;
    const RateTable &t = table_for(src_rate, dst_rate);
    *up = t.up;
    *down = t.down;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lk(mu);
    auto key = std::make_tuple(dev, src_rate, dst_rate);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
    double *d = nullptr;
    if (cudaMalloc(&d, t.w.size() * sizeof(double)) != cudaSuccess) return nullptr;
    if (cudaMemcpyAsync(d, t.w.data(), t.w.size() * sizeof(double), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) {
        cudaFree(d);
        return nullptr;
    }
    cache[key] = d;
    return d;
}

bool launch_resample(const float *in, const int64_t *in_off, const int64_t *out_off, int n_utt, int64_t max_out, int src_rate,
                     int dst_rate, float *out, cudaStream_t st) {
    int up = 1, down = 1;
    const double *tab = resample_device_table(src_rate, dst_rate, &up, &down, st);
    if (!tab) return false;
    const int threads = 256;
    int64_t bx = (max_out + threads - 1) / threads;
    if (bx > 4096) bx = 4096;
    if (bx < 1) bx = 1;
    polyphase_resample_kernel<<<dim3((unsigned)bx, n_utt), dim3(threads), 0, st>>>(in, in_off, out_off, tab, up, down, out);
    return cudaGetLastError() == cudaSuccess;
}

}  // namespace pk

extern "C" {

int64_t pk_resample_len(int64_t n, int32_t src_rate, int32_t dst_rate) {
    if (n < 0 || src_rate <= 0 || dst_rate <= 0) return -1;
    if (src_rate == dst_rate) return n;
    const int g = std::gcd(src_rate, dst_rate);
    const int64_t up = dst_rate / g, down = src_rate / g;
    return (n * up + down - 1) / down;                     // ceil(n * dst / src)
}

// Host instance of the same polyphase filter for engine-less callers (parakeet::resample of the C++ shim).
int64_t pk_resample(const float *in, int64_t n, int32_t src_rate, int32_t dst_rate, float *out, int64_t cap) {
    const int64_t m = pk_resample_len(n, src_rate, dst_rate);
    if (m < 0 || cap < 0 || (n > 0 && !in) || (cap > 0 && !out)) return -1;
    const int64_t lim = m < cap ? m : cap;
    if (src_rate == dst_rate) {
        for (int64_t i = 0; i < lim; ++i) out[i] = in[i];
        return m;
    }
    const pk::RateTable &t = pk::table_for(src_rate, dst_rate);
    for (int64_t i = 0; i < lim; ++i) {
        const int64_t num = i * t.down, center = num / t.up;
        const double *w = t.w.data() + (size_t)(num - center * t.up) * pk::RS_TAPS;
        volatile double sum = 0.0, wsum = 0.0;             // (volatile: keep the products un-fused on FMA-capable hosts)
        for (int k = 0; k < pk::RS_TAPS; ++k) {
            const int64_t j = center - (pk::RS_HALF - 1) + k;
            if (j < 0 || j >= n) continue;
            const double prod = (double)in[j] * w[k];
            sum = sum + prod;
            wsum = wsum + w[k];
        }
        out[i] = wsum > 1e-10 ? (float)(sum / wsum) : 0.0f;
    }
    return m;
}

}  // extern "C"
