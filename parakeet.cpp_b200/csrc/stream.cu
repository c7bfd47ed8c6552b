// stream.cu -- kernels of the STREAMING path (eou-120m, SURVEY.md section 8f row 2; BASELINE configs[3]), many
// streams advanced in lock step, one 160 ms chunk per stream and step.  What they replace in the reference:
//   StreamingAudioPreprocessor::process_chunk          src/audio.cpp:195-259   (stream_prep / mel stream mode / stream_post)
//   CausalConvSubsampling::forward_cached              src/streaming_encoder.cpp:339-385 (remainder cache: stream_post)
//   StreamingConformerAttention::forward_cached        src/streaming_encoder.cpp:160-272 (stream_attention_kernel)
//   CausalConformerConvModule::forward_cached          src/streaming_encoder.cpp:41-80   (stream_dwconv_kernel)
// The per-stream state lives in HBM: pre-emphasis carry + sample overlap, leftover mel frames, per layer a ring
// of the last att_context_left key / value rows and the last k-1 GLU outputs.  All lengths are known on the host
// (they depend only on the chunk sizes), which uploads one StreamPlan row per stream and step.
#include "kernels.h"

namespace pk {
namespace {

// ---- sample / mel-frame bookkeeping around the mel kernel -------------------------------------------------------
// before: sig = [overlap | pre-emphasised chunk] (audio.cpp:206-221; the carried sample feeds the first one),
//         mel_in = [leftover mel frames | (new frames, written by the mel kernel)]
__global__ void stream_prep_kernel(const float *__restrict__ chunk, const StreamPlan *__restrict__ plan, StreamState st,
                                   float *__restrict__ ssig, float *__restrict__ mel_in, int n_mels) {
    const int s = blockIdx.x;
    const StreamPlan p = plan[s];
    const float *x = chunk + p.chunk_off;
    const float *ovl = st.ovl + (size_t)s * STREAM_OVL_CAP;
    float *sig = ssig + p.sig_off;
    const float prev0 = st.last[s];
    for (int i = threadIdx.x; i < p.ovl_len + p.chunk_len; i += blockDim.x) {
        float v;
        if (i < p.ovl_len) {
            v = ovl[i];
        } else {
            const int k = i - p.ovl_len;
            v = x[k] - 0.97f * (k == 0 ? prev0 : x[k - 1]);
        }
        sig[i] = v;
    }
    const float *q = st.melq + (size_t)s * 8 * n_mels;
    float *mi = mel_in + (size_t)p.min_off * n_mels;
    for (int i = threadIdx.x; i < p.left * n_mels; i += blockDim.x) mi[i] = q[i];
}

// after: overlap = sig[consumed:] (audio.cpp:239-240), carry = last raw sample; the largest multiple of 8 mel
// frames goes to the packed encoder input, the rest (< 8 frames) back into the per-stream queue
// (streaming_encoder.cpp:348-385).
__global__ void stream_post_kernel(const float *__restrict__ chunk, const StreamPlan *__restrict__ plan, StreamState st,
                                   const float *__restrict__ ssig, const float *__restrict__ mel_in, int n_mels,
                                   float *__restrict__ feats) {
    const int s = blockIdx.x;
    const StreamPlan p = plan[s];
    const float *sig = ssig + p.sig_off;
    float *ovl = st.ovl + (size_t)s * STREAM_OVL_CAP;
    const int total = p.ovl_len + p.chunk_len, keep = total - p.consumed;       // keep < STREAM_OVL_CAP
    for (int i = threadIdx.x; i < keep; i += blockDim.x) ovl[i] = sig[p.consumed + i];
    if (threadIdx.x == 0 && p.chunk_len > 0) st.last[s] = chunk[p.chunk_off + p.chunk_len - 1];
    const float *mi = mel_in + (size_t)p.min_off * n_mels;
    if (p.take > 0) {
        float *f = feats + (size_t)p.feat_off * n_mels;
        for (int i = threadIdx.x; i < p.take * n_mels; i += blockDim.x) f[i] = mi[i];
    }
    float *q = st.melq + (size_t)s * 8 * n_mels;
    const int rest = p.left + p.nf - p.take;                                     // < 8
    for (int i = threadIdx.x; i < rest * n_mels; i += blockDim.x) q[i] = mi[(size_t)p.take * n_mels + i];
}

// Sortformer streams (Sortformer::diarize_chunk, sortformer.cpp:124-150): every chunk's log-mel is computed on its own
// (centred STFT), so no samples or pre-emphasis carry over; only CausalConvSubsampling's leftover frames
// (streaming_encoder.cpp:348-385) do.  Joined = [queue (left rows) | this chunk's nf rows at mel_new row p.min_off]: the
// first `take` rows go to the packed encoder input, the rest (< 8) back into the queue.
__global__ void diar_stream_join_kernel(const StreamPlan *__restrict__ plan, const float *__restrict__ mel_new,
                                        float *__restrict__ melq, int n_mels, float *__restrict__ feats) {
    const int s = blockIdx.x;
    const StreamPlan p = plan[s];
    float *q = melq + (size_t)s * 8 * n_mels;
    const float *nw = mel_new + (size_t)p.min_off * n_mels;
    const int lq = p.left * n_mels;
    if (p.take > 0) {
        float *f = feats + (size_t)p.feat_off * n_mels;
        for (int i = threadIdx.x; i < p.take * n_mels; i += blockDim.x) f[i] = i < lq ? q[i] : nw[i - lq];
        __syncthreads();                                    // the queue is read above, rewritten below
        const int rest = p.left + p.nf - p.take;            // < 8, all from this chunk (take >= 8 > left)
        const float *src = nw + (size_t)(p.take - p.left) * n_mels;
        for (int i = threadIdx.x; i < rest * n_mels; i += blockDim.x) q[i] = src[i];
    } else {
        for (int i = threadIdx.x; i < p.nf * n_mels; i += blockDim.x) q[lq + i] = nw[i];
    }
}

// ---- cached attention (streaming_encoder.cpp:160-272) ----------------------------------------------------------
// One block per (head, active stream).  Keys = [cached rows (ring, oldest first) | this chunk's rows]; scores
//     ((q_i + u) . k_j + (q_i + v) . PP[pos_j]) / sqrt(hd)
// with the reference's UN-shifted position term: the right-most kv columns of (q + v) . pos_proj(pos_emb(L + C))
// (:224-232), i.e. relative position pos_j = kv - L - C - j for every query row; no mask (the reference's float mask
// is inert on its CPU path, DESIGN.md); softmax; . V.  Afterwards the chunk's K / V rows enter the ring and the
// oldest rows beyond att_context_left drop out (:193-208).  fp32 throughout: 1-2 query rows per stream.
__global__ void __launch_bounds__(128)
stream_attention_kernel(const float *__restrict__ qkv, int ld_qkv, const int32_t *__restrict__ row_off,
                        const int32_t *__restrict__ act_stream, const int32_t *__restrict__ cache_len,
                        const int32_t *__restrict__ ring_start, float *__restrict__ kc, float *__restrict__ vc,
                        int L, int hd, int d_model, const float *__restrict__ pp, int tmax,
                        const float *__restrict__ bu, const float *__restrict__ bv, ActBuf out) {
    extern __shared__ float sm[];
    const int h = blockIdx.x, a = blockIdx.y, s = act_stream[a];
    const int r0 = row_off[a], C = row_off[a + 1] - r0;
    const int cl = cache_len[s], rs = ring_start[s], kv = cl + C;
    float *sk = sm;                               // [kv][hd + 1]
    float *sv = sk + (size_t)(L + C) * (hd + 1);  // [kv][hd + 1]
    float *sq = sv + (size_t)(L + C) * (hd + 1);  // [2][hd]  q + u, q + v of the current query
    float *sc = sq + 2 * hd;                      // [kv] scores
    float *kcs = kc + ((size_t)s * L) * d_model + h * hd, *vcs = vc + ((size_t)s * L) * d_model + h * hd;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < kv * hd; i += nt) {
        const int j = i / hd, c = i - j * hd;
        float kx, vx;
        if (j < cl) {
            const size_t o = (size_t)((rs + j) % L) * d_model + c;
            kx = kcs[o];
            vx = vcs[o];
        } else {
            const size_t o = (size_t)(r0 + j - cl) * ld_qkv + h * hd + c;
            kx = qkv[o + d_model];
            vx = qkv[o + 2 * d_model];
        }
        sk[j * (hd + 1) + c] = kx;
        sv[j * (hd + 1) + c] = vx;
    }
    const float scale = rsqrtf((float)hd);
    for (int i = 0; i < C; ++i) {
        __syncthreads();
        for (int c = tid; c < hd; c += nt) {
            const float q = qkv[(size_t)(r0 + i) * ld_qkv + h * hd + c];
            sq[c] = q + bu[h * hd + c];
            sq[hd + c] = q + bv[h * hd + c];
        }
        __syncthreads();
        for (int j = tid; j < kv; j += nt) {
            const float *prow = pp + (size_t)(kv - L - C - j + tmax - 1) * d_model + h * hd;
            float ac = 0.f, bd = 0.f;
            for (int c = 0; c < hd; ++c) {
                ac = fmaf(sq[c], sk[j * (hd + 1) + c], ac);
                bd = fmaf(sq[hd + c], prow[c], bd);
            }
            sc[j] = (ac + bd) * scale;
        }
        __syncthreads();
        // softmax over kv (max-subtracted, cpu_operations.cpp:3101-3231): thread j exponentiates its own score once; the
        // maximum and the (sequential, in key order) sum are recomputed by every thread from shared memory
        float mx = -INFINITY;
        for (int j = 0; j < kv; ++j) mx = fmaxf(mx, sc[j]);
        __syncthreads();
        for (int j = tid; j < kv; j += nt) sc[j] = expf(sc[j] - mx);
        __syncthreads();
        float sum = 0.f;
        for (int j = 0; j < kv; ++j) sum += sc[j];
        const float inv = 1.0f / sum;
        for (int c = tid; c < hd; c += nt) {
            float o = 0.f;
            for (int j = 0; j < kv; ++j) o = fmaf(sc[j] * inv, sv[j * (hd + 1) + c], o);
            store_act(out, (size_t)(r0 + i) * d_model + h * hd + c, o);
        }
    }
    __syncthreads();
    // ring update: logical row cl + i of the key list goes to slot (rs + cl + i) % L; when kv > L the host advances
    // ring_start by kv - L (the overwritten slots are exactly the dropped oldest rows).  C > L keeps the last L rows.
    const int first = C > L ? C - L : 0;
    for (int i = tid; i < (C - first) * hd; i += nt) {
        const int r = first + i / hd, c = i % hd;
        const size_t o = (size_t)((rs + cl + r) % L) * d_model + c;
        kcs[o] = sk[(cl + r) * (hd + 1) + c];
        vcs[o] = sv[(cl + r) * (hd + 1) + c];
    }
}

// ---- cached causal depthwise conv + folded BatchNorm + SiLU (streaming_encoder.cpp:41-80) ----------------------
// seq = [k-1 cached GLU outputs | C new]; y[t] = bias + sum_j w[j] seq[t + j] (no padding); cache = last k-1 of seq.
// One block per active stream, one thread per channel.
template <int KS>
__global__ void stream_dwconv_kernel(const float *__restrict__ glu, const int32_t *__restrict__ row_off,
                                     const int32_t *__restrict__ act_stream, float *__restrict__ cache, int d,
                                     const float *__restrict__ w, const float *__restrict__ bias, ActBuf out) {
    const int a = blockIdx.x, s = act_stream[a];
    const int r0 = row_off[a], C = row_off[a + 1] - r0;
    float *cs = cache + (size_t)s * (KS - 1) * d;
    for (int ch = threadIdx.x; ch < d; ch += blockDim.x) {
        float win[KS];                       // sliding window seq[t .. t + KS - 1]
#pragma unroll
        for (int j = 0; j < KS - 1; ++j) win[j] = cs[(size_t)j * d + ch];
        float wk[KS];
#pragma unroll
        for (int j = 0; j < KS; ++j) wk[j] = w[(size_t)ch * KS + j];
        const float b = bias[ch];
        for (int t = 0; t < C; ++t) {
            win[KS - 1] = glu[(size_t)(r0 + t) * d + ch];
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < KS; ++j) acc = fmaf(wk[j], win[j], acc);
            acc += b;
            store_act(out, (size_t)(r0 + t) * d + ch, siluf_(acc));
#pragma unroll
            for (int j = 0; j < KS - 1; ++j) win[j] = win[j + 1];
        }
#pragma unroll
        for (int j = 0; j < KS - 1; ++j) cs[(size_t)j * d + ch] = win[j];
    }
}

}  // namespace

void launch_stream_prep(const float *chunk, const StreamPlan *plan, StreamState st, int n_streams, float *ssig, float *mel_in,
                        int n_mels, cudaStream_t s) {
    stream_prep_kernel<<<dim3(n_streams), dim3(256), 0, s>>>(chunk, plan, st, ssig, mel_in, n_mels);
}
void launch_stream_post(const float *chunk, const StreamPlan *plan, StreamState st, int n_streams, const float *ssig,
                        const float *mel_in, int n_mels, float *feats, cudaStream_t s) {
    stream_post_kernel<<<dim3(n_streams), dim3(256), 0, s>>>(chunk, plan, st, ssig, mel_in, n_mels, feats);
}

void launch_diar_stream_join(const StreamPlan *plan, const float *mel_new, float *melq, int n_streams, int n_mels, float *feats,
                             cudaStream_t s) {
    diar_stream_join_kernel<<<dim3(n_streams), dim3(256), 0, s>>>(plan, mel_new, melq, n_mels, feats);
}

size_t stream_attention_smem(int L, int Cmax, int hd) { return sizeof(float) * ((size_t)2 * (L + Cmax) * (hd + 1) + 2 * hd + L + Cmax); }

bool launch_stream_attention(const float *qkv, int ld_qkv, const int32_t *row_off, const int32_t *act_stream, int n_active,
                             int max_C, const int32_t *cache_len, const int32_t *ring_start, float *kc, float *vc, int L,
                             int n_heads, int hd, int d_model, const float *pp, int tmax, const float *bu, const float *bv,
                             ActBuf out, cudaStream_t s) {
    const size_t smem = stream_attention_smem(L, max_C, hd);
    if (smem > 200 * 1024) return false;
    static PerDeviceFlag attr_flag;
    size_t &attr = attr_flag.cur_size();
    if (smem > attr) {
        if (cudaFuncSetAttribute(stream_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return false;
        attr = smem;
    }
    stream_attention_kernel<<<dim3(n_heads, n_active), dim3(128), smem, s>>>(qkv, ld_qkv, row_off, act_stream, cache_len, ring_start, kc, vc,
                                                                      L, hd, d_model, pp, tmax, bu, bv, out);
    return true;
}

bool launch_stream_dwconv(const float *glu, const int32_t *row_off, const int32_t *act_stream, int n_active, float *cache, int d,
                          int ks, const float *w, const float *bias, ActBuf out, cudaStream_t s) {
    if (ks != 9) return false;
    stream_dwconv_kernel<9><<<dim3(n_active), dim3(256), 0, s>>>(glu, row_off, act_stream, cache, d, w, bias, out);
    return true;
}

}  // namespace pk
