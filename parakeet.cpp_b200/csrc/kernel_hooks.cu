// kernel_hooks.cu -- pk_kernel_*: run ONE launcher of the hot path exactly as the engine calls it, on caller-supplied host
// fp32 arrays, and hand back every output buffer whole (tests/test_kernels_fp64.py checks them against float64 math).
//
// Every device output buffer sits between two guard bands of kGuard bytes, and guards and output are pre-filled with 0xFF
// bytes (NaN in fp32 and in bf16).  Each hook returns the number of guard bytes that changed in *guard_bad; elements the
// kernel must not write come back still holding the pattern, so the caller can check the exact set of written elements.
// bf16 planes come back widened to fp32 (exact).  A private stream, synchronous; nothing is cached between calls.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/parakeet_b200.h"
#include "kernels.h"

using namespace pk;

namespace {

constexpr size_t kGuard = (size_t)64 << 10;

// Device buffers of one hook call; freed (and the stream destroyed) on scope exit.
struct HookCtx {
    cudaStream_t st = nullptr;
    std::vector<void *> ptrs;
    struct Guarded {
        uint8_t *base;
        size_t bytes;
    };
    std::vector<Guarded> outs;
    bool ok = true;

    explicit HookCtx(int device) {
        ok = cudaSetDevice(device) == cudaSuccess && cudaStreamCreate(&st) == cudaSuccess;   // blocking: ordered after the memsets and copies
    }
    ~HookCtx() {
        if (st) cudaStreamSynchronize(st);
        for (void *p : ptrs) cudaFree(p);
        if (st) cudaStreamDestroy(st);
    }
    void *alloc(size_t bytes) {
        void *p = nullptr;
        if (cudaMalloc(&p, bytes < 16 ? 16 : bytes) != cudaSuccess) {
            ok = false;
            return nullptr;
        }
        ptrs.push_back(p);
        return p;
    }
    template <typename T>
    T *upload(const T *h, size_t n) {
        T *d = static_cast<T *>(alloc(n * sizeof(T)));
        if (d && h && n && cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) ok = false;
        return d;
    }
    // output buffer of `bytes` inside [guard | bytes | guard], all 0xFF
    template <typename T>
    T *guarded(size_t n) {
        const size_t bytes = n * sizeof(T);
        uint8_t *b = static_cast<uint8_t *>(alloc(bytes + 2 * kGuard));
        if (!b) return nullptr;
        if (cudaMemset(b, 0xFF, bytes + 2 * kGuard) != cudaSuccess) ok = false;
        outs.push_back({b, bytes});
        return reinterpret_cast<T *>(b + kGuard);
    }
    bool sync() { return ok && cudaStreamSynchronize(st) == cudaSuccess && cudaGetLastError() == cudaSuccess; }
    int64_t guard_bad() {
        int64_t bad = 0;
        std::vector<uint8_t> h(kGuard);
        for (const Guarded &g : outs)
            for (const uint8_t *p : {g.base, g.base + kGuard + g.bytes}) {
                if (cudaMemcpy(h.data(), p, kGuard, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
                for (uint8_t v : h) bad += v != 0xFF;
            }
        return bad;
    }
    pk_status finish(int64_t *guard_bad_out) {
        if (!sync()) return PK_ERR_CUDA;
        const int64_t gb = guard_bad();
        if (gb < 0) return PK_ERR_CUDA;
        if (guard_bad_out) *guard_bad_out = gb;
        return PK_OK;
    }
};

bool fetch_f32(float *host, const float *dev, size_t n) {
    return !host || cudaMemcpy(host, dev, n * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess;
}
bool fetch_bf16(float *host, const bf16 *dev, size_t n) {
    if (!host) return true;
    std::vector<bf16> h(n);
    if (n && cudaMemcpy(h.data(), dev, n * sizeof(bf16), cudaMemcpyDeviceToHost) != cudaSuccess) return false;
    for (size_t i = 0; i < n; ++i) host[i] = __bfloat162float(h[i]);
    return true;
}

int max_len(const int32_t *row_off, int n_utt) {
    int m = 0;
    for (int i = 0; i < n_utt; ++i) m = std::max(m, row_off[i + 1] - row_off[i]);
    return m;
}
bool offsets_ok(const int32_t *row_off, int n_utt, int rows_total) {
    if (!row_off || n_utt < 1 || row_off[0] < 0 || row_off[n_utt] > rows_total) return false;
    for (int i = 0; i < n_utt; ++i)
        if (row_off[i + 1] < row_off[i]) return false;
    return true;
}

bool is_act_kind(int k) { return k == EPI_BIAS_RELU_ACT || k == EPI_BIAS_SILU_ACT || k == EPI_BIAS_ACT; }

// pk_kernel_attention (band 0, 0: full attention, the table covers every utterance) and pk_kernel_attention_local (a band:
// the table covers -W..W, W = max(left, right), and sits between two NaN rows)
pk_status attention_hook(int device, int kernel, int math, int n_utt, const int32_t *row_off, int rows_total, int d_model, int n_heads,
                         int tmax, int left, int right, const float *qkv, const float *pp, const float *pos_u, const float *pos_v,
                         float *ctx_f32, float *ctx_hi, float *ctx_lo, int64_t *guard_bad) {
    if (kernel < 0 || kernel > 1 || !offsets_ok(row_off, n_utt, rows_total) || n_heads < 1 || d_model % n_heads || tmax < 1 || !qkv || !pp ||
        !pos_u || !pos_v || left < 0 || right < 0)
        return PK_ERR_INVALID;
    const bool band = left > 0 || right > 0;
    const int hd = d_model / n_heads, maxT = max_len(row_off, n_utt);
    if (maxT < 1 || (band ? std::max(left, right) >= tmax : maxT > tmax)) return PK_ERR_INVALID;
    // the output is what the engine's ctx buffer holds in that math mode: fp32, or bf16 hi (| lo) planes
    const bool f32 = math == PK_MATH_FP32;
    if (f32 ? (kernel != 0 || !ctx_f32) : (!ctx_hi || (math == PK_MATH_BF16X3) != (ctx_lo != nullptr))) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const int d = d_model, NP = 2 * tmax - 1;
    const size_t n_o = (size_t)rows_total * d;
    int32_t *doff = cx.upload(row_off, n_utt + 1);
    float *dqkv = cx.upload(qkv, (size_t)rows_total * 3 * d), *dpp;
    if (band) {              // [NaN row | table | NaN row]
        std::vector<float> h((size_t)(NP + 2) * d, NAN);
        memcpy(&h[d], pp, (size_t)NP * d * sizeof(float));
        dpp = cx.upload(h.data(), h.size());
        if (dpp) dpp += d;
    } else {
        dpp = cx.upload(pp, (size_t)NP * d);
    }
    float *du = cx.upload(pos_u, d), *dv = cx.upload(pos_v, d);
    ActBuf out;
    out.f32 = f32 ? cx.guarded<float>(n_o) : nullptr;
    out.hi = f32 ? nullptr : cx.guarded<bf16>(n_o);
    out.lo = ctx_lo ? cx.guarded<bf16>(n_o) : nullptr;
    if (!cx.ok) return PK_ERR_CUDA;
    bool launched;
    if (kernel == 0) {
        launched = launch_relpos_attention(dqkv, 3 * d, doff, n_utt, maxT, n_heads, hd, dpp, tmax, left, right, du, dv, d, out, cx.st);
    } else {
        // the EPI_QKV_ACT epilogue's layout: q fp32 [M, d], k | v bf16 planes [M, 2 d]; the position table split once at load
        std::vector<float> hq((size_t)rows_total * d), hkv((size_t)rows_total * 2 * d);
        for (int r = 0; r < rows_total; ++r) {
            memcpy(&hq[(size_t)r * d], qkv + (size_t)r * 3 * d, (size_t)d * 4);
            memcpy(&hkv[(size_t)r * 2 * d], qkv + (size_t)r * 3 * d + d, (size_t)2 * d * 4);
        }
        float *dq32 = cx.upload(hq.data(), hq.size()), *dkv = cx.upload(hkv.data(), hkv.size());
        bf16 *kvh = static_cast<bf16 *>(cx.alloc(hkv.size() * 2)), *kvl = static_cast<bf16 *>(cx.alloc(hkv.size() * 2));
        // the planes keep the NaN rows around a band's table (the split of NaN is NaN)
        const int pad = band ? 1 : 0;
        const size_t np_all = (size_t)(NP + 2 * pad) * d;
        bf16 *pph = static_cast<bf16 *>(cx.alloc(np_all * 2)), *ppl = static_cast<bf16 *>(cx.alloc(np_all * 2));
        if (!cx.ok) return PK_ERR_CUDA;
        ActBuf skv; skv.hi = kvh; skv.lo = kvl;
        ActBuf spp; spp.hi = pph; spp.lo = ppl;
        launch_split(dkv, hkv.size(), skv, cx.st);
        launch_split(dpp - (size_t)pad * d, np_all, spp, cx.st);
        launched = launch_relpos_attention_tc(dq32, du, dv, kvh, kvl, 2 * d, doff, n_utt, maxT, n_heads, hd, pph + (size_t)pad * d,
                                              ppl + (size_t)pad * d, tmax, left, right, d, out, cx.st);
    }
    if (!launched) return PK_ERR_INVALID;
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    if (out.f32 && !fetch_f32(ctx_f32, out.f32, n_o)) return PK_ERR_CUDA;
    if (out.hi && !fetch_bf16(ctx_hi, out.hi, n_o)) return PK_ERR_CUDA;
    if (out.lo && !fetch_bf16(ctx_lo, out.lo, n_o)) return PK_ERR_CUDA;
    return PK_OK;
}

}  // namespace

extern "C" {

pk_status pk_kernel_gemm(int device, int path, int math, int cluster, int M, int N, int K, int epi_kind, int qcols, int ldo, float alpha,
                         int in_place, const float *A, const float *W, const float *bias, const float *resid, float *out_f32,
                         float *out_hi, float *out_lo, int64_t *guard_bad) {
    if (path < 0 || path > 2 || epi_kind < EPI_BIAS_F32 || epi_kind > EPI_QKV_ACT || M < 1 || N < 1 || K < 1 || !A || !W) return PK_ERR_INVALID;
    if (math != PK_MATH_BF16X3 && math != PK_MATH_BF16X1 && math != PK_MATH_FP32) return PK_ERR_INVALID;
    if ((path == 0) != (math == PK_MATH_FP32)) return PK_ERR_INVALID;
    if (path != 0 && K % 64 != 0) return PK_ERR_INVALID;
    if (path == 2 && M > 128) return PK_ERR_INVALID;
    if (cluster != 1 && (path != 1 || math != PK_MATH_BF16X3 || !gemm_tc_cluster_supported(N, epi_kind, cluster))) return PK_ERR_INVALID;
    const bool qkv = epi_kind == EPI_QKV_ACT, glu = epi_kind == EPI_GLU_F32, resid_k = epi_kind == EPI_RESID_F32;
    if (qkv && (path == 0 || qcols <= 0 || qcols % 16 != 0 || qcols >= N)) return PK_ERR_INVALID;
    if (glu && (N & 1)) return PK_ERR_INVALID;
    const int n_out = glu ? N / 2 : qkv ? N - qcols : N;    // columns of the [M, ldo] output
    if (ldo < n_out || (resid_k && !resid) || (in_place && !resid_k)) return PK_ERR_INVALID;
    // outputs: fp32 [M, ldo] (q [M, qcols] for QKV) and, for the act kinds off fp32 math, bf16 planes [M, ldo]
    const bool planes = (is_act_kind(epi_kind) || qkv) && path != 0;
    if ((!planes && !out_f32) || (planes && !out_hi) || (qkv && !out_f32)) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t n_o = (size_t)M * ldo, n_f = qkv ? (size_t)M * qcols : n_o;
    float *dA = cx.upload(A, (size_t)M * K), *dW = cx.upload(W, (size_t)N * K), *db = bias ? cx.upload(bias, N) : nullptr;
    float *of = (planes && !qkv) ? nullptr : cx.guarded<float>(n_f);
    bf16 *oh = planes ? cx.guarded<bf16>(n_o) : nullptr, *ol = planes && out_lo ? cx.guarded<bf16>(n_o) : nullptr;
    float *dr = nullptr;
    if (resid_k) {
        if (in_place) {          // out_f32 starts as the residual and aliases it, as in pk_engine::run_blocks
            if (cudaMemcpy(of, resid, n_o * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return PK_ERR_CUDA;
            dr = of;
        } else {
            dr = cx.upload(resid, n_o);
        }
    }
    if (!cx.ok) return PK_ERR_CUDA;
    EpiParams ep;
    ep.kind = epi_kind; ep.bias = db; ep.ldo = ldo; ep.resid = dr; ep.alpha = alpha; ep.qcols = qkv ? qcols : 0;
    ep.out_f32 = of;
    if (planes) { ep.act.hi = oh; ep.act.lo = ol; }
    else if (is_act_kind(epi_kind)) ep.act.f32 = of;      // fp32 math: the activation is plain fp32
    const bool split3 = math == PK_MATH_BF16X3;
    if (path == 0) {
        launch_gemm_simt(dA, K, dW, K, M, N, K, ep, cx.st);
    } else {
        bf16 *Ah = static_cast<bf16 *>(cx.alloc((size_t)M * K * 2)), *Al = static_cast<bf16 *>(cx.alloc((size_t)M * K * 2));
        bf16 *Wh = static_cast<bf16 *>(cx.alloc((size_t)N * K * 2)), *Wl = static_cast<bf16 *>(cx.alloc((size_t)N * K * 2));
        if (!cx.ok) return PK_ERR_CUDA;
        ActBuf sa; sa.hi = Ah; sa.lo = Al;
        ActBuf sw; sw.hi = Wh; sw.lo = Wl;
        launch_split(dA, (size_t)M * K, sa, cx.st);
        launch_split(dW, (size_t)N * K, sw, cx.st);
        if (path == 2) {          // the few-row kernel, twice: its tickets must come back to zero
            const size_t ws_floats = (size_t)2 << 20;
            float *ws = static_cast<float *>(cx.alloc(ws_floats * sizeof(float)));
            unsigned int *tk = static_cast<unsigned int *>(cx.alloc(1024 * sizeof(unsigned int)));
            if (!cx.ok || cudaMemsetAsync(tk, 0, 1024 * sizeof(unsigned int), cx.st) != cudaSuccess) return PK_ERR_CUDA;
            int sms = 0;
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
            for (int rep = 0; rep < 2; ++rep) {
                // in place, the first launch has already added to the residual: start the second from it again
                if (rep && in_place && cudaMemcpyAsync(of, resid, n_o * sizeof(float), cudaMemcpyHostToDevice, cx.st) != cudaSuccess)
                    return PK_ERR_CUDA;
                if (launch_gemm_skinny(Ah, Al, K, Wh, Wl, M, N, K, split3, ep, ws, ws_floats, tk, 1024, sms,
                                       cx.st) != cudaSuccess)
                    return PK_ERR_CUDA;
            }
            std::vector<unsigned int> htk(1024);
            if (!cx.sync() || cudaMemcpy(htk.data(), tk, 1024 * sizeof(unsigned int), cudaMemcpyDeviceToHost) != cudaSuccess) return PK_ERR_CUDA;
            for (unsigned int t : htk)
                if (t != 0) return PK_ERR_CUDA;
        } else {
            TcOperand ta, tw, ta_sl;
            if (!make_tc_operand(&ta, Ah, Al, M, K, 128) || !make_tc_operand(&tw, Wh, Wl, N, K, tc_tile_n(N)))
                return PK_ERR_CUDA;
            if (cluster > 1 && !make_tc_operand(&ta_sl, Ah, Al, M, K, 128 / cluster)) return PK_ERR_CUDA;
            if (launch_gemm_tc(ta, tw, M, N, K, split3, ep, cx.st, cluster, cluster > 1 ? &ta_sl : nullptr) != cudaSuccess) return PK_ERR_CUDA;
        }
    }
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    if (of && !fetch_f32(out_f32, of, n_f)) return PK_ERR_CUDA;
    if (oh && !fetch_bf16(out_hi, oh, n_o)) return PK_ERR_CUDA;
    if (ol && !fetch_bf16(out_lo, ol, n_o)) return PK_ERR_CUDA;
    return PK_OK;
}

pk_status pk_kernel_attention(int device, int kernel, int math, int n_utt, const int32_t *row_off, int rows_total, int d_model, int n_heads,
                              int tmax, const float *qkv, const float *pp, const float *pos_u, const float *pos_v, float *ctx_f32,
                              float *ctx_hi, float *ctx_lo, int64_t *guard_bad) {
    return attention_hook(device, kernel, math, n_utt, row_off, rows_total, d_model, n_heads, tmax, 0, 0, qkv, pp, pos_u, pos_v, ctx_f32,
                          ctx_hi, ctx_lo, guard_bad);
}

pk_status pk_kernel_attention_local(int device, int kernel, int math, int n_utt, const int32_t *row_off, int rows_total, int d_model,
                                    int n_heads, int tmax, int left, int right, const float *qkv, const float *pp, const float *pos_u,
                                    const float *pos_v, float *ctx_f32, float *ctx_hi, float *ctx_lo, int64_t *guard_bad) {
    if (left < 0 || right < 0 || (left == 0 && right == 0)) return PK_ERR_INVALID;
    return attention_hook(device, kernel, math, n_utt, row_off, rows_total, d_model, n_heads, tmax, left, right, qkv, pp, pos_u, pos_v,
                          ctx_f32, ctx_hi, ctx_lo, guard_bad);
}

pk_status pk_kernel_layernorm(int device, int M, int d, const float *x, const float *w1, const float *b1, const float *w2, const float *b2,
                              int want_f32, int planes, float *y1_f32, float *act_f32, float *hi, float *lo, int64_t *guard_bad) {
    if (M < 1 || d < 4 || d > 1024 || d % 4 || !x || !w1 || !b1 || (!w2) != (!b2) || planes < 0 || planes > 3) return PK_ERR_INVALID;
    if ((want_f32 && !y1_f32) || (planes == 3 && !act_f32) || ((planes == 1 || planes == 2) && !hi) || (planes == 2 && !lo)) return PK_ERR_INVALID;
    if (w2 && (!want_f32 || planes == 0)) return PK_ERR_INVALID;    // the chained form: y1 in place, LN2(y1) as the operand
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t n = (size_t)M * d;
    float *dw1 = cx.upload(w1, d), *db1 = cx.upload(b1, d), *dw2 = w2 ? cx.upload(w2, d) : nullptr, *db2 = b2 ? cx.upload(b2, d) : nullptr;
    float *y1 = want_f32 ? cx.guarded<float>(n) : nullptr;
    float *dx;
    if (y1) {                 // LN1 written in place over its input, as pk_engine::run_blocks does
        if (cudaMemcpy(y1, x, n * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return PK_ERR_CUDA;
        dx = y1;
    } else {
        dx = cx.upload(x, n);
    }
    ActBuf act;
    if (planes == 3) act.f32 = cx.guarded<float>(n);
    if (planes == 1 || planes == 2) act.hi = cx.guarded<bf16>(n);
    if (planes == 2) act.lo = cx.guarded<bf16>(n);
    if (!cx.ok) return PK_ERR_CUDA;
    ActBuf none;
    if (w2) launch_layernorm(dx, M, d, dw1, db1, y1, none, dw2, db2, act, cx.st);
    else launch_layernorm(dx, M, d, dw1, db1, y1, act, nullptr, nullptr, none, cx.st);
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    if (!fetch_f32(y1 ? y1_f32 : nullptr, y1, n) || (act.f32 && !fetch_f32(act_f32, act.f32, n)) || (act.hi && !fetch_bf16(hi, act.hi, n)) ||
        (act.lo && !fetch_bf16(lo, act.lo, n)))
        return PK_ERR_CUDA;
    return PK_OK;
}

pk_status pk_kernel_dwconv(int device, int math, int n_utt, const int32_t *row_off, int rows_total, int d, int ks, const float *g,
                           const float *w_tapmajor, const float *bias, float *out_f32, float *hi, float *lo, int64_t *guard_bad) {
    if (!offsets_ok(row_off, n_utt, rows_total) || d < 4 || d % 4 || ks < 1 || !g || !w_tapmajor || !bias) return PK_ERR_INVALID;
    const bool f32 = math == PK_MATH_FP32;
    if (f32 ? !out_f32 : (!hi || (math == PK_MATH_BF16X3) != (lo != nullptr))) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t n = (size_t)rows_total * d;
    int32_t *doff = cx.upload(row_off, n_utt + 1);
    float *dg = cx.upload(g, n), *dw = cx.upload(w_tapmajor, (size_t)ks * d), *db = cx.upload(bias, d);
    ActBuf out;
    out.f32 = f32 ? cx.guarded<float>(n) : nullptr;
    out.hi = f32 ? nullptr : cx.guarded<bf16>(n);
    out.lo = lo ? cx.guarded<bf16>(n) : nullptr;
    if (!cx.ok) return PK_ERR_CUDA;
    if (!launch_dwconv_bn_silu(dg, doff, n_utt, max_len(row_off, n_utt), d, ks, dw, db, out, cx.st)) return PK_ERR_INVALID;
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    if ((out.f32 && !fetch_f32(out_f32, out.f32, n)) || (out.hi && !fetch_bf16(hi, out.hi, n)) || (out.lo && !fetch_bf16(lo, out.lo, n)))
        return PK_ERR_CUDA;
    return PK_OK;
}

pk_status pk_kernel_ctc_argmax(int device, int M, int V, int ld, const float *logits, int32_t *best, float *conf, float *logprobs,
                               int64_t *guard_bad) {
    if (M < 1 || V < 1 || ld < V || !logits || !best || !conf) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    float *dl = cx.upload(logits, (size_t)M * ld);
    int32_t *db = cx.guarded<int32_t>(M);
    float *dc = cx.guarded<float>(M), *dlp = logprobs ? cx.guarded<float>((size_t)M * V) : nullptr;
    if (!cx.ok) return PK_ERR_CUDA;
    launch_ctc_frame_argmax(dl, M, V, ld, db, dc, dlp, cx.st);
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    if (cudaMemcpy(best, db, (size_t)M * 4, cudaMemcpyDeviceToHost) != cudaSuccess || !fetch_f32(conf, dc, M) ||
        (dlp && !fetch_f32(logprobs, dlp, (size_t)M * V)))
        return PK_ERR_CUDA;
    return PK_OK;
}

// bin / bout: the boosted form (pk_kernel_tdt_decode_boosted), else null
static pk_status tdt_hook_run(int device, const pk_tdt_hook_in *in, pk_tdt_hook_out *out, int64_t *guard_bad, const pk_tdt_boost_hook_in *bin,
                              pk_tdt_boost_hook_out *bout) {
    if (!in || !out) return PK_ERR_INVALID;
    const int P = in->P, J = in->J, V = in->V, D = in->n_dur, L = in->L, n = in->n_utt;
    if (P < 32 || P % 32 || J < 32 || J % 32 || V < 2 || D < 0 || D > 8 || L < 1 || L > PK_MAX_LSTM || n < 1 || in->cap < 1 ||
        in->max_steps < 1 || (D == 0 && in->max_sym < 1) || !offsets_ok(in->row_off, n, in->rows) || !in->EP || !in->G0 || !in->W_p ||
        !in->W_out || !in->b_out || (in->cluster != 0 && in->cluster != 2 && in->cluster != 4) || in->max_ctas < 0)
        return PK_ERR_INVALID;
    for (int l = 0; l < L; ++l)
        if (!in->W_hh[l] || (l > 0 && (!in->W_ih[l] || !in->b_ih[l]))) return PK_ERR_INVALID;
    if (in->carry && (!in->h0 || !in->c0 || !in->tok0 || !in->frame_base)) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const int Bpad = (n + 31) / 32 * 32, cap = in->cap, NO = V + D;
    const size_t HS = (size_t)P * Bpad;
    TdtParams p{};
    p.P = P; p.J = J; p.V = V; p.D = D; p.L = L; p.Bpad = Bpad; p.n_utt = n; p.cap = cap; p.max_steps = in->max_steps;
    p.n_dur = D; p.max_sym = in->max_sym;
    for (int i = 0; i < 8; ++i) p.durations[i] = in->durations[i];
    p.EP = cx.upload(in->EP, (size_t)in->rows * J);
    p.row_off = cx.upload(in->row_off, n + 1);
    p.G0 = cx.upload(in->G0, (size_t)V * 4 * P);
    // weights as the engine loads them: unit-major LSTM rows, every matrix split into [hi: K][lo: K] bf16 rows
    auto split = [&](const float *w, int rows, int K) {
        float *dw = cx.upload(w, (size_t)rows * K);
        bf16 *s = static_cast<bf16 *>(cx.alloc((size_t)rows * 2 * K * sizeof(bf16)));
        if (s) launch_tdt_split_rows(dw, rows, K, s, cx.st);
        return static_cast<const bf16 *>(s);
    };
    std::vector<float> um((size_t)4 * P * P);
    for (int l = 0; l < L; ++l) {
        lstm_unit_major(in->W_hh[l], P, um.data());
        p.Whh[l] = split(um.data(), 4 * P, P);
        if (l > 0) {
            lstm_unit_major(in->W_ih[l], P, um.data());
            p.Wih[l] = split(um.data(), 4 * P, P);
            p.bih[l] = cx.upload(in->b_ih[l], (size_t)4 * P);
        }
    }
    p.Wp = split(in->W_p, J, P);
    p.Wout = split(in->W_out, NO, J);
    p.bout = cx.upload(in->b_out, NO);
    // h: bf16 [hi|lo][L][2][Bpad][P], zero except the carried state in plane 0
    bf16 *hb = cx.guarded<bf16>(2 * L * 2 * HS);
    bf16 *zb = cx.guarded<bf16>((size_t)2 * Bpad * J);
    {
        std::vector<float> h((size_t)L * 2 * HS, 0.f);
        if (in->carry)
            for (int l = 0; l < L; ++l)
                for (int b = 0; b < n; ++b) memcpy(&h[(size_t)l * 2 * HS + (size_t)b * P], in->h0 + ((size_t)l * n + b) * P, (size_t)P * 4);
        float *dh = cx.upload(h.data(), h.size());
        if (!cx.ok) return PK_ERR_CUDA;
        ActBuf sh; sh.hi = hb; sh.lo = hb + (size_t)L * 2 * HS;
        launch_split(dh, h.size(), sh, cx.st);
    }
    p.hbuf = reinterpret_cast<float *>(hb);
    p.z = reinterpret_cast<float *>(zb);
    p.tok = cx.guarded<int32_t>((size_t)n * (1 + cap));
    p.t_start = cx.guarded<int32_t>((size_t)n * cap);
    p.t_end = cx.guarded<int32_t>((size_t)n * cap);
    p.t_conf = cx.guarded<float>((size_t)n * cap);
    p.overflow = cx.guarded<int32_t>(n);
    constexpr int kMaxGrid = 256;           // launch_tdt_decode never plans a larger grid
    p.pl_max = static_cast<float *>(cx.alloc((size_t)3 * kMaxGrid * Bpad * sizeof(float)));
    p.pl_sum = static_cast<float *>(cx.alloc((size_t)3 * kMaxGrid * Bpad * sizeof(float)));
    p.key_lab = static_cast<unsigned long long *>(cx.alloc((size_t)3 * Bpad * 8));
    p.key_dur = static_cast<unsigned long long *>(cx.alloc((size_t)3 * Bpad * 8));
    p.bar = static_cast<unsigned int *>(cx.alloc(1024 * sizeof(unsigned int)));
    p.dbg = static_cast<long long *>(cx.alloc(8 * sizeof(long long)));
    if (in->carry) {
        p.carry = 1;
        std::vector<float> c((size_t)L * Bpad * P, 0.f);
        for (int l = 0; l < L; ++l)
            memcpy(&c[(size_t)l * Bpad * P], in->c0 + (size_t)l * n * P, (size_t)n * P * 4);
        p.c_state = cx.guarded<float>(c.size());
        p.tok_state = cx.guarded<int32_t>(n);
        p.frame_base = cx.upload(in->frame_base, n);
        if (!cx.ok || cudaMemcpy(p.c_state, c.data(), c.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
            cudaMemcpy(p.tok_state, in->tok0, (size_t)n * 4, cudaMemcpyHostToDevice) != cudaSuccess)
            return PK_ERR_CUDA;
    }
    const int BW = (V + 31) / 32;
    if (bin) {
        // one trie slot per row, as pk_set_boost_rows lays them out; the state on entry: the root, or the caller's active sets
        if (D == 0 || !bin->row_off || !bin->boost || (in->carry && (!bin->trie_active0 || !bin->trie_nact0))) return PK_ERR_INVALID;
        std::vector<int32_t> slots((size_t)n * BOOST_SLOT_INTS, 0), act((size_t)n * BOOST_MAX_ACTIVE, 0), nact(n, 1), first, tk, cd;
        std::vector<uint32_t> bits((size_t)n * BW, 0u);
        for (int b = 0; b < n; ++b) {
            int32_t *slot = &slots[(size_t)b * BOOST_SLOT_INTS], *tok = slot + BOOST_SLOT_NODES + 1, *child = tok + BOOST_SLOT_EDGES;
            if (bin->row_off[b + 1] < bin->row_off[b]) return PK_ERR_INVALID;
            if (bin->row_off[b + 1] > bin->row_off[b]) {
                if (!bin->phrase_ids || !bin->phrase_off || !boost_trie_csr(bin->phrase_ids, bin->phrase_off, bin->row_off[b], bin->row_off[b + 1], first, tk, cd))
                    return PK_ERR_INVALID;
                if ((int)first.size() - 1 > BOOST_SLOT_NODES) return PK_ERR_CAPACITY;
                memcpy(slot, first.data(), first.size() * 4);
                memcpy(tok, tk.data(), tk.size() * 4);
                memcpy(child, cd.data(), cd.size() * 4);
            }
            if (in->carry) {
                nact[b] = bin->trie_nact0[b];
                if (nact[b] < 1 || nact[b] > BOOST_MAX_ACTIVE) return PK_ERR_INVALID;
                memcpy(&act[(size_t)b * BOOST_MAX_ACTIVE], bin->trie_active0 + (size_t)b * BOOST_MAX_ACTIVE, (size_t)nact[b] * 4);
            }
            const int n_nodes = slot[0] == slot[1] ? 1 : (int)first.size() - 1;
            for (int a = 0; a < nact[b]; ++a) {
                const int node = act[(size_t)b * BOOST_MAX_ACTIVE + a];
                if (node < 0 || node >= n_nodes) return PK_ERR_INVALID;
                for (int e = slot[node]; e < slot[node + 1]; ++e)
                    if (tok[e] >= 0 && tok[e] < V) bits[(size_t)b * BW + (tok[e] >> 5)] |= 1u << (tok[e] & 31);
            }
        }
        BoostSlots bs;
        bs.slots = cx.upload(slots.data(), slots.size());
        bs.val = cx.upload(bin->boost, n);
        p.boost_on = 1;
        p.trie = bs.trie();
        // (the decode reads the bitmaps of all Bpad rows: the padding rows read zeros)
        p.boost_bits = cx.guarded<uint32_t>((size_t)Bpad * BW);
        p.trie_active = cx.guarded<int32_t>((size_t)n * BOOST_MAX_ACTIVE);
        p.trie_nact = cx.guarded<int32_t>(n);
        if (!cx.ok || cudaMemset(p.boost_bits, 0, (size_t)Bpad * BW * 4) != cudaSuccess) return PK_ERR_CUDA;
        if (in->carry) {
            // entries past a row's active set stay 0xFF: the kernel must not read them
            for (int b = 0; b < n; ++b)
                if (cudaMemcpy(p.trie_active + (size_t)b * BOOST_MAX_ACTIVE, &act[(size_t)b * BOOST_MAX_ACTIVE], (size_t)nact[b] * 4, cudaMemcpyHostToDevice) != cudaSuccess)
                    return PK_ERR_CUDA;
            if (cudaMemcpy(p.trie_nact, nact.data(), (size_t)n * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaMemcpy(p.boost_bits, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess)
                return PK_ERR_CUDA;
        }
    }
    if (!cx.ok || !cx.sync()) return PK_ERR_CUDA;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    TdtLaunchCtl ctl;
    ctl.cluster = in->cluster;
    ctl.no_stage = in->no_stage != 0;
    const cudaError_t ce = launch_tdt_decode(p, in->max_ctas ? std::min(in->max_ctas, sms) : sms, cx.st, &ctl);
    if (ce == cudaErrorLaunchOutOfResources && ctl.grid == 0) {
        cudaGetLastError();
        return PK_ERR_INVALID;               // (a forced cluster size that does not fit)
    }
    if (ce != cudaSuccess) return PK_ERR_CUDA;
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    out->grid = ctl.grid; out->cl = ctl.CL; out->upc = ctl.UPC; out->opc = ctl.OPC;
    out->out_in_smem = ctl.out_in_smem; out->wih_in_smem = ctl.wih_in_smem; out->staged_ih = ctl.staged_ih; out->wstage_rows = ctl.wstage_rows;
    long long dbg[8];
    if (cudaMemcpy(dbg, p.dbg, sizeof(dbg), cudaMemcpyDeviceToHost) != cudaSuccess) return PK_ERR_CUDA;
    out->steps = (int32_t)dbg[7];
    const int kb = (out->steps - 1) % 3, G = ctl.grid;
    auto fetch_i32 = [](int32_t *host, const int32_t *dev, size_t cnt) {
        return !host || cudaMemcpy(host, dev, cnt * 4, cudaMemcpyDeviceToHost) == cudaSuccess;
    };
    if (!fetch_i32(out->tok, p.tok, (size_t)n * (1 + cap)) || !fetch_i32(out->t_start, p.t_start, (size_t)n * cap) ||
        !fetch_i32(out->t_end, p.t_end, (size_t)n * cap) || !fetch_f32(out->t_conf, p.t_conf, (size_t)n * cap) ||
        !fetch_i32(out->overflow, p.overflow, n))
        return PK_ERR_CUDA;
    // h planes and z: drop the batch padding rows
    for (int pl = 0; pl < 2; ++pl) {
        float *dst = pl ? out->h_lo : out->h_hi;
        if (dst)
            for (int s = 0; s < L * 2; ++s)
                if (!fetch_bf16(dst + (size_t)s * n * P, hb + (size_t)pl * L * 2 * HS + (size_t)s * HS, (size_t)n * P)) return PK_ERR_CUDA;
        float *zd = pl ? out->z_lo : out->z_hi;
        if (!fetch_bf16(zd, zb + (size_t)pl * Bpad * J, (size_t)n * J)) return PK_ERR_CUDA;
    }
    std::vector<unsigned long long> keys(2 * (size_t)Bpad);
    std::vector<float> pm((size_t)G * Bpad), ps((size_t)G * Bpad);
    if (cudaMemcpy(keys.data(), p.key_lab + (size_t)kb * Bpad, (size_t)Bpad * 8, cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(keys.data() + Bpad, p.key_dur + (size_t)kb * Bpad, (size_t)Bpad * 8, cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(pm.data(), p.pl_max + (size_t)kb * G * Bpad, pm.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(ps.data(), p.pl_sum + (size_t)kb * G * Bpad, ps.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
        return PK_ERR_CUDA;
    for (int b = 0; b < n; ++b) {
        for (int which = 0; which < 2; ++which) {     // the packing of tdt.cu's pack_key
            const unsigned long long k = keys[(size_t)which * Bpad + b];
            uint32_t u = (uint32_t)(k >> 32);
            u = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
            float v;
            memcpy(&v, &u, 4);
            const int32_t idx = k ? (int32_t)(0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFu)) : -1;
            if (which == 0) {
                if (out->lab_val) out->lab_val[b] = v;
                if (out->lab_idx) out->lab_idx[b] = idx;
            } else {
                if (out->dur_val) out->dur_val[b] = v;
                if (out->dur_idx) out->dur_idx[b] = idx;
            }
        }
        if (out->lse) {
            double gmax = -INFINITY, s = 0.0;
            for (int q = 0; q < G; ++q) gmax = std::max(gmax, (double)pm[(size_t)q * Bpad + b]);
            for (int q = 0; q < G; ++q)
                if (pm[(size_t)q * Bpad + b] > -INFINITY) s += (double)ps[(size_t)q * Bpad + b] * std::exp((double)pm[(size_t)q * Bpad + b] - gmax);
            out->lse[b] = gmax + std::log(s);
        }
    }
    if (in->carry) {
        std::vector<float> c((size_t)L * Bpad * P);
        if (cudaMemcpy(c.data(), p.c_state, c.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess || !fetch_i32(out->tok_state, p.tok_state, n))
            return PK_ERR_CUDA;
        if (out->c_state)
            for (int l = 0; l < L; ++l) memcpy(out->c_state + (size_t)l * n * P, &c[(size_t)l * Bpad * P], (size_t)n * P * 4);
    }
    if (bout && (!fetch_i32(bout->trie_active, p.trie_active, (size_t)n * BOOST_MAX_ACTIVE) || !fetch_i32(bout->trie_nact, p.trie_nact, n) ||
                 !fetch_i32(reinterpret_cast<int32_t *>(bout->boost_bits), reinterpret_cast<const int32_t *>(p.boost_bits), (size_t)n * BW)))
        return PK_ERR_CUDA;
    return PK_OK;
}

pk_status pk_kernel_tdt_decode(int device, const pk_tdt_hook_in *in, pk_tdt_hook_out *out, int64_t *guard_bad) {
    return tdt_hook_run(device, in, out, guard_bad, nullptr, nullptr);
}

pk_status pk_kernel_tdt_decode_boosted(int device, const pk_tdt_boost_hook_in *in, pk_tdt_boost_hook_out *out, int64_t *guard_bad) {
    if (!in || !out) return PK_ERR_INVALID;
    return tdt_hook_run(device, &in->dec, &out->dec, guard_bad, in, out);
}

}  // extern "C"

namespace {

// the active-stream list of a streaming hook: distinct ids in [0, n_streams), row offsets over rows_total
bool streams_ok(int n_streams, int n_active, const int32_t *act, const int32_t *row_off, int rows_total) {
    if (n_streams < 1 || n_active < 1 || n_active > n_streams || !act || !offsets_ok(row_off, n_active, rows_total)) return false;
    std::vector<char> seen(n_streams, 0);
    for (int a = 0; a < n_active; ++a) {
        if (act[a] < 0 || act[a] >= n_streams || seen[act[a]]) return false;
        seen[act[a]] = 1;
    }
    return true;
}

// ctx / conv output in the engine's layout for the math mode: fp32, or bf16 hi (| lo) planes
bool act_out_ok(int math, const float *f32, const float *hi, const float *lo) {
    if (math == PK_MATH_FP32) return f32 != nullptr;
    if (math != PK_MATH_BF16X3 && math != PK_MATH_BF16X1) return false;
    return hi && (math == PK_MATH_BF16X3) == (lo != nullptr);
}

ActBuf guarded_act(HookCtx &cx, int math, size_t n, bool lo) {
    ActBuf o;
    if (math == PK_MATH_FP32) o.f32 = cx.guarded<float>(n);
    else o.hi = cx.guarded<bf16>(n);
    if (lo) o.lo = cx.guarded<bf16>(n);
    return o;
}

bool fetch_act(const ActBuf &o, float *f32, float *hi, float *lo, size_t n) {
    return (!o.f32 || fetch_f32(f32, o.f32, n)) && (!o.hi || fetch_bf16(hi, o.hi, n)) && (!o.lo || fetch_bf16(lo, o.lo, n));
}

// a guarded copy of host state (rings, conv caches) that the kernel updates in place
float *guarded_state(HookCtx &cx, const float *h, size_t n) {
    float *d = cx.guarded<float>(n);
    if (d && cudaMemcpy(d, h, n * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) cx.ok = false;
    return d;
}

}  // namespace

extern "C" {

pk_status pk_kernel_stream_attention(int device, int math, int n_streams, int n_active, const int32_t *act_stream, const int32_t *row_off,
                                     int rows_total, const int32_t *cache_len, const int32_t *ring_start, int L, int d_model, int n_heads,
                                     int tmax, const float *qkv, const float *pp, const float *pos_u, const float *pos_v, const float *kc,
                                     const float *vc, float *ctx_f32, float *ctx_hi, float *ctx_lo, float *kc_out, float *vc_out,
                                     int64_t *guard_bad) {
    if (!streams_ok(n_streams, n_active, act_stream, row_off, rows_total) || !cache_len || !ring_start || L < 1 || n_heads < 1 ||
        d_model % n_heads || !qkv || !pp || !pos_u || !pos_v || !kc || !vc || !kc_out || !vc_out || !act_out_ok(math, ctx_f32, ctx_hi, ctx_lo))
        return PK_ERR_INVALID;
    for (int s = 0; s < n_streams; ++s)
        if (cache_len[s] < 0 || cache_len[s] > L || ring_start[s] < 0 || ring_start[s] >= L) return PK_ERR_INVALID;
    const int maxC = max_len(row_off, n_active);
    if (maxC < 1 || L + maxC > tmax) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const int d = d_model;
    const size_t n_o = (size_t)rows_total * d, n_ring = (size_t)n_streams * L * d;
    int32_t *dact = cx.upload(act_stream, n_active), *doff = cx.upload(row_off, n_active + 1);
    int32_t *dcl = cx.upload(cache_len, n_streams), *drs = cx.upload(ring_start, n_streams);
    float *dqkv = cx.upload(qkv, (size_t)rows_total * 3 * d), *dpp = cx.upload(pp, (size_t)(2 * tmax - 1) * d);
    float *du = cx.upload(pos_u, d), *dv = cx.upload(pos_v, d);
    float *dkc = guarded_state(cx, kc, n_ring), *dvc = guarded_state(cx, vc, n_ring);
    ActBuf out = guarded_act(cx, math, n_o, ctx_lo != nullptr);
    if (!cx.ok) return PK_ERR_CUDA;
    if (!launch_stream_attention(dqkv, 3 * d, doff, dact, n_active, maxC, dcl, drs, dkc, dvc, L, n_heads, d / n_heads, d, dpp, tmax, du, dv,
                                 out, cx.st))
        return PK_ERR_INVALID;
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    if (!fetch_act(out, ctx_f32, ctx_hi, ctx_lo, n_o) || !fetch_f32(kc_out, dkc, n_ring) || !fetch_f32(vc_out, dvc, n_ring)) return PK_ERR_CUDA;
    return PK_OK;
}

pk_status pk_kernel_stream_dwconv(int device, int math, int n_streams, int n_active, const int32_t *act_stream, const int32_t *row_off,
                                  int rows_total, int d, int ks, const float *glu, const float *w, const float *bias, const float *cache,
                                  float *out_f32, float *hi, float *lo, float *cache_out, int64_t *guard_bad) {
    if (!streams_ok(n_streams, n_active, act_stream, row_off, rows_total) || d < 1 || ks < 2 || !glu || !w || !bias || !cache ||
        !cache_out || !act_out_ok(math, out_f32, hi, lo))
        return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t n_o = (size_t)rows_total * d, n_c = (size_t)n_streams * (ks - 1) * d;
    int32_t *dact = cx.upload(act_stream, n_active), *doff = cx.upload(row_off, n_active + 1);
    float *dg = cx.upload(glu, n_o), *dw = cx.upload(w, (size_t)d * ks), *db = cx.upload(bias, d);
    float *dc = guarded_state(cx, cache, n_c);
    ActBuf out = guarded_act(cx, math, n_o, lo != nullptr);
    if (!cx.ok) return PK_ERR_CUDA;
    if (!launch_stream_dwconv(dg, doff, dact, n_active, dc, d, ks, dw, db, out, cx.st)) return PK_ERR_INVALID;
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    if (!fetch_act(out, out_f32, hi, lo, n_o) || !fetch_f32(cache_out, dc, n_c)) return PK_ERR_CUDA;
    return PK_OK;
}

// Sortformer's transformer attention (attention_mha.cu) as the engine runs it in `math`: the fp32 kernel with PK_MATH_FP32,
// else the mma.sync kernel on q fp32 and k | v split into bf16 planes.  qkv [rows_total][3 d] fp32; ctx [rows_total][d] as
// the engine's transformer context buffer holds it (fp32 with PK_MATH_FP32, else bf16 hi | lo planes).
pk_status pk_kernel_mha(int device, int math, int n_utt, const int32_t *row_off, int rows_total, int d_model, int n_heads, const float *qkv,
                        float *ctx_f32, float *ctx_hi, float *ctx_lo, int64_t *guard_bad) {
    if (!offsets_ok(row_off, n_utt, rows_total) || n_heads < 1 || d_model % n_heads || !qkv) return PK_ERR_INVALID;
    const bool f32 = math == PK_MATH_FP32;
    if (f32 ? !ctx_f32 : (!ctx_hi || (math == PK_MATH_BF16X3) != (ctx_lo != nullptr))) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const int d = d_model;
    const size_t n_o = (size_t)rows_total * d;
    int32_t *doff = cx.upload(row_off, n_utt + 1);
    float *dqkv = cx.upload(qkv, (size_t)rows_total * 3 * d);
    ActBuf out;
    out.f32 = f32 ? cx.guarded<float>(n_o) : nullptr;
    out.hi = f32 ? nullptr : cx.guarded<bf16>(n_o);
    out.lo = ctx_lo ? cx.guarded<bf16>(n_o) : nullptr;
    if (!cx.ok) return PK_ERR_CUDA;
    bool launched;
    if (f32) {
        launched = launch_mha_attention(dqkv, 3 * d, doff, n_utt, max_len(row_off, n_utt), n_heads, d / n_heads, d, out, cx.st);
    } else {
        // the EPI_QKV_ACT epilogue's layout: q fp32 [M, d], k | v bf16 planes [M, 2 d]
        std::vector<float> hq((size_t)rows_total * d), hkv((size_t)rows_total * 2 * d);
        for (int r = 0; r < rows_total; ++r) {
            memcpy(&hq[(size_t)r * d], qkv + (size_t)r * 3 * d, (size_t)d * 4);
            memcpy(&hkv[(size_t)r * 2 * d], qkv + (size_t)r * 3 * d + d, (size_t)2 * d * 4);
        }
        float *dq32 = cx.upload(hq.data(), hq.size()), *dkv = cx.upload(hkv.data(), hkv.size());
        ActBuf skv;
        skv.hi = static_cast<bf16 *>(cx.alloc(hkv.size() * 2));
        skv.lo = math == PK_MATH_BF16X3 ? static_cast<bf16 *>(cx.alloc(hkv.size() * 2)) : nullptr;
        if (!cx.ok) return PK_ERR_CUDA;
        launch_split(dkv, hkv.size(), skv, cx.st);
        launched = launch_mha_attention_tc(dq32, skv.hi, skv.lo, 2 * d, doff, n_utt, max_len(row_off, n_utt), n_heads, d / n_heads, d, out, cx.st);
    }
    if (!launched) return PK_ERR_INVALID;
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    if (!fetch_f32(ctx_f32, out.f32, n_o) || (out.hi && !fetch_bf16(ctx_hi, out.hi, n_o)) || (out.lo && !fetch_bf16(ctx_lo, out.lo, n_o)))
        return PK_ERR_CUDA;
    return PK_OK;
}

// Sortformer's fused speaker head (speaker_head.cu): x [M][D], w1 [D][D] (first_hidden_, as stored), w2 [S][D] -> probs [M][S].
pk_status pk_kernel_speaker_head(int device, int M, int D, int S, const float *x, const float *w1, const float *b1, const float *w2,
                                 const float *b2, float *probs, int64_t *guard_bad) {
    if (M < 1 || D < 1 || S < 1 || !x || !w1 || !b1 || !w2 || !b2 || !probs) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    std::vector<float> w1t((size_t)D * D);
    for (int n = 0; n < D; ++n)
        for (int k = 0; k < D; ++k) w1t[(size_t)k * D + n] = w1[(size_t)n * D + k];
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    float *dx = cx.upload(x, (size_t)M * D), *dw1 = cx.upload(w1t.data(), w1t.size()), *db1 = cx.upload(b1, D);
    float *dw2 = cx.upload(w2, (size_t)S * D), *db2 = cx.upload(b2, S);
    float *dp = cx.guarded<float>((size_t)M * S);
    if (!cx.ok) return PK_ERR_CUDA;
    if (!launch_speaker_head(dx, M, D, S, dw1, db1, dw2, db2, dp, sms, cx.st)) return PK_ERR_INVALID;
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    return fetch_f32(probs, dp, (size_t)M * S) ? PK_OK : PK_ERR_CUDA;
}

}  // extern "C"

extern "C" pk_status pk_kernel_ctc_beam(int device, int n_utt, const int32_t *row_off, int rows, int V, const float *logprobs, int width,
                                        const pk_lm *lm, const pk_vocab *vocab, float alpha, float beta, int cap, int32_t *tok,
                                        int32_t *t_start, int32_t *t_end, float *t_conf, int32_t *topk_id, float *topk_lp, float *blank_lp,
                                        int32_t *bp, int64_t *guard_bad) {
    if (V < 2 || rows < 0 || width < 1 || width > PK_CTC_BEAM_MAX || cap < 1 || !tok || (rows > 0 && !logprobs) ||
        !offsets_ok(row_off, n_utt, rows) || (lm && !vocab))
        return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t R = std::max(rows, 1);
    const float *dlp = cx.upload(logprobs, (size_t)rows * V);
    const int32_t *doff = cx.upload(row_off, (size_t)n_utt + 1);
    int32_t *dtok = cx.guarded<int32_t>((size_t)n_utt * (1 + cap));
    int32_t *dst = cx.guarded<int32_t>((size_t)n_utt * cap), *den = cx.guarded<int32_t>((size_t)n_utt * cap);
    float *dcf = cx.guarded<float>((size_t)n_utt * cap);
    int32_t *did = cx.guarded<int32_t>(R * width), *dbp = cx.guarded<int32_t>(R * width);
    float *dtl = cx.guarded<float>(R * width), *dbl = cx.guarded<float>(R);
    if (!cx.ok) return PK_ERR_CUDA;
    DeviceLM dlm;
    DevicePieces dpc;
    const std::string msg = ctc_beam_tables(lm, vocab, V, [&cx](const void *h, size_t bytes) -> void * {
        return cx.upload(static_cast<const uint8_t *>(h), bytes);
    }, &dlm, &dpc);
    dlm.set_weights(alpha, beta);
    if (!msg.empty() || !cx.ok) return msg.empty() || msg.rfind("cudaMalloc", 0) == 0 ? PK_ERR_CUDA : PK_ERR_INVALID;
    launch_ctc_frame_topk(dlp, rows, V, width, did, dtl, dbl, cx.st);
    launch_ctc_beam(dlp, did, dtl, dbl, doff, n_utt, V, width, cap, dlm, dpc, dbp, dtok, dst, den, dcf, cx.st);
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    auto get_i = [](int32_t *h, const int32_t *d, size_t n) { return !h || cudaMemcpy(h, d, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess; };
    if (!get_i(tok, dtok, (size_t)n_utt * (1 + cap)) || !get_i(t_start, dst, (size_t)n_utt * cap) || !get_i(t_end, den, (size_t)n_utt * cap) ||
        !fetch_f32(t_conf, dcf, (size_t)n_utt * cap) || !get_i(topk_id, did, (size_t)rows * width) || !fetch_f32(topk_lp, dtl, (size_t)rows * width) ||
        !fetch_f32(blank_lp, dbl, rows) || !get_i(bp, dbp, (size_t)rows * width))
        return PK_ERR_CUDA;
    return PK_OK;
}

extern "C" pk_status pk_kernel_ctc_align(int device, int n_utt, const int32_t *row_off, int rows, int V, const float *logprobs,
                                         const int32_t *tgt, const int32_t *tgt_off, int cap, int32_t *tok, int32_t *t_start,
                                         int32_t *t_end, float *t_conf, double *score, double *loglik, int32_t *path,
                                         int64_t *guard_bad) {
    if (V < 2 || rows < 0 || cap < 1 || !tok || (rows > 0 && !logprobs) || !offsets_ok(row_off, n_utt, rows) || !tgt_off ||
        tgt_off[0] != 0)
        return PK_ERR_INVALID;
    for (int b = 0; b < n_utt; ++b) {
        if (tgt_off[b + 1] < tgt_off[b]) return PK_ERR_INVALID;
        if (tgt_off[b + 1] - tgt_off[b] > PK_ALIGN_MAX_TOKENS) return PK_ERR_CAPACITY;
    }
    const int n_tgt = tgt_off[n_utt];
    if (n_tgt > 0 && !tgt) return PK_ERR_INVALID;
    for (int i = 0; i < n_tgt; ++i)
        if (tgt[i] < 0 || tgt[i] > V - 2) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t R = std::max(rows, 1);
    const int stride = 2 * std::min(max_len(row_off, n_utt), PK_ALIGN_MAX_TOKENS) + 1;   // as the engine sizes it from Tmax
    const float *dlp = cx.upload(logprobs, (size_t)rows * V);
    const int32_t *doff = cx.upload(row_off, (size_t)n_utt + 1);
    const int32_t *dtg = cx.upload(tgt, (size_t)n_tgt), *dto = cx.upload(tgt_off, (size_t)n_utt + 1);
    uint8_t *dbp = static_cast<uint8_t *>(cx.alloc(R * stride));
    int32_t *dbest = static_cast<int32_t *>(cx.alloc(R * sizeof(int32_t)));
    float *dconf = static_cast<float *>(cx.alloc(R * sizeof(float)));
    int32_t *dtok = cx.guarded<int32_t>((size_t)n_utt * (1 + cap));
    int32_t *dst = cx.guarded<int32_t>((size_t)n_utt * cap), *den = cx.guarded<int32_t>((size_t)n_utt * cap);
    float *dcf = cx.guarded<float>((size_t)n_utt * cap);
    double *dsc = cx.guarded<double>(n_utt), *dll = cx.guarded<double>(n_utt);
    int32_t *dpath = cx.guarded<int32_t>(R);
    if (!cx.ok) return PK_ERR_CUDA;
    launch_ctc_align(dlp, doff, n_utt, V, dtg, dto, dbp, stride, dbest, dconf, dsc, dll, dpath, cx.st);
    launch_ctc_collapse(dbest, dconf, doff, n_utt, V - 1, cap, dtok, dst, den, dcf, cx.st);
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    auto get = [](void *h, const void *d, size_t bytes) { return !h || cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost) == cudaSuccess; };
    if (!get(tok, dtok, (size_t)n_utt * (1 + cap) * 4) || !get(t_start, dst, (size_t)n_utt * cap * 4) ||
        !get(t_end, den, (size_t)n_utt * cap * 4) || !get(t_conf, dcf, (size_t)n_utt * cap * 4) || !get(score, dsc, (size_t)n_utt * 8) ||
        !get(loglik, dll, (size_t)n_utt * 8) || !get(path, dpath, (size_t)rows * 4))
        return PK_ERR_CUDA;
    return PK_OK;
}

namespace {

int conv_len3(int n) { return (n - 1) / 2 + 1; }   // 3 taps, stride 2, padding 1

// the engine's mel tables, uploaded into the hook's buffers
MelTables hook_mel_tables(HookCtx &cx, int n_mels) {
    return build_mel_tables(n_mels, [&cx](const void *h, size_t bytes) -> void * {
        return cx.upload(static_cast<const uint8_t *>(h), bytes);
    });
}

bool mel_bins_ok(int n_mels) { return n_mels >= 8 && n_mels <= MEL_NORM_THREADS && n_mels % 8 == 0; }

}  // namespace

extern "C" {

// K1 (+ K2) as pk_engine::run_mel launches them.  Utterance b = pcm[pcm_off[b] .. pcm_off[b+1]) (samples before pcm_off[0]
// are uploaded too and must not be read); frame_off as the engine derives it (1 + n / 160 frames each).  normalize = 1:
// logmel_out = the intermediate log-mel, feats_out = the normalised features; normalize = 0 (Sortformer): logmel_out = the
// log-mel the kernel writes into the engine's feature buffer, feats_out = NULL.
pk_status pk_kernel_mel(int device, int n_utt, const int64_t *pcm_off, const float *pcm, int n_mels, int normalize, float *logmel_out,
                        float *feats_out, int64_t *guard_bad) {
    if (n_utt < 1 || !pcm_off || !pcm || pcm_off[0] < 0 || !mel_bins_ok(n_mels) || !logmel_out || (normalize != 0) != (feats_out != nullptr))
        return PK_ERR_INVALID;
    std::vector<int32_t> frame_off(n_utt + 1, 0);
    int maxF = 0;
    for (int b = 0; b < n_utt; ++b) {
        const int64_t n = pcm_off[b + 1] - pcm_off[b];
        if (n < (normalize ? 400 : 2) || n > ((int64_t)1 << 30)) return PK_ERR_INVALID;
        const int F = (int)(1 + n / 160);
        frame_off[b + 1] = frame_off[b] + F;
        maxF = std::max(maxF, F);
    }
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t n_o = (size_t)frame_off[n_utt] * n_mels;
    const MelTables tb = hook_mel_tables(cx, n_mels);
    int64_t *doff = cx.upload(pcm_off, n_utt + 1);
    int32_t *dfo = cx.upload(frame_off.data(), n_utt + 1);
    float *dpcm = cx.upload(pcm, (size_t)pcm_off[n_utt]);
    float *lm = cx.guarded<float>(n_o), *ft = normalize ? cx.guarded<float>(n_o) : nullptr;
    float *part = normalize ? static_cast<float *>(cx.alloc(mel_part_floats(n_utt, n_mels) * sizeof(float))) : nullptr;
    if (!cx.ok) return PK_ERR_CUDA;
    if (normalize) launch_mel(dpcm, doff, dfo, n_utt, maxF, n_mels, tb, lm, ft, part, cx.st, true);
    else launch_mel(dpcm, doff, dfo, n_utt, maxF, n_mels, tb, nullptr, lm, nullptr, cx.st, false);
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    return fetch_f32(logmel_out, lm, n_o) && (!ft || fetch_f32(feats_out, ft, n_o)) ? PK_OK : PK_ERR_CUDA;
}

// The streaming K1 as pk_stream_step launches it: stream b's pre-emphasised signal sig[sig_off[b] .. sig_off[b+1]) gives
// n_frames[b] frames (frame f reads samples f * 160 .. f * 160 + 511) into rows out_row[b] + f of logmel_out [rows_total][n_mels].
pk_status pk_kernel_mel_stream(int device, int n_streams, const int64_t *sig_off, const float *sig, const int32_t *n_frames,
                               const int32_t *out_row, int rows_total, int n_mels, float *logmel_out, int64_t *guard_bad) {
    if (n_streams < 1 || !sig_off || !sig || !n_frames || !out_row || rows_total < 1 || sig_off[0] < 0 || !mel_bins_ok(n_mels) || !logmel_out)
        return PK_ERR_INVALID;
    int maxF = 0;
    for (int b = 0; b < n_streams; ++b) {
        const int64_t n = sig_off[b + 1] - sig_off[b];
        if (n < 0 || n_frames[b] < 0 || out_row[b] < 0 || (int64_t)out_row[b] + n_frames[b] > rows_total) return PK_ERR_INVALID;
        if (n_frames[b] > 0 && (int64_t)(n_frames[b] - 1) * 160 + 512 > n) return PK_ERR_INVALID;
        maxF = std::max(maxF, n_frames[b]);
    }
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t n_o = (size_t)rows_total * n_mels;
    const MelTables tb = hook_mel_tables(cx, n_mels);
    int64_t *doff = cx.upload(sig_off, n_streams + 1);
    int32_t *dnf = cx.upload(n_frames, n_streams), *drow = cx.upload(out_row, n_streams);
    float *dsig = cx.upload(sig, (size_t)sig_off[n_streams]);
    float *lm = cx.guarded<float>(n_o);
    if (!cx.ok) return PK_ERR_CUDA;
    launch_mel_stream(dsig, doff, dnf, drow, n_streams, maxF, n_mels, tb, lm, cx.st);
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    return fetch_f32(logmel_out, lm, n_o) ? PK_OK : PK_ERR_CUDA;
}

// K3 (conv1 + ReLU + dw1) as pk_engine::run_conv1 launches it: utterance b = feature rows [frame_off[b], frame_off[b+1]) of
// feats [rows_total][mel] (other rows may exist and must not be read); weights [C][9] as stored.  Output rows
// (s2_off[b] + t2) * f2n + f2 of C channels, s2_off as the engine derives it, in sub1's form for `math`: out_f32, or hi and,
// with PK_MATH_BF16X3, lo.
pk_status pk_kernel_subsample_conv1(int device, int math, int n_utt, const int32_t *frame_off, int rows_total, const float *feats, int mel,
                                    int C, const float *w1, const float *b1, const float *wd, const float *bd, float *out_f32, float *hi,
                                    float *lo, int64_t *guard_bad) {
    if (!offsets_ok(frame_off, n_utt, rows_total) || mel < 2 || mel % 2 || mel > MEL_NORM_THREADS || C < 4 || C % 4 || C > 1024 || !feats ||
        !w1 || !b1 || !wd || !bd || !act_out_ok(math, out_f32, hi, lo))
        return PK_ERR_INVALID;
    std::vector<int32_t> s2_off(n_utt + 1, 0);
    int maxT2 = 0;
    for (int b = 0; b < n_utt; ++b) {
        const int F = frame_off[b + 1] - frame_off[b];
        if (F < 1) return PK_ERR_INVALID;
        const int t2 = conv_len3(conv_len3(F));
        s2_off[b + 1] = s2_off[b] + t2;
        maxT2 = std::max(maxT2, t2);
    }
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t n_o = (size_t)s2_off[n_utt] * conv_len3(conv_len3(mel)) * C;
    int32_t *dfo = cx.upload(frame_off, n_utt + 1), *ds2 = cx.upload(s2_off.data(), n_utt + 1);
    float *df = cx.upload(feats, (size_t)rows_total * mel);
    float *dw1 = cx.upload(w1, (size_t)C * 9), *db1 = cx.upload(b1, C), *dwd = cx.upload(wd, (size_t)C * 9), *dbd = cx.upload(bd, C);
    ActBuf out = guarded_act(cx, math, n_o, lo != nullptr);
    if (!cx.ok) return PK_ERR_CUDA;
    launch_subsample_conv1_dw1(df, dfo, ds2, n_utt, maxT2, mel, C, dw1, db1, dwd, dbd, out, cx.st);
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    return fetch_act(out, out_f32, hi, lo, n_o) ? PK_OK : PK_ERR_CUDA;
}

// K4 (depthwise 3x3, stride 2, padding 1 on channels-last rows) as pk_engine::run_subsample_tail launches it for dw2_:
// utterance b has in_rows[b] time rows of fin frequency rows of C channels, packed in order in `in`; its output has
// conv_len(in_rows[b]) x conv_len(fin) rows, packed in the same order.  wd tap-major [9][C] (as dw2_wt), bd [C].  Output in
// sub3's form for `math`.
pk_status pk_kernel_subsample_dw(int device, int math, int n_utt, const int32_t *in_rows, int fin, int C, const float *in, const float *wd_tapmajor,
                                 const float *bd, float *out_f32, float *hi, float *lo, int64_t *guard_bad) {
    if (n_utt < 1 || !in_rows || fin < 1 || C < 4 || C % 4 || !in || !wd_tapmajor || !bd || !act_out_ok(math, out_f32, hi, lo))
        return PK_ERR_INVALID;
    std::vector<int32_t> in_off(n_utt + 1, 0), out_off(n_utt + 1, 0);
    for (int b = 0; b < n_utt; ++b) {
        if (in_rows[b] < 1 || (int64_t)in_off[b] + in_rows[b] > INT32_MAX) return PK_ERR_INVALID;
        in_off[b + 1] = in_off[b] + in_rows[b];
        out_off[b + 1] = out_off[b] + conv_len3(in_rows[b]);
    }
    const int fout = conv_len3(fin);
    const int64_t out_rows = (int64_t)out_off[n_utt] * fout;
    if (out_rows > INT32_MAX) return PK_ERR_INVALID;
    HookCtx cx(device);
    if (!cx.ok) return PK_ERR_CUDA;
    const size_t n_o = (size_t)out_rows * C;
    int32_t *drows = cx.upload(in_rows, n_utt), *din = cx.upload(in_off.data(), n_utt + 1), *dout = cx.upload(out_off.data(), n_utt + 1);
    float *dx = cx.upload(in, (size_t)in_off[n_utt] * fin * C), *dw = cx.upload(wd_tapmajor, (size_t)9 * C), *db = cx.upload(bd, C);
    ActBuf out = guarded_act(cx, math, n_o, lo != nullptr);
    if (!cx.ok) return PK_ERR_CUDA;
    launch_subsample_dw(dx, drows, din, dout, n_utt, fin, C, dw, db, out, (int)out_rows, cx.st);
    pk_status rc = cx.finish(guard_bad);
    if (rc) return rc;
    return fetch_act(out, out_f32, hi, lo, n_o) ? PK_OK : PK_ERR_CUDA;
}

}  // extern "C"
