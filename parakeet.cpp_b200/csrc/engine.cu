// engine.cu -- the engine behind the C-ABI (include/parakeet_b200.h): weight loading and
// layout, workspace, and the orchestration of the sm_90a kernels for
//     PCM -> log-mel -> FastConformer encoder -> CTC / TDT greedy decode.
//
// Reference call stack being replaced (SURVEY.md section 3.2/3.3):
//   Transcriber::Transcriber / to_gpu        include/parakeet/transcribe.hpp:59-71
//   Transcriber::transcribe                  include/parakeet/transcribe.hpp:99-179
//   preprocess_audio                         src/audio.cpp:100-158
//   FastConformerEncoder::forward            src/encoder.cpp:253-271 (and :9-241)
//   CTCDecoder::forward + ctc_greedy_decode  src/ctc.cpp:12-127
//   tdt_greedy_decode(_with_timestamps)      src/tdt.cpp:36-201
//
// Data layout in HBM: utterances are PACKED, not padded: a batch is one row-major matrix
// whose rows are (utterance, time[, freq]) and per-utterance prefix offsets say where each
// utterance starts.  GEMMs run over all rows at once; length-aware kernels (convolutions,
// attention, decode) use the offsets, so every utterance sees exactly the zero padding /
// sequence end the batch-1 reference gives it.
#include "engine.h"

#include <algorithm>
#include <cstdlib>
#include <unordered_map>

namespace pk_detail {
std::string &create_err() {
    thread_local std::string s;
    return s;
}
}  // namespace pk_detail
#define g_create_err (create_err())

// ===================================================================== weights

pk_status pk_engine::get_vec(const SafeTensors &st, const std::string &name, int n, float **out) {
    std::vector<float> h;
    std::string e;
    if (!st.read_f32(name, h, n, e)) return fail(PK_ERR_MISSING, e);
    *out = upload(h);
    return *out ? PK_OK : fail(PK_ERR_CUDA, "cudaMalloc failed for " + name);
}

pk_status pk_engine::finish_weight(std::vector<float> &w, std::vector<float> *b, int N, int K, GemmWeight &out) {
    out.N = N;
    out.K = K;
    out.w = upload(w);
    if (!out.w) return fail(PK_ERR_CUDA, "cudaMalloc failed (weight)");
    if (b) {
        out.bias = upload(*b);
        if (!out.bias) return fail(PK_ERR_CUDA, "cudaMalloc failed (bias)");
    }
    if (cfg.math != PK_MATH_FP32) {
        std::vector<bf16> hi(w.size()), lo(w.size());
        for (size_t i = 0; i < w.size(); ++i) {
            hi[i] = __float2bfloat16_rn(w[i]);
            lo[i] = __float2bfloat16_rn(w[i] - __bfloat162float(hi[i]));
        }
        out.hi = upload(hi);
        out.lo = upload(lo);
        if (!out.hi || !out.lo) return fail(PK_ERR_CUDA, "cudaMalloc failed (split weight)");
        if (K % 64 != 0) return fail(PK_ERR_INVALID, "wgmma GEMM needs K % 64 == 0");
        if (!make_tc_operand(&out.tc, out.hi, out.lo, N, K, tc_tile_n(N)))
            return fail(PK_ERR_CUDA, "cuTensorMapEncodeTiled failed for a weight");
    }
    return PK_OK;
}

pk_status pk_engine::make_weight(const SafeTensors &st, const std::string &wname, const std::string &bname, int N,
                                 int K, GemmWeight &out, const std::vector<int> *row_perm,
                                 const std::vector<int> *col_perm, float scale) {
    std::vector<float> w, b;
    std::string e;
    if (!st.read_f32(wname, w, (int64_t)N * K, e)) return fail(PK_ERR_MISSING, e);
    if (!bname.empty() && !st.read_f32(bname, b, N, e)) return fail(PK_ERR_MISSING, e);
    if (row_perm || col_perm) {
        std::vector<float> w2(w.size()), b2(b.size());
        for (int n = 0; n < N; ++n) {
            const int sn = row_perm ? (*row_perm)[n] : n;
            for (int k = 0; k < K; ++k) {
                const int sk = col_perm ? (*col_perm)[k] : k;
                w2[(size_t)n * K + k] = w[(size_t)sn * K + sk];
            }
            if (!b.empty()) b2[n] = b[sn];
        }
        w.swap(w2);
        if (!b.empty()) b.swap(b2);
    }
    if (scale != 1.0f) {
        for (auto &v : w) v *= scale;
        for (auto &v : b) v *= scale;
    }
    return finish_weight(w, bname.empty() ? nullptr : &b, N, K, out);
}

pk_status pk_engine::load(const char *path) {
    SafeTensors st;
    std::string e;
    if (!st.open(path, e)) return fail(PK_ERR_IO, e);
    const pk_config &c = cfg;
    const int C = c.sub_channels, d = c.d_model, ff = c.ff, H = c.n_heads, hd = d / H;
    pk_status s;

    // ---- mel tables (mel.cu)
    mel_tb = build_mel_tables(c.mel_bins, [this](const void *h, size_t bytes) -> void * {
        std::vector<uint8_t> v(static_cast<const uint8_t *>(h), static_cast<const uint8_t *>(h) + bytes);
        return upload(v);
    });

    // ---- subsampling (encoder.cpp:208-241)
    const std::string sp = enc_prefix + "subsampling_.";
    if ((s = get_vec(st, sp + "conv1_.weight", C * 9, &c1_w))) return s;
    if ((s = get_vec(st, sp + "conv1_.bias", C, &c1_b))) return s;
    if ((s = get_vec(st, sp + "dw1_.weight", C * 9, &dw1_w))) return s;
    if ((s = get_vec(st, sp + "dw1_.bias", C, &dw1_b))) return s;
    if ((s = get_vec(st, sp + "dw2_.weight", C * 9, &dw2_w))) return s;
    {
        std::vector<float> w, wt((size_t)C * 9);
        if (!st.read_f32(sp + "dw2_.weight", w, (int64_t)C * 9, e)) return fail(PK_ERR_MISSING, e);
        for (int ch = 0; ch < C; ++ch)
            for (int k = 0; k < 9; ++k) wt[(size_t)k * C + ch] = w[(size_t)ch * 9 + k];
        dw2_wt = upload(wt);
    }
    if ((s = get_vec(st, sp + "dw2_.bias", C, &dw2_b))) return s;
    if ((s = make_weight(st, sp + "conv2_.weight", sp + "conv2_.bias", C, C, conv2))) return s;
    if ((s = make_weight(st, sp + "conv3_.weight", sp + "conv3_.bias", C, C, conv3))) return s;
    {
        // reference flattens (C, F') channel-major (encoder.cpp:236-238): k_ref = c*F' + f.
        // Our rows are (f, c): k = f*C + c.
        std::vector<int> colp((size_t)C * f3n);
        for (int f = 0; f < f3n; ++f)
            for (int ch = 0; ch < C; ++ch) colp[(size_t)f * C + ch] = ch * f3n + f;
        // xscaling (StreamingFastConformerEncoder::forward, streaming_encoder.cpp:403-407): the NEST encoder multiplies the
        // subsampling output by sqrt(d) before layer 0.  Folded into proj_ here, before the hi/lo split: (s W) x + s b
        // rounds differently from s (W x + b) by about one fp32 rounding.
        const float xscale = diar ? std::sqrt((float)d) : 1.0f;
        if ((s = make_weight(st, sp + "proj_.weight", sp + "proj_.bias", d, C * f3n, proj, nullptr, &colp, xscale))) return s;
    }

    // ---- relative position table input: emb(p) for p = -(pos_tmax-1) .. pos_tmax-1, fp32 math as
    // encoder.cpp:9-30 (row index here = p + pos_tmax - 1).  Row p is the same whatever the table's extent.
    const int NP = 2 * pos_tmax - 1;
    std::vector<float> emb((size_t)NP * d);
    for (int r = 0; r < NP; ++r) {
        const float position = (float)(r - (pos_tmax - 1));
        for (int i = 0; i < d; i += 2) {
            const float div_term = std::exp((float)i * (-std::log(10000.0f) / d));
            emb[(size_t)r * d + i] = std::sin(position * div_term);
            if (i + 1 < d) emb[(size_t)r * d + i + 1] = std::cos(position * div_term);
        }
    }
    float *d_emb = upload(emb);
    if (!d_emb) return fail(PK_ERR_CUDA, "cudaMalloc failed (pos emb)");

    layers.resize(c.n_layers);
    for (int i = 0; i < c.n_layers; ++i) {
        LayerW &L = layers[i];
        const std::string lp = enc_prefix + "layers_." + std::to_string(i) + ".";
        for (int f = 0; f < 2; ++f) {
            const std::string fp = lp + (f == 0 ? "ffn1_." : "ffn2_.");
            if ((s = get_vec(st, fp + "norm_.weight", d, &L.ffn_ln_w[f]))) return s;
            if ((s = get_vec(st, fp + "norm_.bias", d, &L.ffn_ln_b[f]))) return s;
            if ((s = make_weight(st, fp + "fc1_.weight", fp + "fc1_.bias", ff, d, L.fc1[f]))) return s;
            if ((s = make_weight(st, fp + "fc2_.weight", fp + "fc2_.bias", d, ff, L.fc2[f]))) return s;
        }
        const std::string ap = lp + "attn_.";
        if ((s = get_vec(st, ap + "norm_.weight", d, &L.att_ln_w))) return s;
        if ((s = get_vec(st, ap + "norm_.bias", d, &L.att_ln_b))) return s;
        {
            std::vector<float> w((size_t)3 * d * d), b((size_t)3 * d), t;
            const char *names[3] = {"q_proj", "k_proj", "v_proj"};
            for (int q = 0; q < 3; ++q) {
                if (!st.read_f32(ap + "mha_." + names[q] + ".weight", t, (int64_t)d * d, e)) return fail(PK_ERR_MISSING, e);
                memcpy(&w[(size_t)q * d * d], t.data(), t.size() * 4);
                if (!st.read_f32(ap + "mha_." + names[q] + ".bias", t, d, e)) return fail(PK_ERR_MISSING, e);
                memcpy(&b[(size_t)q * d], t.data(), t.size() * 4);
            }
            if ((s = finish_weight(w, &b, 3 * d, d, L.qkv))) return s;
        }
        if ((s = make_weight(st, ap + "mha_.out_proj.weight", ap + "mha_.out_proj.bias", d, d, L.out))) return s;
        if ((s = get_vec(st, ap + "pos_bias_u_", H * hd, &L.pos_u))) return s;
        if ((s = get_vec(st, ap + "pos_bias_v_", H * hd, &L.pos_v))) return s;
        {
            // PP = emb . Wpos^T (pos_proj_ has no bias, encoder.cpp:80), exact fp32 GEMM
            float *wpos;
            if ((s = get_vec(st, ap + "pos_proj_.weight", d * d, &wpos))) return s;
            L.pp = dalloc<float>((size_t)NP * d);
            if (!L.pp) return fail(PK_ERR_CUDA, "cudaMalloc failed (pp)");
            EpiParams ep;
            ep.kind = EPI_BIAS_F32;
            ep.out_f32 = L.pp;
            ep.ldo = d;
            launch_gemm_simt(d_emb, d, wpos, d, NP, d, d, ep, stream);
            ++launches;
            if (cfg.math != PK_MATH_FP32 && (hd == 64 || hd == 128)) {
                L.pp_hi = dalloc<bf16>((size_t)NP * d);
                L.pp_lo = dalloc<bf16>((size_t)NP * d);
                if (!L.pp_hi || !L.pp_lo) return fail(PK_ERR_CUDA, "cudaMalloc failed (pp planes)");
                ActBuf sp;
                sp.hi = L.pp_hi;
                sp.lo = L.pp_lo;
                launch_split(L.pp, (size_t)NP * d, sp, stream);
                ++launches;
            }
        }
        const std::string cp = lp + "conv_.";
        if ((s = get_vec(st, cp + "norm_.weight", d, &L.conv_ln_w))) return s;
        if ((s = get_vec(st, cp + "norm_.bias", d, &L.conv_ln_b))) return s;
        {
            // GLU pairs channel j with j+d (operations.cpp:1450-1476): interleave the rows so
            // the pair sits in adjacent GEMM columns.
            std::vector<int> rowp((size_t)2 * d);
            for (int j = 0; j < d; ++j) {
                rowp[2 * j] = j;
                rowp[2 * j + 1] = d + j;
            }
            if ((s = make_weight(st, cp + "pointwise_conv1_.weight", cp + "pointwise_conv1_.bias", 2 * d, d, L.pw1, &rowp))) return s;
        }
        if ((s = make_weight(st, cp + "pointwise_conv2_.weight", cp + "pointwise_conv2_.bias", d, d, L.pw2))) return s;
        {
            // fold BatchNorm1d(eval) (normalization.cpp:48-104, eps 1e-5) into the depthwise conv
            const int ks = c.conv_kernel;
            std::vector<float> w, b, g, be, mu, var;
            if (!st.read_f32(cp + "depthwise_conv_.weight", w, (int64_t)d * ks, e)) return fail(PK_ERR_MISSING, e);
            if (!st.read_f32(cp + "depthwise_conv_.bias", b, d, e)) return fail(PK_ERR_MISSING, e);
            if (!st.read_f32(cp + "batch_norm_.weight", g, d, e)) return fail(PK_ERR_MISSING, e);
            if (!st.read_f32(cp + "batch_norm_.bias", be, d, e)) return fail(PK_ERR_MISSING, e);
            if (!st.read_f32(cp + "batch_norm_.running_mean", mu, d, e)) return fail(PK_ERR_MISSING, e);
            if (!st.read_f32(cp + "batch_norm_.running_var", var, d, e)) return fail(PK_ERR_MISSING, e);
            for (int ch = 0; ch < d; ++ch) {
                const double sc = (double)g[ch] / std::sqrt((double)var[ch] + 1e-5);
                for (int j = 0; j < ks; ++j) w[(size_t)ch * ks + j] = (float)((double)w[(size_t)ch * ks + j] * sc);
                b[ch] = (float)(((double)b[ch] - (double)mu[ch]) * sc + (double)be[ch]);
            }
            L.dw_w = upload(w);
            std::vector<float> wt((size_t)d * ks);
            for (int ch = 0; ch < d; ++ch)
                for (int j = 0; j < ks; ++j) wt[(size_t)j * d + ch] = w[(size_t)ch * ks + j];
            L.dw_wt = upload(wt);
            L.dw_b = upload(b);
        }
        if ((s = get_vec(st, lp + "final_norm_.weight", d, &L.fin_ln_w))) return s;
        if ((s = get_vec(st, lp + "final_norm_.bias", d, &L.fin_ln_b))) return s;
    }

    if (diar) {   // Sortformer (sortformer.cpp:42-48): projection_, transformer_, first_hidden_, output_proj_ (hidden_to_spks_ unused)
        const int Dt = sf.t_hidden, S = sf.max_speakers;
        if ((s = make_weight(st, "projection_.weight", "projection_.bias", Dt, d, t_proj))) return s;
        tlayers.resize(sf.t_layers);
        for (int i = 0; i < sf.t_layers; ++i) {
            TLayerW &L = tlayers[i];
            const std::string lp = "transformer_.layers_." + std::to_string(i) + ".";
            std::vector<float> w((size_t)3 * Dt * Dt), b((size_t)3 * Dt), t;
            const char *names[3] = {"q_proj", "k_proj", "v_proj"};
            for (int q = 0; q < 3; ++q) {
                if (!st.read_f32(lp + "mha_." + names[q] + ".weight", t, (int64_t)Dt * Dt, e)) return fail(PK_ERR_MISSING, e);
                memcpy(&w[(size_t)q * Dt * Dt], t.data(), t.size() * 4);
                if (!st.read_f32(lp + "mha_." + names[q] + ".bias", t, Dt, e)) return fail(PK_ERR_MISSING, e);
                memcpy(&b[(size_t)q * Dt], t.data(), t.size() * 4);
            }
            if ((s = finish_weight(w, &b, 3 * Dt, Dt, L.qkv))) return s;
            if ((s = make_weight(st, lp + "mha_.out_proj.weight", lp + "mha_.out_proj.bias", Dt, Dt, L.out))) return s;
            if ((s = make_weight(st, lp + "fc1_.weight", lp + "fc1_.bias", sf.t_ff, Dt, L.fc1))) return s;
            if ((s = make_weight(st, lp + "fc2_.weight", lp + "fc2_.bias", Dt, sf.t_ff, L.fc2))) return s;
            if ((s = get_vec(st, lp + "norm1_.weight", Dt, &L.n1_w))) return s;
            if ((s = get_vec(st, lp + "norm1_.bias", Dt, &L.n1_b))) return s;
            if ((s = get_vec(st, lp + "norm2_.weight", Dt, &L.n2_w))) return s;
            if ((s = get_vec(st, lp + "norm2_.bias", Dt, &L.n2_b))) return s;
        }
        {
            std::vector<float> w1, w1t((size_t)Dt * Dt);
            if (!st.read_f32("first_hidden_.weight", w1, (int64_t)Dt * Dt, e)) return fail(PK_ERR_MISSING, e);
            for (int n = 0; n < Dt; ++n)
                for (int k = 0; k < Dt; ++k) w1t[(size_t)k * Dt + n] = w1[(size_t)n * Dt + k];
            head_w1t = upload(w1t);
            if (!head_w1t) return fail(PK_ERR_CUDA, "cudaMalloc failed (speaker head)");
        }
        if ((s = get_vec(st, "first_hidden_.bias", Dt, &head_b1))) return s;
        if ((s = get_vec(st, "output_proj_.weight", S * Dt, &head_w2))) return s;
        if ((s = get_vec(st, "output_proj_.bias", S, &head_b2))) return s;
        PK_CUDA(cudaStreamSynchronize(stream));
        PK_CUDA(cudaGetLastError());
        return PK_OK;
    }

    // ---- heads
    const int V = c.vocab, P = c.pred_hidden, J = c.joint_hidden, D = c.n_durations;
    if (c.has_ctc) {
        if ((s = make_weight(st, "ctc_decoder_.proj_.weight", "ctc_decoder_.proj_.bias", V, d, ctc_head))) return s;
    }
    const std::string jp = c.joint_prefix_tdt ? "tdt_joint_." : "joint_.";
    if ((s = make_weight(st, jp + "enc_proj_.weight", jp + "enc_proj_.bias", J, d, enc_proj))) return s;
    if ((s = get_vec(st, jp + "pred_proj_.weight", J * P, &Wp))) return s;
    if (D == 0) {   // RNNTJoint (rnnt.cpp:30-44): one output head out_proj_ over the V labels
        if ((s = get_vec(st, jp + "out_proj_.weight", V * J, &Wout))) return s;
        if ((s = get_vec(st, jp + "out_proj_.bias", V, &bout))) return s;
    } else {
        std::vector<float> w((size_t)(V + D) * J), b((size_t)V + D), t;
        if (!st.read_f32(jp + "label_proj_.weight", t, (int64_t)V * J, e)) return fail(PK_ERR_MISSING, e);
        memcpy(w.data(), t.data(), t.size() * 4);
        if (!st.read_f32(jp + "duration_proj_.weight", t, (int64_t)D * J, e)) return fail(PK_ERR_MISSING, e);
        memcpy(&w[(size_t)V * J], t.data(), t.size() * 4);
        if (!st.read_f32(jp + "label_proj_.bias", t, V, e)) return fail(PK_ERR_MISSING, e);
        memcpy(b.data(), t.data(), t.size() * 4);
        if (!st.read_f32(jp + "duration_proj_.bias", t, D, e)) return fail(PK_ERR_MISSING, e);
        memcpy(&b[V], t.data(), t.size() * 4);
        Wout = upload(w);
        bout = upload(b);
    }
    {
        float *embed, *wih0, *b0;
        if ((s = get_vec(st, "prediction_.embed_.weight", V * P, &embed))) return s;
        for (int l = 0; l < c.lstm_layers; ++l) {
            const std::string q = "prediction_.lstm_.cells_." + std::to_string(l) + ".";
            if ((s = get_vec(st, q + "hidden_proj_.weight", 4 * P * P, &Whh[l]))) return s;
            if ((s = get_vec(st, q + "input_proj_.weight", 4 * P * P, &Wih[l]))) return s;
            // unit-major copies for the decode kernel (row = unit*4 + gate; gate order i,f,g,o of lstm.cpp:20-24)
            {
                std::vector<float> src, dst((size_t)4 * P * P);
                for (int which = 0; which < 2; ++which) {
                    if (!st.read_f32(q + (which ? "input_proj_.weight" : "hidden_proj_.weight"), src, (int64_t)4 * P * P, e)) return fail(PK_ERR_MISSING, e);
                    lstm_unit_major(src.data(), P, dst.data());
                    float *d = upload(dst);
                    if (!d) return fail(PK_ERR_CUDA, "cudaMalloc failed (LSTM weights)");
                    (which ? Wih_um[l] : Whh_um[l]) = d;
                }
            }
            if ((s = get_vec(st, q + "input_proj_.bias", 4 * P, &bih[l]))) return s;
        }
        wih0 = Wih[0];
        b0 = bih[0];
        // G0[token] = W_ih0 . E[token] + b0 (lstm.cpp:17 first term, rnnt.cpp:24)
        G0 = dalloc<float>((size_t)V * 4 * P);
        if (!G0) return fail(PK_ERR_CUDA, "cudaMalloc failed (G0)");
        EpiParams ep;
        ep.kind = EPI_BIAS_F32;
        ep.bias = b0;
        ep.out_f32 = G0;
        ep.ldo = 4 * P;
        launch_gemm_simt(embed, P, wih0, P, V, 4 * P, P, ep, stream);
        ++launches;
    }
    {   // decode-kernel weights, split once into bf16 hi/lo rows
        auto split = [&](const float *src, int rows, int K, bf16 **out) {
            *out = dalloc<bf16>((size_t)rows * 2 * (K + 4));
            if (*out) launch_tdt_split_rows(src, rows, K, *out, stream);
            ++launches;
            return *out != nullptr;
        };
        bool ok = split(Wp, J, P, &Wp_s) && split(Wout, V + D, J, &Wout_s);
        for (int l = 0; l < c.lstm_layers && ok; ++l)
            ok = split(Whh_um[l], 4 * P, P, &Whh_s[l]) && split(Wih_um[l], 4 * P, P, &Wih_s[l]);
        if (!ok) return fail(PK_ERR_CUDA, "cudaMalloc failed (TDT split weights)");
    }
    PK_CUDA(cudaStreamSynchronize(stream));
    PK_CUDA(cudaGetLastError());
    return PK_OK;
}

// ===================================================================== workspace

pk_status pk_engine::alloc_workspace() {
    const pk_config &c = cfg;
    const int C = c.sub_channels, d = c.d_model;
    const size_t B = Bmax;
    const int t1 = conv_len(Fmax), t2 = conv_len(t1);
    const size_t rows2 = B * t2 * f2n, rows3 = B * (size_t)Tmax * f3n, Mx = B * (size_t)Tmax;
    d_pcm = dalloc<float>(B * (size_t)c.max_samples + 8);
    d_pcm_alt = dalloc<float>(B * (size_t)c.max_samples + 8);
    d_pcm_off = dalloc<int64_t>(B + 1);
    d_frame_off = dalloc<int32_t>(B + 1);
    d_s2_off = dalloc<int32_t>(B + 1);
    d_row_off = dalloc<int32_t>(B + 1);
    d_t2_rows = dalloc<int32_t>(B + 1);
    logmel = dalloc<float>(B * (size_t)Fmax * c.mel_bins);
    mel_part = dalloc<float>(mel_part_floats((int)B, c.mel_bins));
    feats = dalloc<float>(B * (size_t)Fmax * c.mel_bins);
    sub1 = act_alloc(rows2, C);
    sub2 = dalloc<float>(rows2 * C);
    sub3 = act_alloc(rows3, C);
    sub4 = act_alloc(rows3, C);
    if (cfg.math != PK_MATH_FP32 && sub4.hi && (!make_tc_operand(&sub4.tc, sub4.hi, sub4.lo, Mx, (size_t)C * f3n, 128) || !make_tc_operand(&sub4.tc32, sub4.hi, sub4.lo, Mx, (size_t)C * f3n, 32))) sub4.hi = nullptr;   // viewed as [M][C*F'] by proj_
    x = dalloc<float>(Mx * d);
    ln = act_alloc(Mx, d);
    ffh = act_alloc(Mx, c.ff);
    qkv = dalloc<float>(Mx * 3 * d);
    if (cfg.math != PK_MATH_FP32 && (c.d_model / c.n_heads == 64 || c.d_model / c.n_heads == 128)) {
        qkvp_hi = dalloc<bf16>(Mx * 2 * d);
        qkvp_lo = dalloc<bf16>(Mx * 2 * d);
        if (!qkvp_hi || !qkvp_lo) return fail(PK_ERR_CUDA, "cudaMalloc failed (qkv planes)");
    }
    ctx = act_alloc(Mx, d);
    glu = dalloc<float>(Mx * d);
    cv = act_alloc(Mx, d);
    const int ldv = (c.vocab + 3) & ~3;
    logits = dalloc<float>(Mx * ldv);
    EP = dalloc<float>(Mx * c.joint_hidden);
    best = dalloc<int32_t>(Mx);
    bconf = dalloc<float>(Mx);
    tok = dalloc<int32_t>(B * (1 + (size_t)cap));
    t_start = dalloc<int32_t>(B * (size_t)cap);
    t_end = dalloc<int32_t>(B * (size_t)cap);
    t_conf = dalloc<float>(B * (size_t)cap);
    Bpad = ((Bmax + 31) / 32) * 32;
    const size_t HS = (size_t)c.pred_hidden * Bpad;
    hbuf = dalloc<float>(HS * 2 * c.lstm_layers);                  // bf16 hi + lo planes
    zbuf = dalloc<float>((size_t)c.joint_hidden * Bpad);           // bf16 hi + lo planes
    tdt_ints = dalloc<int32_t>((size_t)Bpad + 512);               // overflow flags | grid-barrier counters (8 lines)
    tdt_keys = dalloc<unsigned long long>((size_t)6 * Bpad + 8);
    const size_t PG = (size_t)3 * num_sms * Bpad;
    pl_max = dalloc<float>(PG);
    pl_sum = dalloc<float>(PG);
    skinny_ws_floats = (size_t)2 << 20;                                       // 8 MB: >= (2 SMs' worth of CTAs) x 128 x 32 fp32 tiles
    skinny_ws = dalloc<float>(skinny_ws_floats);
    skinny_tickets = dalloc<unsigned int>(SKINNY_TICKETS);
    if (skinny_tickets) cudaMemsetAsync(skinny_tickets, 0, SKINNY_TICKETS * sizeof(unsigned int), stream);
    if (!pl_sum || !tdt_keys || !hbuf || !x || !sub2 || !d_pcm || !t_conf || !skinny_ws || !skinny_tickets || !mel_part) return fail(PK_ERR_CUDA, "cudaMalloc failed (workspace)");
    if (cfg.math != PK_MATH_FP32 && (!sub1.hi || !sub3.hi || !sub4.hi || !ln.hi || !ffh.hi || !ctx.hi || !cv.hi))
        return fail(PK_ERR_CUDA, "workspace: cudaMalloc or cuTensorMapEncodeTiled failed for an activation operand");
    if (diar) {
        const int Dt = sf.t_hidden;
        t_x = dalloc<float>(Mx * Dt);
        t_qkv = dalloc<float>(Mx * 3 * Dt);
        if (cfg.math != PK_MATH_FP32) {
            t_kv_hi = dalloc<bf16>(Mx * 2 * Dt);
            if (cfg.math == PK_MATH_BF16X3) t_kv_lo = dalloc<bf16>(Mx * 2 * Dt);
            if (!t_kv_hi || (cfg.math == PK_MATH_BF16X3 && !t_kv_lo)) return fail(PK_ERR_CUDA, "cudaMalloc failed (k | v planes)");
        }
        probs = dalloc<float>(Mx * sf.max_speakers);
        t_ln = act_alloc(Mx, Dt);
        t_ctx = act_alloc(Mx, Dt);
        t_ff = act_alloc(Mx, sf.t_ff);
        if (!t_x || !t_qkv || !probs || (cfg.math == PK_MATH_FP32 ? (!t_ln.f32 || !t_ctx.f32 || !t_ff.f32) : (!t_ln.hi || !t_ctx.hi || !t_ff.hi)))
            return fail(PK_ERR_CUDA, "cudaMalloc or cuTensorMapEncodeTiled failed (transformer workspace)");
        PK_CUDA(cudaMallocHost(&h_probs, Mx * sf.max_speakers * sizeof(float)));
    }
    PK_CUDA(cudaMallocHost(&h_pcm, (B * (size_t)c.max_samples + 8) * sizeof(float)));
    PK_CUDA(cudaMallocHost(&h_meta, (size_t)(8 * (B + 1)) * sizeof(int32_t)));
    PK_CUDA(cudaMallocHost(&h_tok, B * (1 + (size_t)cap) * sizeof(int32_t)));
    PK_CUDA(cudaMallocHost(&h_ts, B * (size_t)cap * sizeof(int32_t)));
    PK_CUDA(cudaMallocHost(&h_te, B * (size_t)cap * sizeof(int32_t)));
    PK_CUDA(cudaMallocHost(&h_tc, B * (size_t)cap * sizeof(float)));
    return PK_OK;
}

// Derive every per-utterance extent from either sample offsets or mel frame counts.
pk_status pk_engine::set_batch_shapes(const int32_t *n_frames, const int64_t *offsets, int n) {
    if (n <= 0) return fail(PK_ERR_INVALID, "empty batch");
    if (n > Bmax) return fail(PK_ERR_CAPACITY, "batch of " + std::to_string(n) + " exceeds max_batch " + std::to_string(Bmax));
    n_utt = n;
    probs_valid = false;
    pcm_off.assign(n + 1, 0);
    frame_off.assign(n + 1, 0);
    s2_off.assign(n + 1, 0);
    row_off.assign(n + 1, 0);
    t2_rows.assign(n + 1, 0);
    maxF = maxT2 = maxT = 0;
    for (int i = 0; i < n; ++i) {
        int F;
        if (offsets) {
            const int64_t ns = offsets[i + 1] - offsets[i];
            if (ns < 400) return fail(PK_ERR_INVALID, "utterance shorter than one 400-sample window");
            if (ns > cfg.max_samples) return fail(PK_ERR_CAPACITY, "utterance exceeds max_samples");
            pcm_off[i + 1] = pcm_off[i] + ns;
            F = (int)(1 + ns / 160);
        } else {
            F = n_frames[i];
            if (F < 2) return fail(PK_ERR_INVALID, "utterance needs at least 2 mel frames");
            if (F > Fmax) return fail(PK_ERR_CAPACITY, "utterance exceeds max frames");
        }
        const int t2 = conv_len(conv_len(F)), T = enc_frames(F);
        frame_off[i + 1] = frame_off[i] + F;
        s2_off[i + 1] = s2_off[i] + t2;
        row_off[i + 1] = row_off[i] + T;
        t2_rows[i] = t2;
        maxF = std::max(maxF, F);
        maxT2 = std::max(maxT2, t2);
        maxT = std::max(maxT, T);
    }
    M = row_off[n];
    M2 = s2_off[n] * f2n;
    return band_rows_ok();
}

// A band engine's batch holds at most the encoder rows of 3 h of audio in all (DESIGN.md section 16: the row x width products
// the offline kernels form in int are audited up to there).  Full-attention engines are bounded by their capacity instead.
pk_status pk_engine::band_rows_ok() {
    static const int kMaxRows = enc_frames(1 + PK_LOCAL_ATT_MAX_SAMPLES / 160);
    if ((cfg.local_att_left || cfg.local_att_right) && M > kMaxRows)
        return fail(PK_ERR_CAPACITY, "limited-context attention: a batch of " + std::to_string(M) + " encoder frames; at most " +
                                         std::to_string(kMaxRows) + " (3 h of audio) per batch");
    return PK_OK;
}

pk_status pk_engine::upload_shapes() {
    const int n = n_utt;
    int32_t *m = h_meta;
    PK_CUDA(cudaEventSynchronize(ev_h2d));  // pinned staging of the previous batch fully consumed
    memcpy(m, frame_off.data(), (n + 1) * 4);
    memcpy(m + (n + 1), s2_off.data(), (n + 1) * 4);
    memcpy(m + 2 * (n + 1), row_off.data(), (n + 1) * 4);
    memcpy(m + 3 * (n + 1), t2_rows.data(), (n + 1) * 4);
    memcpy(m + 4 * (n + 1), pcm_off.data(), (n + 1) * 8);
    PK_CUDA(cudaMemcpyAsync(d_frame_off, m, (n + 1) * 4, cudaMemcpyHostToDevice, stream));
    PK_CUDA(cudaMemcpyAsync(d_s2_off, m + (n + 1), (n + 1) * 4, cudaMemcpyHostToDevice, stream));
    PK_CUDA(cudaMemcpyAsync(d_row_off, m + 2 * (n + 1), (n + 1) * 4, cudaMemcpyHostToDevice, stream));
    PK_CUDA(cudaMemcpyAsync(d_t2_rows, m + 3 * (n + 1), (n + 1) * 4, cudaMemcpyHostToDevice, stream));
    PK_CUDA(cudaMemcpyAsync(d_pcm_off, m + 4 * (n + 1), (n + 1) * 8, cudaMemcpyHostToDevice, stream));
    PK_CUDA(cudaEventRecord(ev_h2d, stream));
    return PK_OK;
}

// ===================================================================== pipeline

void pk_engine::gemm(const Act &A, int lda, const GemmWeight &W, int M_, EpiParams epi) {
    epi.bias = W.bias;
    Scope sc(this, CAT_GEMM, 2.0 * M_ * W.N * W.K);
    if (cfg.math == PK_MATH_FP32) {
        launch_gemm_simt(A.f32, lda, W.w, W.K, M_, W.N, W.K, epi, stream);
    } else if (skinny && M_ <= 128 && skinny_ws && W.N <= 32 * SKINNY_TICKETS) {
        // one row tile: weight-streaming bound -- split over N and K so that every SM pulls weights (gemm_skinny.cu)
        cudaError_t ce = launch_gemm_skinny(A.hi, A.lo, lda, W.hi, W.lo, M_, W.N, W.K, cfg.math == PK_MATH_BF16X3, epi, skinny_ws, skinny_ws_floats,
                                            skinny_tickets, SKINNY_TICKETS, num_sms, stream);
        if (ce != cudaSuccess && gemm_err == PK_OK) gemm_err = fail(PK_ERR_CUDA, std::string("skinny GEMM launch: ") + cudaGetErrorString(ce));
    } else {
        const int cl = (gemm_cluster == 2 || gemm_cluster == 4) && lda == W.K ? gemm_cluster : 1;
        cudaError_t ce = launch_gemm_tc(A.tc, W.tc, M_, W.N, W.K, cfg.math == PK_MATH_BF16X3, epi, stream, cl, cl == 4 ? &A.tc32 : &A.tc64);
        if (ce != cudaSuccess && gemm_err == PK_OK) gemm_err = fail(PK_ERR_CUDA, std::string("wgmma GEMM launch: ") + cudaGetErrorString(ce));
    }
    ++launches;
}

// Front end of utterances [u0, u1): the offset arrays hold absolute positions in the packed
// buffers, so a sub-range is just a shifted view of them.
pk_status pk_engine::run_mel(int u0, int u1) {
    if (u1 < 0) u1 = n_utt;
    if (u1 <= u0) return PK_OK;
    Scope sc(this, CAT_MEL);
    launch_mel(pcm_src ? pcm_src : d_pcm, d_pcm_off + u0, d_frame_off + u0, u1 - u0, maxF, cfg.mel_bins, mel_tb, logmel, feats,
               mel_part + mel_part_floats(u0, cfg.mel_bins), stream, !diar);
    launches += diar ? 1 : 3;
    PK_CUDA(cudaGetLastError());
    return PK_OK;
}

// conv1_ + ReLU + dw1_ of ConvSubsampling (encoder.cpp:219-241), first kernel of the encoder
pk_status pk_engine::run_conv1(int u0, int u1) {
    if (u1 < 0) u1 = n_utt;
    if (u1 <= u0) return PK_OK;
    const pk_config &c = cfg;
    Scope sc(this, CAT_SUBSAMPLE);
    launch_subsample_conv1_dw1(feats, d_frame_off + u0, d_s2_off + u0, u1 - u0, maxT2, c.mel_bins, c.sub_channels, c1_w, c1_b,
                               dw1_w, dw1_b, sub1, stream);
    ++launches;
    PK_CUDA(cudaGetLastError());
    return PK_OK;
}

void pk_engine::layernorm(const float *in, int width, const float *w1, const float *b1, float *out1, ActBuf act1, const float *w2,
                          const float *b2, ActBuf act2) {
    Scope sc(this, CAT_LAYERNORM);
    launch_layernorm(in, M, width, w1, b1, out1, act1, w2, b2, act2, stream);
    ++launches;
}

// conv2_ .. proj_ of ConvSubsampling (encoder.cpp:219-241) on the staged batch into x; conv1_/dw1_ already ran (run_conv1)
pk_status pk_engine::run_subsample_tail() {
    const pk_config &c = cfg;
    const int C = c.sub_channels, d = c.d_model;
    {
        EpiParams ep;
        ep.kind = EPI_BIAS_RELU_F32;
        ep.out_f32 = sub2;
        ep.ldo = C;
        gemm(sub1, C, conv2, M2, ep);
    }
    {
        Scope sc(this, CAT_SUBSAMPLE);
        launch_subsample_dw(sub2, d_t2_rows, d_s2_off, d_row_off, n_utt, f2n, C, dw2_wt, dw2_b, sub3, M * f3n, stream);
    }
    ++launches;
    {
        EpiParams ep;
        ep.kind = EPI_BIAS_RELU_ACT;
        ep.act = sub4;
        ep.ldo = C;
        gemm(sub3, C, conv3, M * f3n, ep);
    }
    {
        EpiParams ep;
        ep.kind = EPI_BIAS_F32;
        ep.out_f32 = x;
        ep.ldo = d;
        gemm(sub4, C * f3n, proj, M, ep);
    }
    PK_CUDA(cudaGetLastError());
    return PK_OK;
}

pk_status pk_engine::run_encoder(float *sub_out_host, float *layers_out_host) {
    if (pk_status s = run_subsample_tail()) return s;
    if (sub_out_host) {
        PK_CUDA(cudaMemcpyAsync(sub_out_host, x, (size_t)M * cfg.d_model * 4, cudaMemcpyDeviceToHost, stream));
        PK_CUDA(cudaStreamSynchronize(stream));
    }
    return run_blocks(false, layers_out_host);
}

// Conformer blocks (encoder.cpp:196-204; streaming_encoder.cpp:430-472).  Every residual GEMM is followed by the LayerNorm
// that consumes its result: ffn1 -> attention norm, attention out -> conv norm, conv pw2 -> ffn2 norm, ffn2 -> final_norm_
// chained with the next block's ffn1_.norm_.  Only the attention and the depthwise conv differ between the offline and the
// cached (streaming) forms.
pk_status pk_engine::run_blocks(bool cached, float *layers_out_host) {
    const pk_config &c = cfg;
    const int d = c.d_model, H = c.n_heads, hd = d / H;
    // a streaming step: the active streams, their K / V ring lengths and starts (d_meta) and the rows of the longest chunk
    const int32_t *s_act = nullptr, *s_cl = nullptr, *s_rs = nullptr;
    int n_act = 0, maxC = 0;
    if (cached) {
        s_act = ss->meta_d(StreamSet::ACT); s_cl = ss->meta_d(StreamSet::CACHE_LEN); s_rs = ss->meta_d(StreamSet::RING_START);
        n_act = (int)ss->act.size();
        for (int n : ss->nC) maxC = std::max(maxC, n);
    }
    // PK_DEBUG_SUBBLOCKS=n (bisecting aid, offline encoder): stop after n residual sub-blocks; x is returned as is.
    int dbg_stop = -1, dbg_cnt = 0;
    if (const char *ev = cached ? nullptr : getenv("PK_DEBUG_SUBBLOCKS")) dbg_stop = atoi(ev);
    auto resid = [&](float alpha) {           // x += alpha * (A . W^T + b)
        EpiParams e;
        e.kind = EPI_RESID_F32;
        e.out_f32 = x;
        e.resid = x;
        e.ldo = d;
        e.alpha = alpha;
        return e;
    };
    ActBuf none;
    layernorm(x, d, layers[0].ffn_ln_w[0], layers[0].ffn_ln_b[0], nullptr, ln);
    for (int i = 0; i < c.n_layers; ++i) {
        const LayerW &L = layers[i];
        for (int f = 0; f < 2; ++f) {
            // FeedForward (encoder.cpp:39-46): x += 0.5 * fc2(silu(fc1(LN(x))))
            EpiParams e1;
            e1.kind = EPI_BIAS_SILU_ACT;
            e1.act = ffh;
            e1.ldo = c.ff;
            gemm(ln, d, L.fc1[f], M, e1);
            gemm(ffh, c.ff, L.fc2[f], M, resid(0.5f));
            if (f == 0) {
                layernorm(x, d, L.att_ln_w, L.att_ln_b, nullptr, ln);
            } else if (i + 1 < c.n_layers) {
                // final_norm_ of this block chained with the next block's ffn1_.norm_
                layernorm(x, d, L.fin_ln_w, L.fin_ln_b, x, none, layers[i + 1].ffn_ln_w[0], layers[i + 1].ffn_ln_b[0], ln);
            } else {
                // after the last block the normalised output is also written in GEMM-operand form for the heads
                layernorm(x, d, L.fin_ln_w, L.fin_ln_b, x, cfg.math == PK_MATH_FP32 ? none : (ActBuf)ln);
            }
            if (++dbg_cnt == dbg_stop) return PK_OK;
            if (f == 1) break;
            // ConformerAttention (encoder.cpp:111-186); cached: over each stream's K / V ring (streaming_encoder.cpp:160-272)
            const bool tc_attn = !cached && L.pp_hi && qkvp_hi && attn_tc;
            EpiParams eq;
            if (tc_attn) {   // k | v land as bf16 hi/lo planes [M, 2 d], q as fp32 [M, d] (the attention kernel adds pos_bias_u / _v)
                eq.kind = EPI_QKV_ACT;
                eq.act.hi = qkvp_hi;
                eq.act.lo = qkvp_lo;
                eq.ldo = 2 * d;
                eq.out_f32 = qkv;
                eq.qcols = d;
            } else {
                eq.kind = EPI_BIAS_F32;
                eq.out_f32 = qkv;
                eq.ldo = 3 * d;
            }
            gemm(ln, d, L.qkv, M, eq);
            {
                Scope sc(this, CAT_ATTENTION);
                const size_t ring = cached ? (size_t)i * ss->S * ss->L * d : 0;   // layer i's K / V rings
                const bool ok = cached
                    ? launch_stream_attention(qkv, 3 * d, d_row_off, s_act, n_act, maxC, s_cl, s_rs, ss->kc + ring, ss->vc + ring, ss->L, H, hd, d,
                                              L.pp, pos_tmax, L.pos_u, L.pos_v, ctx, stream)
                    : tc_attn
                    ? launch_relpos_attention_tc(qkv, L.pos_u, L.pos_v, qkvp_hi, qkvp_lo, 2 * d, d_row_off, n_utt, maxT, H, hd, L.pp_hi, L.pp_lo, pos_tmax,
                                                 c.local_att_left, c.local_att_right, d, ctx, stream)
                    : launch_relpos_attention(qkv, 3 * d, d_row_off, n_utt, maxT, H, hd, L.pp, pos_tmax, c.local_att_left, c.local_att_right, L.pos_u,
                                              L.pos_v, d, ctx, stream);
                if (!ok)
                    return fail(PK_ERR_INVALID, cached ? "stream attention: chunk too long for one block's shared memory" : "unsupported head_dim " + std::to_string(hd));
            }
            ++launches;
            gemm(ctx, d, L.out, M, resid(1.0f));
            layernorm(x, d, L.conv_ln_w, L.conv_ln_b, nullptr, ln);
            if (++dbg_cnt == dbg_stop) return PK_OK;
            // ConformerConvModule (encoder.cpp:59-75); cached: causal, over each stream's conv cache (streaming_encoder.cpp:41-80)
            EpiParams eg;
            eg.kind = EPI_GLU_F32;
            eg.out_f32 = glu;
            eg.ldo = d;
            gemm(ln, d, L.pw1, M, eg);
            {
                Scope sc(this, CAT_DWCONV);
                const bool ok = cached
                    ? launch_stream_dwconv(glu, d_row_off, s_act, n_act, ss->convc + (size_t)i * ss->S * (c.conv_kernel - 1) * d, d, c.conv_kernel,
                                           L.dw_w, L.dw_b, cv, stream)
                    : launch_dwconv_bn_silu(glu, d_row_off, n_utt, maxT, d, c.conv_kernel, L.dw_wt, L.dw_b, cv, stream);
                if (!ok) return fail(PK_ERR_INVALID, "unsupported conv_kernel");
            }
            ++launches;
            gemm(cv, d, L.pw2, M, resid(1.0f));
            layernorm(x, d, L.ffn_ln_w[1], L.ffn_ln_b[1], nullptr, ln);
            if (++dbg_cnt == dbg_stop) return PK_OK;
        }
        if (layers_out_host) {
            PK_CUDA(cudaMemcpyAsync(layers_out_host + (size_t)i * M * d, x, (size_t)M * d * 4, cudaMemcpyDeviceToHost, stream));
        }
    }
    PK_CUDA(cudaGetLastError());
    return PK_OK;
}

// encoder output as a GEMM operand
static Act enc_operand(pk_engine *e) {
    if (e->cfg.math == PK_MATH_FP32) {
        Act a;
        a.f32 = e->x;
        return a;
    }
    return e->ln;
}

// The CTC head and the frame arg-max, then decoder `dec` in the same CAT_CTC scope: the greedy collapse (or, boosted,
// log-probs + boost as phrase_boost.cpp:94-102), the per-frame top-W and the beam search, one CTA per utterance
// (ctc_beam.cu), or the alignment of the targets of pk_set_align_targets (ctc_align.cu), which overwrites the frame labels
// and confidences of the arg-max with its best path, then the greedy collapse of that path.  The decoders that read the
// log-probs find them in the idle qkv workspace unless the caller gives a destination.
pk_status pk_engine::run_ctc(pk_decoder dec, float *logprobs_dev) {
    const pk_config &c = cfg;
    if (!c.has_ctc) return fail(PK_ERR_INVALID, "this model has no CTC head");
    const bool greedy = dec == PK_DECODER_CTC;
    if (!logprobs_dev && (!greedy || boosting())) {
        if ((size_t)M * c.vocab > (size_t)Bmax * Tmax * 3 * c.d_model) return fail(PK_ERR_CAPACITY, "CTC decode: workspace too small for the log-probs");
        logprobs_dev = qkv;
    }
    const int ldv = (c.vocab + 3) & ~3;
    EpiParams ep;
    ep.kind = EPI_BIAS_F32;
    ep.out_f32 = logits;
    ep.ldo = ldv;
    gemm(enc_operand(this), c.d_model, ctc_head, M, ep);
    {
        Scope sc(this, CAT_CTC);
        launch_ctc_frame_argmax(logits, M, c.vocab, ldv, best, bconf, logprobs_dev, stream);
        if (dec == PK_DECODER_CTC_BEAM) {
            launch_ctc_frame_topk(logprobs_dev, M, c.vocab, beam_w, beam_topk_id, beam_topk_lp, beam_blank, stream);
            launch_ctc_beam(logprobs_dev, beam_topk_id, beam_topk_lp, beam_blank, d_row_off, n_utt, c.vocab, beam_w, cap, beam_lm, beam_pc,
                            beam_bp, tok, t_start, t_end, t_conf, stream);
        } else {
            if (dec == PK_DECODER_CTC_ALIGN)
                launch_ctc_align(logprobs_dev, d_row_off, n_utt, c.vocab, align_ids, align_off, align_bp, align_stride, best, bconf,
                                 align_score, align_loglik, nullptr, stream);
            if (greedy && boosting())
                launch_ctc_boosted_decode(logprobs_dev, best, bconf, d_row_off, n_utt, c.vocab, c.vocab - 1, cap, boost_trie(), tok, t_start, t_end, t_conf, stream);
            else
                launch_ctc_collapse(best, bconf, d_row_off, n_utt, c.vocab - 1, cap, tok, t_start, t_end, t_conf, stream);
        }
    }
    launches += greedy ? 2 : 3;
    last_tdt = false;
    PK_CUDA(cudaGetLastError());
    return PK_OK;
}

pk_status pk_engine::run_tdt() {
    TdtParams p{};
    p.Bpad = ((n_utt + 31) / 32) * 32; p.n_utt = n_utt; p.max_sym = cfg.max_symbols;
    p.max_steps = maxT + cap + 2; p.row_off = d_row_off; p.hbuf = hbuf;
    p.boost_on = boosting() ? 1 : 0; p.trie = boost_trie(); p.boost_bits = boost_bits; p.trie_active = trie_active; p.trie_nact = trie_nact;
    return tdt_decode(p);
}

// enc_proj for all frames at once (joint's first Linear, tdt.cpp:17), then the decode kernel with the weights and
// workspaces every decode shares.
pk_status pk_engine::tdt_decode(TdtParams &p) {
    const pk_config &c = cfg;
    EpiParams ep;
    ep.kind = EPI_BIAS_F32;
    ep.out_f32 = EP;
    ep.ldo = c.joint_hidden;
    gemm(enc_operand(this), c.d_model, enc_proj, M, ep);

    p.P = c.pred_hidden; p.J = c.joint_hidden; p.V = c.vocab; p.D = c.n_durations; p.L = c.lstm_layers;
    p.cap = cap; p.n_dur = c.n_durations;
    for (int i = 0; i < 8; ++i) p.durations[i] = c.durations[i];
    p.EP = EP; p.G0 = G0;
    for (int l = 0; l < c.lstm_layers; ++l) { p.Whh[l] = Whh_s[l]; p.Wih[l] = Wih_s[l]; p.bih[l] = bih[l]; }
    p.Wp = Wp_s; p.Wout = Wout_s; p.bout = bout;
    p.z = zbuf;
    p.overflow = tdt_ints; p.bar = reinterpret_cast<unsigned int *>(tdt_ints + Bpad);
    p.pl_max = pl_max; p.pl_sum = pl_sum;
    p.key_lab = tdt_keys; p.key_dur = tdt_keys + 3 * (size_t)Bpad;
    p.dbg = reinterpret_cast<long long *>(tdt_keys + 6 * (size_t)Bpad);
    p.tok = tok; p.t_start = t_start; p.t_end = t_end; p.t_conf = t_conf;
    // a decode without carried state starts from zero LSTM state, token = blank (SOS), t = 0 (tdt.cpp:49-59)
    if (!p.carry) PK_CUDA(cudaMemsetAsync(p.hbuf, 0, (size_t)p.P * p.Bpad * 2 * p.L * sizeof(float), stream));
    cudaError_t ce;
    {
        Scope sc(this, CAT_TDT);
        ce = launch_tdt_decode(p, num_sms, stream);
    }
    launches += 2;
    last_tdt = true;
    if (ce != cudaSuccess) return fail(PK_ERR_CUDA, std::string("tdt_decode launch: ") + cudaGetErrorString(ce));
    PK_CUDA(cudaGetLastError());
    return PK_OK;
}

// Sortformer::forward after the NEST encoder (sortformer.cpp:54-67; transformer.cpp:15-62 with pre_ln = false): projection_,
// 18 post-norm blocks
//     x = norm1_(x + out_proj(MHA(x)));   x = norm2_(x + fc2(ReLU(fc1(x))))
// then the fused speaker head.  The fp32 residual stream is t_x; every LayerNorm also writes the next GEMM's operand.
pk_status pk_engine::run_diar_head() {
    const int Dt = sf.t_hidden, H = sf.t_heads;
    const bool f32 = cfg.math == PK_MATH_FP32;
    Act xo;                                   // t_x as a GEMM operand
    if (f32) xo.f32 = t_x; else xo = t_ln;
    ActBuf planes;                            // what a LayerNorm writes besides t_x
    if (!f32) planes = t_ln;
    {
        EpiParams ep;
        ep.kind = EPI_BIAS_F32;
        ep.out_f32 = t_x;
        ep.ldo = Dt;
        gemm(enc_operand(this), cfg.d_model, t_proj, M, ep);
        if (!f32) {
            Scope sc(this, CAT_LAYERNORM);
            launch_split(t_x, (size_t)M * Dt, t_ln, stream);
            ++launches;
        }
    }
    for (const TLayerW &L : tlayers) {
        EpiParams eq;
        if (f32) {           // q | k | v fp32 [M][3 d] for the CUDA-core attention
            eq.kind = EPI_BIAS_F32;
            eq.out_f32 = t_qkv;
            eq.ldo = 3 * Dt;
        } else {             // q fp32 [M][d], k | v bf16 planes [M][2 d] for the tensor-core attention
            eq.kind = EPI_QKV_ACT;
            eq.out_f32 = t_qkv;
            eq.qcols = Dt;
            eq.act.hi = t_kv_hi;
            eq.act.lo = t_kv_lo;
            eq.ldo = 2 * Dt;
        }
        gemm(xo, Dt, L.qkv, M, eq);
        {
            Scope sc(this, CAT_MHA);
            const bool ok = f32 ? launch_mha_attention(t_qkv, 3 * Dt, d_row_off, n_utt, maxT, H, Dt / H, Dt, t_ctx, stream)
                                : launch_mha_attention_tc(t_qkv, t_kv_hi, t_kv_lo, 2 * Dt, d_row_off, n_utt, maxT, H, Dt / H, Dt, t_ctx, stream);
            if (!ok) return fail(PK_ERR_INVALID, "transformer attention: unsupported head_dim " + std::to_string(Dt / H));
        }
        ++launches;
        EpiParams er;
        er.kind = EPI_RESID_F32;
        er.out_f32 = t_x;
        er.resid = t_x;
        er.ldo = Dt;
        er.alpha = 1.0f;
        gemm(t_ctx, Dt, L.out, M, er);
        layernorm(t_x, Dt, L.n1_w, L.n1_b, t_x, planes);
        EpiParams e1;
        e1.kind = EPI_BIAS_RELU_ACT;
        e1.act = t_ff;
        e1.ldo = sf.t_ff;
        gemm(xo, Dt, L.fc1, M, e1);
        gemm(t_ff, sf.t_ff, L.fc2, M, er);
        layernorm(t_x, Dt, L.n2_w, L.n2_b, t_x, planes);
    }
    {
        Scope sc(this, CAT_HEAD);
        if (!launch_speaker_head(t_x, M, Dt, sf.max_speakers, head_w1t, head_b1, head_w2, head_b2, probs, num_sms, stream))
            return fail(PK_ERR_INVALID, "speaker head: unsupported shape");
    }
    ++launches;
    PK_CUDA(cudaGetLastError());
    return PK_OK;
}

pk_status pk_engine::fetch(pk_tokens *out) {
    if (!out || !out->ids || !out->len) return fail(PK_ERR_INVALID, "pk_tokens needs ids and len");
    const size_t n = n_utt;
    PK_CUDA(cudaMemcpyAsync(h_tok, tok, n * (1 + cap) * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    if (out->start) PK_CUDA(cudaMemcpyAsync(h_ts, t_start, n * cap * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    if (out->end) PK_CUDA(cudaMemcpyAsync(h_te, t_end, n * cap * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    if (out->conf) PK_CUDA(cudaMemcpyAsync(h_tc, t_conf, n * cap * sizeof(float), cudaMemcpyDeviceToHost, stream));
    int32_t *h_ovf = h_meta + 6 * (Bmax + 1);      // (upload_shapes uses the first 6 (n+1) ints)
    if (last_tdt) PK_CUDA(cudaMemcpyAsync(h_ovf, tdt_ints, n * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    PK_CUDA(cudaStreamSynchronize(stream));
    truncated = 0;
    if (last_tdt)
        for (size_t b = 0; b < n; ++b) truncated += h_ovf[b] != 0;
    for (size_t b = 0; b < n; ++b) {
        const int32_t len = h_tok[b * (1 + cap)];
        if (len > out->cap) return fail(PK_ERR_CAPACITY, "pk_tokens.cap too small for utterance " + std::to_string(b));
        out->len[b] = len;
        memcpy(out->ids + b * out->cap, h_tok + b * (1 + cap) + 1, (size_t)len * 4);
        if (out->start) memcpy(out->start + b * out->cap, h_ts + b * cap, (size_t)len * 4);
        if (out->end) memcpy(out->end + b * out->cap, h_te + b * cap, (size_t)len * 4);
        if (out->conf) memcpy(out->conf + b * out->cap, h_tc + b * cap, (size_t)len * 4);
    }
    return PK_OK;
}

// Runs `body` (a sequence of launches on the engine stream whose kernel arguments depend only on `key`) as ONE CUDA graph
// once the key has been seen twice: first sight runs eagerly (which also completes every lazy one-time initialisation),
// second sight captures + instantiates, later sights replay.  Falls back to plain launches if capture is not possible.
pk_status pk_engine::run_graphed(const std::string &key, const std::function<pk_status()> &body) {
    if (!use_graphs || prof_on) return body();
    if (graphs.size() >= 32 && graphs.find(key) == graphs.end()) {
        // Bound the cache at INSERTION: with variable-length audio nearly every batch shape is new.  Drop the
        // entries that never got a graph first; if the instantiated graphs alone fill it, drop those too.
        for (auto it = graphs.begin(); it != graphs.end();)
            it = it->second.exec ? std::next(it) : graphs.erase(it);
        if (graphs.size() >= 24) {
            for (auto &kv : graphs) cudaGraphExecDestroy(kv.second.exec);
            graphs.clear();
        }
    }
    auto &g = graphs[key];
    if (g.exec) {
        cudaError_t ce = cudaGraphLaunch(g.exec, stream);
        if (ce != cudaSuccess) return fail(PK_ERR_CUDA, std::string("cudaGraphLaunch: ") + cudaGetErrorString(ce));
        launches += g.launches;
        return PK_OK;
    }
    if (g.seen++ == 0) return body();
    const int64_t l0 = launches;
    cudaError_t ce = cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal);
    if (ce != cudaSuccess) return fail(PK_ERR_CUDA, std::string("cudaStreamBeginCapture: ") + cudaGetErrorString(ce));
    pk_status s = body();
    cudaGraph_t graph = nullptr;
    ce = cudaStreamEndCapture(stream, &graph);
    if (s != PK_OK || ce != cudaSuccess || !graph) {
        if (graph) cudaGraphDestroy(graph);
        cudaGetLastError();
        use_graphs = false;     // capture not possible here: stay on plain launches
        launches = l0;
        return body();
    }
    g.launches = launches - l0;
    ce = cudaGraphInstantiate(&g.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) {
        g.exec = nullptr;
        cudaGetLastError();
        use_graphs = false;
        launches = l0;
        return body();
    }
    ce = cudaGraphLaunch(g.exec, stream);
    if (ce != cudaSuccess) return fail(PK_ERR_CUDA, std::string("cudaGraphLaunch: ") + cudaGetErrorString(ce));
    return PK_OK;
}

// ===================================================================== C-ABI

extern "C" {

void pk_config_110m(pk_config *c) {
    memset(c, 0, sizeof(*c));
    c->mel_bins = 80; c->sub_channels = 256; c->d_model = 512; c->n_layers = 17; c->n_heads = 8; c->ff = 2048;
    c->conv_kernel = 9; c->vocab = 1025; c->pred_hidden = 640; c->lstm_layers = 1; c->joint_hidden = 640;
    c->n_durations = 5;
    for (int i = 0; i < 5; ++i) c->durations[i] = i;
    c->has_ctc = 1; c->joint_prefix_tdt = 1; c->max_symbols = 10;
    c->max_batch = 64; c->max_samples = 160000; c->math = PK_MATH_BF16X3;
}

void pk_config_tdt_600m(pk_config *c) {
    pk_config_110m(c);
    c->mel_bins = 128; c->d_model = 1024; c->n_layers = 24; c->ff = 4096; c->vocab = 8193; c->lstm_layers = 2;
    c->has_ctc = 0; c->joint_prefix_tdt = 0; c->max_batch = 16; c->max_samples = 480000;
}

void pk_config_rnnt_600m(pk_config *c) {
    pk_config_110m(c);
    c->d_model = 1024; c->n_layers = 24; c->ff = 4096; c->lstm_layers = 2;
    c->n_durations = 0;
    for (int i = 0; i < 8; ++i) c->durations[i] = 0;
    c->has_ctc = 0; c->joint_prefix_tdt = 0; c->max_symbols = 10; c->max_batch = 16; c->max_samples = 480000;
}

void pk_config_nemotron_600m(pk_config *c) {
    pk_config_110m(c);
    c->d_model = 1024; c->n_layers = 24; c->ff = 4096; c->vocab = 8193; c->lstm_layers = 2;
    c->has_ctc = 0; c->joint_prefix_tdt = 0; c->max_symbols = 10; c->max_batch = 64; c->max_samples = 102400;
}

int32_t pk_mel_frames(int64_t n_samples) { return (int32_t)(1 + n_samples / 160); }
int32_t pk_encoder_frames(int32_t f) { return enc_frames(f); }

const char *pk_last_error(const pk_engine *e) { return e ? e->err.c_str() : g_create_err.c_str(); }

static pk_status create_engine(const pk_config &c, const pk_sortformer_config *sf, const char *path, int device, pk_engine **out);

pk_status pk_engine_create(const pk_config *cfg, const char *path, int device, pk_engine **out) {
    if (!cfg || !path || !out) {
        g_create_err = "null argument";
        return PK_ERR_INVALID;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        g_create_err = "no CUDA device: this engine has no CPU fallback";
        return PK_ERR_CUDA;
    }
    if (device < 0 || device >= ndev) {
        g_create_err = "bad device index";
        return PK_ERR_INVALID;
    }
    const pk_config &c = *cfg;
    if (c.d_model % 128 || c.d_model % c.n_heads || c.mel_bins % 8 || c.sub_channels % 4 || c.ff % 16 ||
        c.pred_hidden % 32 || c.joint_hidden % 32 || c.lstm_layers < 1 || c.lstm_layers > PK_MAX_LSTM ||
        c.n_durations < 0 || c.n_durations > 8 || c.max_batch < 1 || c.max_samples < 400 || c.sub_channels > 1024) {
        g_create_err = "unsupported model shape in pk_config";
        return PK_ERR_INVALID;
    }
    if (c.mel_bins < 8 || c.mel_bins > MEL_NORM_THREADS) {
        g_create_err = "mel_bins must be a multiple of 8 in 8.." + std::to_string(MEL_NORM_THREADS) + " (the feature normalisation runs " +
                       std::to_string(MEL_NORM_THREADS) + " / mel_bins frame groups per block)";
        return PK_ERR_INVALID;
    }
    if (c.n_durations == 0) {      // RNN-T joint (ParakeetRNNT, rnnt.cpp:48-52)
        if (c.joint_prefix_tdt != 0 || c.has_ctc != 0) {
            g_create_err = "RNN-T model (n_durations = 0): ParakeetRNNT has keys \"joint_.\" (joint_prefix_tdt = 0) and no CTC head (has_ctc = 0)";
            return PK_ERR_INVALID;
        }
        if (c.max_symbols < 1 || c.max_symbols > 64) {
            g_create_err = "RNN-T model (n_durations = 0): max_symbols must be in 1..64";
            return PK_ERR_INVALID;
        }
    }
    if (c.math != PK_MATH_FP32 && c.math != PK_MATH_BF16X3 && c.math != PK_MATH_BF16X1) {
        g_create_err = "unknown pk_math mode";
        return PK_ERR_INVALID;
    }
    if (c.local_att_left < 0 || c.local_att_right < 0) {
        g_create_err = "local_att_left and local_att_right must be >= 0 (0, 0: full attention)";
        return PK_ERR_INVALID;
    }
    if ((c.local_att_left || c.local_att_right) && c.max_samples > PK_LOCAL_ATT_MAX_SAMPLES) {
        g_create_err = "limited-context attention supports max_samples <= " + std::to_string(PK_LOCAL_ATT_MAX_SAMPLES) +
                       " (3 h of 16 kHz audio); asked for " + std::to_string(c.max_samples);
        return PK_ERR_CAPACITY;
    }
    return create_engine(c, nullptr, path, device, out);
}

// Everything of engine creation after the config checks; sf != NULL: a Sortformer engine (pk_sortformer_create).
static pk_status create_engine(const pk_config &c, const pk_sortformer_config *sf, const char *path, int device, pk_engine **out) {
    auto e = std::make_unique<pk_engine>();
    e->cfg = c;
    if (sf) {
        e->diar = true;
        e->sf = *sf;
        e->enc_prefix = "nest_encoder_.";
        // every row through the same GEMM kernel whatever the batch: an utterance's activities do not depend on its batch
        e->skinny = false;
    }
    if (const char *ev = getenv("PK_ATTN_TC")) e->attn_tc = atoi(ev) != 0;
    if (const char *ev = getenv("PK_GEMM_CLUSTER")) e->gemm_cluster = atoi(ev);
    e->device = device;
    if (cudaSetDevice(device) != cudaSuccess) {
        g_create_err = "cudaSetDevice failed";
        return PK_ERR_CUDA;
    }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    e->num_sms = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) {
        g_create_err = "cudaStreamCreate failed";
        return PK_ERR_CUDA;
    }
    bool ev_ok = cudaEventCreateWithFlags(&e->ev_h2d, cudaEventDisableTiming) == cudaSuccess &&
                 cudaEventCreateWithFlags(&e->ev_front, cudaEventDisableTiming) == cudaSuccess &&
                 cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; i < pk_engine::H2D_CHUNKS && ev_ok; ++i)
        ev_ok = cudaEventCreateWithFlags(&e->ev_chunk[i], cudaEventDisableTiming) == cudaSuccess;
    ev_ok = ev_ok && cudaEventCreateWithFlags(&e->ev_prefetch, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_pcm_free[0], cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_pcm_free[1], cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming) == cudaSuccess;
    if (!ev_ok) {
        g_create_err = "cudaEventCreate / cudaStreamCreate failed";
        return PK_ERR_CUDA;
    }
    e->Bmax = c.max_batch;
    e->Fmax = 1 + c.max_samples / 160;
    e->Tmax = pk_encoder_frames(e->Fmax);
    // A band's table covers -W..W, W = the larger side, but never more than an utterance can reach (|i - j| <= Tmax - 1): a band
    // wider than Tmax costs what full attention costs, and its rows are those of the full table (same output bytes).
    e->pos_tmax = (c.local_att_left || c.local_att_right) ? std::min(std::max(c.local_att_left, c.local_att_right), e->Tmax - 1) + 1 : e->Tmax;
    e->f1n = conv_len(c.mel_bins);
    e->f2n = conv_len(e->f1n);
    e->f3n = conv_len(e->f2n);
    // token row capacity: RNN-T emits at most max_symbols tokens per frame, so its hypotheses are never cut
    e->cap = (c.n_durations == 0 ? c.max_symbols : 2) * e->Tmax + 8;
    pk_status s = e->load(path);
    if (s == PK_OK) s = e->alloc_workspace();
    if (s != PK_OK) {
        g_create_err = e->err;
        pk_engine_destroy(e.release());
        return s;
    }
    *out = e.release();
    return PK_OK;
}

void pk_engine_destroy(pk_engine *e) {
    if (!e) return;
    cudaSetDevice(e->device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    for (void *p : e->allocs) cudaFree(p);
    for (void *p : e->beam_tab) cudaFree(p);
    for (auto &kv : e->graphs)
        if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    for (auto &r : e->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    for (auto ev : e->ev_pool) cudaEventDestroy(ev);
    pk_stream_free(e);
    if (e->nccl_comm && nccl_api().ok) nccl_api().CommDestroy(e->nccl_comm);
    if (e->h_job) cudaFreeHost(e->h_job);
    if (e->h_pcm) cudaFreeHost(e->h_pcm);
    if (e->h_meta) cudaFreeHost(e->h_meta);
    if (e->h_tok) cudaFreeHost(e->h_tok);
    if (e->h_ts) cudaFreeHost(e->h_ts);
    if (e->h_te) cudaFreeHost(e->h_te);
    if (e->h_tc) cudaFreeHost(e->h_tc);
    if (e->h_probs) cudaFreeHost(e->h_probs);
    for (int i = 0; i < 2; ++i) {
        if (e->h_bstage[i]) cudaFreeHost(e->h_bstage[i]);
        if (e->ev_bstage[i]) cudaEventDestroy(e->ev_bstage[i]);
    }
    if (e->ev_h2d) cudaEventDestroy(e->ev_h2d);
    if (e->ev_front) cudaEventDestroy(e->ev_front);
    for (int i = 0; i < pk_engine::H2D_CHUNKS; ++i)
        if (e->ev_chunk[i]) cudaEventDestroy(e->ev_chunk[i]);
    if (e->ev_prefetch) cudaEventDestroy(e->ev_prefetch);
    for (int i = 0; i < 2; ++i)
        if (e->ev_pcm_free[i]) cudaEventDestroy(e->ev_pcm_free[i]);
    if (e->ev_join) cudaEventDestroy(e->ev_join);
    if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

void *pk_stream(pk_engine *e) { return e ? (void *)e->stream : nullptr; }
int64_t pk_launch_count(const pk_engine *e) { return e ? e->launches : 0; }

pk_status pk_profile_begin(pk_engine *e) {
    if (!e) return PK_ERR_INVALID;
    e->prof_on = true;
    return PK_OK;
}

pk_status pk_profile_end(pk_engine *e, double *ms, int64_t *counts, double *flops, int32_t n) {
    // n >= 8: callers sized for the eight ASR classes (mel .. tdt) still get those; the diarization classes follow them
    if (!e || !ms || !counts || n < pk_engine::CAT_MHA) return PK_ERR_INVALID;
    cudaStreamSynchronize(e->stream);
    for (int i = 0; i < n; ++i) { ms[i] = 0; counts[i] = 0; if (flops) flops[i] = 0; }
    for (auto &r : e->prof) {
        float t = 0.f;
        cudaEventElapsedTime(&t, r.a, r.b);
        if (r.cat < n) {
            ms[r.cat] += t;
            counts[r.cat] += 1;
            if (flops) flops[r.cat] += r.flops;
        }
        e->ev_pool.push_back(r.a);
        e->ev_pool.push_back(r.b);
    }
    e->prof.clear();
    e->prof_on = false;
    return PK_OK;
}

const char *pk_profile_names(void) { return "mel,subsample,gemm,layernorm,attention,dwconv,ctc,tdt,mha,speaker_head"; }

pk_status pk_flush_l2(pk_engine *e) {
    if (!e) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (!e->l2_scratch) {
        e->l2_scratch_bytes = (size_t)256 << 20;   // > the 50 MB L2 of an H100
        if (cudaMalloc(&e->l2_scratch, e->l2_scratch_bytes) != cudaSuccess) return e->fail(PK_ERR_CUDA, "cudaMalloc (L2 scratch)");
        e->allocs.push_back(e->l2_scratch);
    }
    cudaError_t ce = cudaMemsetAsync(e->l2_scratch, (int)(++e->l2_flushes & 0xff), e->l2_scratch_bytes, e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("L2 flush: ") + cudaGetErrorString(ce));
    return PK_OK;
}

// Runs one GEMM through the wgmma kernel and through the fp32 CUDA-core kernel on seeded
// random data and returns max |tc - fp32| and max |fp32| (GPU self-check used by the tests).
pk_status pk_selftest_gemm(int device, int M, int N, int K, int epi_kind, int math, uint32_t seed, float *max_err,
                           float *max_ref) {
    if (cudaSetDevice(device) != cudaSuccess) return PK_ERR_CUDA;
    if (K % 64 != 0 || (epi_kind == EPI_GLU_F32 && (N & 1))) return PK_ERR_INVALID;
    const int qcols = epi_kind == EPI_QKV_ACT ? N / 3 : 0;     // fused q/k/v projection: N = 3 d -> fp32 q [M, d] + planes [M, 2 d]
    if (epi_kind == EPI_QKV_ACT && (N % 3 != 0 || qcols % 16 != 0)) return PK_ERR_INVALID;
    cudaStream_t st;
    cudaStreamCreate(&st);
    const bool act_out = epi_kind == EPI_BIAS_RELU_ACT || epi_kind == EPI_BIAS_SILU_ACT || epi_kind == EPI_BIAS_ACT ||
                         epi_kind == EPI_QKV_ACT;
    const int No = epi_kind == EPI_GLU_F32 ? N / 2 : N - qcols;
    std::vector<float> hA((size_t)M * K), hW((size_t)N * K), hb(N), hr((size_t)M * No);
    uint32_t sd = seed * 2654435761u + 12345u;
    auto rnd = [&]() { sd = sd * 1664525u + 1013904223u; return ((sd >> 8) & 0xffff) / 32768.0f - 1.0f; };
    for (auto &v : hA) v = rnd();
    for (auto &v : hW) v = rnd() * 0.1f;
    for (auto &v : hb) v = rnd();
    for (auto &v : hr) v = rnd();
    float *dA, *dW, *db, *dr, *o_ref, *o_tc, *q_ref = nullptr, *q_tc = nullptr;
    bf16 *Ah, *Al, *Wh, *Wl, *oh, *ol;
    if (qcols) { cudaMalloc(&q_ref, (size_t)M * qcols * 4); cudaMalloc(&q_tc, (size_t)M * qcols * 4); }
    cudaMalloc(&dA, hA.size() * 4); cudaMalloc(&dW, hW.size() * 4); cudaMalloc(&db, hb.size() * 4);
    cudaMalloc(&dr, hr.size() * 4); cudaMalloc(&o_ref, hr.size() * 4); cudaMalloc(&o_tc, hr.size() * 4);
    cudaMalloc(&Ah, hA.size() * 2); cudaMalloc(&Al, hA.size() * 2); cudaMalloc(&Wh, hW.size() * 2); cudaMalloc(&Wl, hW.size() * 2);
    cudaMalloc(&oh, hr.size() * 2); cudaMalloc(&ol, hr.size() * 2);
    cudaMemcpy(dA, hA.data(), hA.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dW, hW.data(), hW.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(db, hb.data(), hb.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dr, hr.data(), hr.size() * 4, cudaMemcpyHostToDevice);
    cudaDeviceSynchronize();
    ActBuf sa; sa.hi = Ah; sa.lo = Al;
    ActBuf sw; sw.hi = Wh; sw.lo = Wl;
    launch_split(dA, hA.size(), sa, st);
    launch_split(dW, hW.size(), sw, st);
    EpiParams ep;
    ep.kind = epi_kind; ep.bias = db; ep.ldo = No; ep.resid = dr; ep.alpha = 0.5f;
    ep.qcols = qcols;
    ep.out_f32 = qcols ? q_ref : o_ref;
    ActBuf ref_act; ref_act.f32 = o_ref;
    ep.act = ref_act;
    launch_gemm_simt(dA, K, dW, K, M, N, K, ep, st);
    TcOperand ta, tw;
    pk_status rc = PK_OK;
    const int cl = getenv("PK_GEMM_CLUSTER") ? atoi(getenv("PK_GEMM_CLUSTER")) : 1;
    TcOperand ta_sl;
    if (!make_tc_operand(&ta, Ah, Al, M, K, 128) || !make_tc_operand(&tw, Wh, Wl, N, K, tc_tile_n(N))) rc = PK_ERR_CUDA;
    if (rc == PK_OK && (cl == 2 || cl == 4) && !make_tc_operand(&ta_sl, Ah, Al, M, K, 128 / cl)) rc = PK_ERR_CUDA;
    if (rc == PK_OK) {
        ep.out_f32 = qcols ? q_tc : o_tc;
        ActBuf tc_act; tc_act.hi = oh; tc_act.lo = ol;
        ep.act = tc_act;
        const bool use_skinny = getenv("PK_SELFTEST_SKINNY") && atoi(getenv("PK_SELFTEST_SKINNY")) && M <= 128;
        float *sws = nullptr;
        unsigned int *stk = nullptr;
        if (use_skinny) {           // the few-row kernel (gemm_skinny.cu) on the same operands
            cudaMalloc(&sws, ((size_t)2 << 20) * sizeof(float));
            cudaMalloc(&stk, 1024 * sizeof(unsigned int));
            cudaMemsetAsync(stk, 0, 1024 * sizeof(unsigned int), st);
            int sms = 0;
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
            for (int rep = 0; rep < 2 && rc == PK_OK; ++rep)      // twice: the tickets must come back to zero
                if (launch_gemm_skinny(Ah, Al, K, Wh, Wl, M, N, K, math == PK_MATH_BF16X3, ep, sws, (size_t)2 << 20, stk, 1024, sms, st) != cudaSuccess) rc = PK_ERR_CUDA;
            cudaStreamSynchronize(st);
            cudaFree(sws);
            cudaFree(stk);
        } else if (launch_gemm_tc(ta, tw, M, N, K, math == PK_MATH_BF16X3, ep, st, cl, &ta_sl) != cudaSuccess) rc = PK_ERR_CUDA;
        if (rc == PK_OK && !use_skinny && getenv("PK_SELFTEST_TIME")) {   // warm, back-to-back timing of the wgmma launch
            cudaEvent_t e0, e1;
            cudaEventCreate(&e0); cudaEventCreate(&e1);
            // enough launches for a timed window of >= 50 ms (a shorter one measures clock ramp and scheduling), sized from
            // 5 warm launches
            float ms_probe = 0.f;
            cudaEventRecord(e0, st);
            for (int i = 0; i < 5; ++i) launch_gemm_tc(ta, tw, M, N, K, math == PK_MATH_BF16X3, ep, st, cl, &ta_sl);
            cudaEventRecord(e1, st);
            cudaStreamSynchronize(st);
            cudaEventElapsedTime(&ms_probe, e0, e1);
            const int reps = (int)std::min(20000.0, std::max(20.0, std::ceil(60.0 / std::max(ms_probe / 5.0, 1e-4))));
            cudaEventRecord(e0, st);
            for (int i = 0; i < reps; ++i) launch_gemm_tc(ta, tw, M, N, K, math == PK_MATH_BF16X3, ep, st, cl, &ta_sl);
            cudaEventRecord(e1, st);
            cudaStreamSynchronize(st);
            float ms = 0.f;
            cudaEventElapsedTime(&ms, e0, e1);
            const double us = 1e3 * ms / reps, tf = 2.0 * M * N * K / (us * 1e-6) / 1e12;
            fprintf(stderr, "gemm_tc M=%d N=%d K=%d epi=%d math=%d: %.2f us  %.1f TFLOP/s algorithmic (x%d MMA), %d launches in %.1f ms\n",
                    M, N, K, epi_kind, math, us, tf, math == PK_MATH_BF16X3 ? 3 : 1, reps, ms);
            cudaEventDestroy(e0); cudaEventDestroy(e1);
        }
    }
    if (cudaStreamSynchronize(st) != cudaSuccess) rc = PK_ERR_CUDA;
    if (rc == PK_OK) {
        std::vector<float> r(hr.size()), t(hr.size());
        cudaMemcpy(r.data(), o_ref, r.size() * 4, cudaMemcpyDeviceToHost);
        if (act_out) {
            std::vector<bf16> h(hr.size()), l(hr.size());
            cudaMemcpy(h.data(), oh, h.size() * 2, cudaMemcpyDeviceToHost);
            cudaMemcpy(l.data(), ol, l.size() * 2, cudaMemcpyDeviceToHost);
            for (size_t i = 0; i < t.size(); ++i) t[i] = __bfloat162float(h[i]) + __bfloat162float(l[i]);
        } else {
            cudaMemcpy(t.data(), o_tc, t.size() * 4, cudaMemcpyDeviceToHost);
        }
        float me = 0.f, mr = 0.f;
        for (size_t i = 0; i < t.size(); ++i) {
            const float e = std::fabs(t[i] - r[i]);
            if (!(e <= me)) me = e;            // NaN-propagating max
            mr = std::max(mr, std::fabs(r[i]));
        }
        if (qcols) {                           // the fp32 q columns of the fused projection
            std::vector<float> qr((size_t)M * qcols), qt((size_t)M * qcols);
            cudaMemcpy(qr.data(), q_ref, qr.size() * 4, cudaMemcpyDeviceToHost);
            cudaMemcpy(qt.data(), q_tc, qt.size() * 4, cudaMemcpyDeviceToHost);
            for (size_t i = 0; i < qt.size(); ++i) {
                const float e = std::fabs(qt[i] - qr[i]);
                if (!(e <= me)) me = e;
                mr = std::max(mr, std::fabs(qr[i]));
            }
        }
        *max_err = me;
        *max_ref = mr;
    }
    for (void *p : {(void *)dA, (void *)dW, (void *)db, (void *)dr, (void *)o_ref, (void *)o_tc, (void *)Ah, (void *)Al,
                    (void *)Wh, (void *)Wl, (void *)oh, (void *)ol, (void *)q_ref, (void *)q_tc})
        cudaFree(p);
    cudaStreamDestroy(st);
    return rc;
}

// Debug aid: cycles CTA 0 of the last TDT decode spent in {P1, B1, P2, B2, P3, B3, P4} and the
// number of lock-step decode steps (out[7]).
pk_status pk_debug_tdt_phases(pk_engine *e, int64_t *out8) {
    if (!e || !out8) return PK_ERR_INVALID;
    cudaStreamSynchronize(e->stream);
    cudaMemcpy(out8, e->tdt_keys + 6 * (size_t)e->Bpad, 8 * sizeof(int64_t), cudaMemcpyDeviceToHost);
    return PK_OK;
}

// Debug aid: cycles CTA 0 spent in the sections of the decode kernel's passes since the last call
// {x staging, products, partial store + cluster barrier, DSMEM gather + finalise, number of passes}.
pk_status pk_debug_tdt_passes(pk_engine *e, int64_t *out8) {
    if (!e || !out8) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream);
    long long v[8];
    tdt_pass_profile(v, true);
    for (int i = 0; i < 8; ++i) out8[i] = v[i];
    return PK_OK;
}

pk_status pk_sync(pk_engine *e) {
    if (!e) return PK_ERR_INVALID;
    cudaError_t ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("sync: ") + cudaGetErrorString(ce));
    return PK_OK;
}

pk_status pk_stage_pcm(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt) {
    if (!e || !pcm || !offsets) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    pk_status s = e->set_batch_shapes(nullptr, offsets, n_utt);
    if (s) return s;
    e->pcm_src = nullptr;
    const size_t total = (size_t)e->pcm_off[n_utt];
    cudaEventSynchronize(e->ev_h2d);  // previous batch's staging copies have left the pinned buffers
    // Is the caller's buffer already page-locked and packed back to back?  Then DMA straight from it.
    bool packed = true;
    for (int i = 0; i < n_utt; ++i) packed = packed && (offsets[i] - offsets[0] == e->pcm_off[i]);
    cudaPointerAttributes at;
    const bool pinned = cudaPointerGetAttributes(&at, pcm) == cudaSuccess && at.type == cudaMemoryTypeHost;
    cudaGetLastError();   // an unregistered host pointer is not an error for us
    cudaError_t ce = cudaSuccess;
    e->front_done = false;
    if (e->pref.valid) {
        const bool same = e->pref.pcm == pcm && e->pref.n == n_utt &&
                          std::equal(e->pref.off.begin(), e->pref.off.end(), offsets);
        e->pref.valid = false;
        if (same) {      // the samples are already on their way into the second buffer: adopt it
            if ((s = e->upload_shapes())) return s;
            std::swap(e->d_pcm, e->d_pcm_alt);
            e->pcm_cur ^= 1;
            ce = cudaStreamWaitEvent(e->stream, e->ev_prefetch, 0);
            if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("prefetch wait: ") + cudaGetErrorString(ce));
            if ((s = e->run_mel())) return s;
            if ((s = e->run_conv1())) return s;
            cudaEventRecord(e->ev_pcm_free[e->pcm_cur], e->stream);
            e->front_done = true;
            return PK_OK;
        }
    }
    if (pinned && packed) {
        // DMA in utterance groups on the copy stream; mel + conv1/dw1 of a group start as soon as it has
        // landed, under the DMA of the next group (the copy of 64 x 10 s is ~0.8 ms of PCIe time).
        if ((s = e->upload_shapes())) return s;
        ce = cudaEventRecord(e->ev_front, e->stream);                  // d_pcm of the previous batch is free
        if (ce == cudaSuccess) ce = cudaStreamWaitEvent(e->copy_stream, e->ev_front, 0);
        const int nch = std::min<int>(pk_engine::H2D_CHUNKS, n_utt);
        int u0 = 0;
        for (int i = 0; i < nch && ce == cudaSuccess; ++i) {
            // group boundaries balanced by samples
            int u1 = (i == nch - 1) ? n_utt : u0 + 1;
            while (i < nch - 1 && u1 < n_utt - (nch - 1 - i) && (size_t)e->pcm_off[u1] < total * (size_t)(i + 1) / nch) ++u1;
            const size_t o0 = (size_t)e->pcm_off[u0], o1 = (size_t)e->pcm_off[u1];
            ce = cudaMemcpyAsync(e->d_pcm + o0, pcm + offsets[0] + o0, (o1 - o0) * sizeof(float), cudaMemcpyHostToDevice,
                                 e->copy_stream);
            if (ce == cudaSuccess) ce = cudaEventRecord(e->ev_chunk[i], e->copy_stream);
            if (ce == cudaSuccess) ce = cudaStreamWaitEvent(e->stream, e->ev_chunk[i], 0);
            if (ce != cudaSuccess) break;
            if ((s = e->run_mel(u0, u1))) return s;
            if ((s = e->run_conv1(u0, u1))) return s;
            u0 = u1;
        }
        if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("H2D pcm: ") + cudaGetErrorString(ce));
        cudaEventRecord(e->ev_pcm_free[e->pcm_cur], e->stream);
        e->front_done = true;
        return PK_OK;
    }
    // pageable -> pinned staging -> device, utterance by utterance so the DMA of utterance i
    // overlaps the host copy of utterance i+1; utterances are re-packed back to back
    for (int i = 0; i < n_utt && ce == cudaSuccess; ++i) {
        const size_t ns = (size_t)(offsets[i + 1] - offsets[i]);
        memcpy(e->h_pcm + e->pcm_off[i], pcm + offsets[i], ns * sizeof(float));
        ce = cudaMemcpyAsync(e->d_pcm + e->pcm_off[i], e->h_pcm + e->pcm_off[i], ns * sizeof(float),
                             cudaMemcpyHostToDevice, e->stream);
    }
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("H2D pcm: ") + cudaGetErrorString(ce));
    return e->upload_shapes();
}

pk_status pk_prefetch_pcm(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt) {
    if (!e || !pcm || !offsets) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (n_utt <= 0 || n_utt > e->Bmax) return e->fail(PK_ERR_CAPACITY, "bad batch size");
    cudaPointerAttributes at;
    const bool pinned = cudaPointerGetAttributes(&at, pcm) == cudaSuccess && at.type == cudaMemoryTypeHost;
    cudaGetLastError();
    const int64_t total = offsets[n_utt] - offsets[0];
    bool ok = pinned && total > 0;
    for (int i = 0; i < n_utt && ok; ++i) {
        const int64_t ns = offsets[i + 1] - offsets[i];
        ok = ns >= 400 && ns <= e->cfg.max_samples;
    }
    if (!ok) return e->fail(PK_ERR_INVALID, "pk_prefetch_pcm needs a page-locked, packed buffer of valid utterances");
    // the second buffer was last read by the front end of the batch before the current one
    cudaError_t ce = cudaStreamWaitEvent(e->copy_stream, e->ev_pcm_free[e->pcm_cur ^ 1], 0);
    if (ce == cudaSuccess)
        ce = cudaMemcpyAsync(e->d_pcm_alt, pcm + offsets[0], (size_t)total * sizeof(float), cudaMemcpyHostToDevice, e->copy_stream);
    if (ce == cudaSuccess) ce = cudaEventRecord(e->ev_prefetch, e->copy_stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_prefetch_pcm: ") + cudaGetErrorString(ce));
    e->pref.pcm = pcm;
    e->pref.n = n_utt;
    e->pref.off.assign(offsets, offsets + n_utt + 1);
    e->pref.valid = true;
    return PK_OK;
}

// Front end (mel + conv1/dw1; 3 launches, always plain launches) unless pk_stage_pcm already ran it
// group by group under the H2D copy.
static pk_status run_front(pk_engine *e) {
    if (e->front_done) return PK_OK;
    pk_status s;
    if ((s = e->run_mel())) return s;
    if ((s = e->run_conv1())) return s;
    cudaEventRecord(e->ev_pcm_free[e->pcm_cur], e->stream);
    e->front_done = true;
    return PK_OK;
}
// TDT and RNN-T share the decode kernel but not the joint: each decoder runs only on its own model
// (a model without a CTC head rejects PK_DECODER_CTC in run_ctc).
static pk_status check_decoder(pk_engine *e, pk_decoder dec) {
    if (e->diar) return e->fail(PK_ERR_INVALID, "a Sortformer engine has no decoder: use pk_sortformer_forward / pk_diarize_batch");
    if (dec == PK_DECODER_CTC_BEAM) {
        if (!e->cfg.has_ctc) return e->fail(PK_ERR_INVALID, "PK_DECODER_CTC_BEAM: this model has no CTC head");
        if (!e->beam_w) return e->fail(PK_ERR_INVALID, "PK_DECODER_CTC_BEAM: call pk_set_ctc_beam first");
        if (e->boosting()) return e->fail(PK_ERR_INVALID, "PK_DECODER_CTC_BEAM: phrase boosting is set (beam search does not boost)");
        return PK_OK;
    }
    if (dec == PK_DECODER_CTC_ALIGN) {
        if (!e->cfg.has_ctc) return e->fail(PK_ERR_INVALID, "PK_DECODER_CTC_ALIGN: this model has no CTC head");
        if (!e->align_rows) return e->fail(PK_ERR_INVALID, "PK_DECODER_CTC_ALIGN: call pk_set_align_targets first");
        return PK_OK;
    }
    const bool rnnt_model = e->cfg.n_durations == 0;
    if (dec == PK_DECODER_TDT && rnnt_model)
        return e->fail(PK_ERR_INVALID, "PK_DECODER_TDT on an RNN-T model (n_durations = 0): use PK_DECODER_RNNT");
    if (dec == PK_DECODER_RNNT && !rnnt_model)
        return e->fail(PK_ERR_INVALID, "PK_DECODER_RNNT on a TDT model: use PK_DECODER_TDT");
    return PK_OK;
}
// The targets must name every row of the staged batch (checked once the batch is staged)
static pk_status check_align_rows(pk_engine *e, pk_decoder dec) {
    if (dec != PK_DECODER_CTC_ALIGN || e->align_rows == e->n_utt) return PK_OK;
    return e->fail(PK_ERR_INVALID, "PK_DECODER_CTC_ALIGN: the targets have " + std::to_string(e->align_rows) + " rows, the batch " +
                                       std::to_string(e->n_utt));
}
static pk_status run_pipeline(pk_engine *e, pk_decoder dec) {   // everything after the front end
    pk_status s;
    if ((s = e->run_encoder(nullptr, nullptr))) return s;
    return e->run_decoder(dec);
}

// The ~250 launches of one batch are replayed as ONE CUDA graph once a batch shape has been seen
// twice (first sight runs eagerly, which also completes every lazy one-time initialisation).
static pk_status run_asr_graph(pk_engine *e, pk_decoder dec);
pk_status pk_run_staged(pk_engine *e, pk_decoder dec) {
    if (!e || e->n_utt <= 0) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (e->gemm_err) return e->gemm_err;
    if (pk_status ds = check_decoder(e, dec)) return ds;
    if (pk_status ds = check_align_rows(e, dec)) return ds;
    {
        pk_status fs = run_front(e);
        e->front_done = false;      // a second pk_run_staged of the same staged batch re-runs the front end
        if (fs) return fs;
    }
    return run_asr_graph(e, dec);
}

static pk_status run_asr_graph(pk_engine *e, pk_decoder dec) {
    e->align_last = false;
    // (the alignment targets live in buffers that never move: one 'a' graph serves every set of targets)
    std::string key(1, dec == PK_DECODER_CTC ? 'c' : (dec == PK_DECODER_RNNT ? 'r' : (dec == PK_DECODER_CTC_BEAM ? 'B' : (dec == PK_DECODER_CTC_ALIGN ? 'a' : 't'))));
    if (dec == PK_DECODER_CTC_BEAM) {                   // width, tables, weights: pk_set_ctc_beam drops the 'B' graphs of old tables
        const int32_t wg[2] = {e->beam_w, e->beam_gen};
        const double ab[2] = {e->beam_lm.alpha_ln10, e->beam_lm.beta};
        key.append(reinterpret_cast<const char *>(wg), sizeof(wg));
        key.append(reinterpret_cast<const char *>(ab), sizeof(ab));
    }
    // (per-row lists live in buffers that never move: one graph serves every set of lists)
    const int32_t bg = e->brows_on ? -1 : (e->boost_on ? e->boost_gen : 0);
    key.append(reinterpret_cast<const char *>(&bg), sizeof(bg));
    key.append(reinterpret_cast<const char *>(e->frame_off.data()), e->frame_off.size() * sizeof(int32_t));
    const pk_status s = e->run_graphed(key, [e, dec]() { return run_pipeline(e, dec); });
    e->align_last = s == PK_OK && dec == PK_DECODER_CTC_ALIGN;
    return s;
}

pk_status pk_fetch_tokens(pk_engine *e, pk_tokens *out) {
    if (!e) return PK_ERR_INVALID;
    if (e->diar) return e->fail(PK_ERR_INVALID, "a Sortformer engine has no decoder: use pk_fetch_probs");
    cudaSetDevice(e->device);
    return e->fetch(out);
}

pk_status pk_transcribe_batch(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, pk_decoder dec,
                              pk_tokens *out) {
    pk_status s;
    if ((s = pk_stage_pcm(e, pcm, offsets, n_utt))) return s;
    if ((s = pk_run_staged(e, dec))) return s;
    return pk_fetch_tokens(e, out);
}

pk_status pk_token_buffer(pk_engine *e, void **dev_ptr, int32_t *rows, int32_t *row_ints) {
    if (!e || !dev_ptr) return PK_ERR_INVALID;
    *dev_ptr = e->tok;
    if (rows) *rows = e->n_utt;
    if (row_ints) *row_ints = 1 + e->cap;
    return PK_OK;
}

// ===================================================================== jobs and the single exchange step
// SURVEY.md section 8e / BASELINE configs[4]: a rank transcribes its block of clips in micro-batches; the token
// rows (len, ids...) of every micro-batch are appended to a device-resident job buffer; ONE ncclAllGather of that
// buffer (on the engine stream, no host synchronisation) assembles the result of all ranks.

pk_status pk_job_begin(pk_engine *e, int64_t rows_local, int32_t world) {
    if (!e || rows_local < 1 || world < 1) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    const size_t W = 1 + (size_t)e->cap;
    if (rows_local * world > e->job_alloc_rows || !e->job_tok) {     // (grow-only; freed with the engine)
        cudaStreamSynchronize(e->stream);
        e->job_tok = e->dalloc<int32_t>((size_t)rows_local * W);
        e->job_all = e->dalloc<int32_t>((size_t)world * rows_local * W);
        if (!e->job_tok || !e->job_all) return e->fail(PK_ERR_CUDA, "cudaMalloc failed (job buffers)");
        if (e->h_job) cudaFreeHost(e->h_job);
        e->h_job_ints = (size_t)world * rows_local * W;
        if (cudaMallocHost(&e->h_job, e->h_job_ints * sizeof(int32_t)) != cudaSuccess) return e->fail(PK_ERR_CUDA, "cudaMallocHost failed (job rows)");
        e->job_alloc_rows = rows_local * world;
    }
    e->job_cap_rows = rows_local;
    e->job_world = world;
    e->job_rows = 0;
    // rows a rank does not fill (a short last block) stay (len = 0)
    cudaError_t ce = cudaMemsetAsync(e->job_tok, 0, (size_t)rows_local * W * sizeof(int32_t), e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_job_begin: ") + cudaGetErrorString(ce));
    return PK_OK;
}

pk_status pk_job_append(pk_engine *e) {
    if (!e || !e->job_tok || e->n_utt <= 0) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (e->job_rows + e->n_utt > e->job_cap_rows) return e->fail(PK_ERR_CAPACITY, "pk_job_append: job buffer full");
    const size_t W = 1 + (size_t)e->cap;
    cudaError_t ce = cudaMemcpyAsync(e->job_tok + (size_t)e->job_rows * W, e->tok, (size_t)e->n_utt * W * sizeof(int32_t),
                                     cudaMemcpyDeviceToDevice, e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_job_append: ") + cudaGetErrorString(ce));
    e->job_rows += e->n_utt;
    return PK_OK;
}

pk_status pk_job_stage_pcm(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt) {
    if (!e || !pcm || !offsets || n_utt < 1) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    const int64_t total = offsets[n_utt] - offsets[0];
    if (total <= 0) return e->fail(PK_ERR_INVALID, "pk_job_stage_pcm: empty job");
    if ((size_t)total + 8 > e->job_pcm_cap) {
        cudaStreamSynchronize(e->stream);
        e->job_pcm = e->dalloc<float>((size_t)total + 8);
        if (!e->job_pcm) return e->fail(PK_ERR_CUDA, "cudaMalloc failed (job PCM)");
        e->job_pcm_cap = (size_t)total + 8;
    }
    e->job_off.assign(n_utt + 1, 0);
    for (int i = 0; i <= n_utt; ++i) e->job_off[i] = offsets[i] - offsets[0];
    cudaError_t ce = cudaMemcpyAsync(e->job_pcm, pcm + offsets[0], (size_t)total * sizeof(float), cudaMemcpyHostToDevice, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_job_stage_pcm: ") + cudaGetErrorString(ce));
    return PK_OK;
}

pk_status pk_job_select(pk_engine *e, int32_t first, int32_t n_utt) {
    if (!e) return PK_ERR_INVALID;
    if (e->job_off.empty() || first < 0 || n_utt < 1 || (size_t)first + (size_t)n_utt > e->job_off.size() - 1)
        return e->fail(PK_ERR_INVALID, "pk_job_select: range outside the staged job");
    cudaSetDevice(e->device);
    pk_status s = e->set_batch_shapes(nullptr, e->job_off.data() + first, n_utt);
    if (s) return s;
    if ((s = e->upload_shapes())) return s;
    e->pcm_src = e->job_pcm + e->job_off[first];
    e->front_done = false;
    return PK_OK;
}

pk_status pk_nccl_unique_id(void *id128) {
    if (!id128) return PK_ERR_INVALID;
    const NcclApi &n = nccl_api();
    if (!n.ok) {
        g_create_err = n.why;
        return PK_ERR_NCCL;
    }
    NcclApi::UniqueId id;
    if (n.GetUniqueId(&id) != 0) {
        g_create_err = "ncclGetUniqueId failed";
        return PK_ERR_NCCL;
    }
    memcpy(id128, id.internal, sizeof(id.internal));
    return PK_OK;
}

pk_status pk_comm_init_rank(pk_engine *e, const void *id128, int32_t rank, int32_t world) {
    if (!e || !id128 || world < 1 || rank < 0 || rank >= world) return PK_ERR_INVALID;
    const NcclApi &n = nccl_api();
    if (!n.ok) return e->fail(PK_ERR_NCCL, n.why);
    cudaSetDevice(e->device);
    if (e->nccl_comm) {
        n.CommDestroy(e->nccl_comm);
        e->nccl_comm = nullptr;
    }
    NcclApi::UniqueId id;
    memcpy(id.internal, id128, sizeof(id.internal));
    const int rc = n.CommInitRank(&e->nccl_comm, world, id, rank);
    if (rc != 0) return e->fail(PK_ERR_NCCL, std::string("ncclCommInitRank: ") + n.GetErrorString(rc));
    e->nccl_rank = rank;
    e->nccl_world = world;
    return PK_OK;
}

pk_status pk_allgather_tokens(pk_engine *e, void *nccl_comm) {
    if (!e || !e->job_tok) return PK_ERR_INVALID;
    const NcclApi &n = nccl_api();
    if (!n.ok) return e->fail(PK_ERR_NCCL, n.why);
    void *comm = nccl_comm ? nccl_comm : e->nccl_comm;
    if (!comm) return e->fail(PK_ERR_NCCL, "pk_allgather_tokens: no communicator (pk_comm_init_rank or pass an ncclComm_t)");
    cudaSetDevice(e->device);
    const size_t cnt = (size_t)e->job_cap_rows * (1 + (size_t)e->cap);
    const int rc = n.AllGather(e->job_tok, e->job_all, cnt, /*ncclInt32*/ 2, comm, e->stream);
    if (rc != 0) return e->fail(PK_ERR_NCCL, std::string("ncclAllGather: ") + n.GetErrorString(rc));
    ++e->launches;
    return PK_OK;
}

pk_status pk_job_fetch(pk_engine *e, int32_t gathered, int32_t *rows_out, int64_t n_rows, int32_t *row_ints) {
    if (!e || !e->job_tok) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    const size_t W = 1 + (size_t)e->cap;
    if (row_ints) *row_ints = (int32_t)W;
    if (!rows_out) return PK_OK;
    const int64_t have = gathered ? e->job_world * e->job_cap_rows : e->job_cap_rows;
    if (n_rows < 0 || n_rows > have) return e->fail(PK_ERR_CAPACITY, "pk_job_fetch: more rows than the job holds");
    cudaError_t ce = cudaMemcpyAsync(e->h_job, gathered ? e->job_all : e->job_tok, (size_t)n_rows * W * sizeof(int32_t),
                                     cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_job_fetch: ") + cudaGetErrorString(ce));
    memcpy(rows_out, e->h_job, (size_t)n_rows * W * sizeof(int32_t));
    return PK_OK;
}

// ===================================================================== non-16 kHz input (SURVEY.md section 8f row 4)
// Raw samples at `src_rate` go to the device as they are; the polyphase kernel (resample.cu) writes the 16 kHz signal
// straight into the staged PCM buffer, so the resampled audio never exists on the host.
static pk_status stage_raw(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, std::vector<int64_t> &in_off) {
    in_off.assign(n_utt + 1, 0);
    for (int i = 0; i < n_utt; ++i) {
        if (offsets[i + 1] < offsets[i]) return e->fail(PK_ERR_INVALID, "offsets must be non-decreasing");
        in_off[i + 1] = in_off[i] + (offsets[i + 1] - offsets[i]);
    }
    const size_t total = (size_t)in_off[n_utt];
    if (total + 8 > e->d_raw_cap) {
        cudaStreamSynchronize(e->stream);
        e->d_raw = e->dalloc<float>(total + 8);
        if (!e->d_raw) return e->fail(PK_ERR_CUDA, "cudaMalloc failed (raw PCM)");
        e->d_raw_cap = total + 8;
    }
    if (!e->d_raw_off) {
        e->d_raw_off = e->dalloc<int64_t>(2 * ((size_t)e->Bmax + 1));
        if (!e->d_raw_off) return e->fail(PK_ERR_CUDA, "cudaMalloc failed (raw offsets)");
    }
    cudaError_t ce = cudaSuccess;
    for (int i = 0; i < n_utt && ce == cudaSuccess; ++i)      // (pageable or pinned; utterances need not be packed)
        if (in_off[i + 1] > in_off[i])
            ce = cudaMemcpyAsync(e->d_raw + in_off[i], pcm + offsets[i], (size_t)(in_off[i + 1] - in_off[i]) * sizeof(float),
                                 cudaMemcpyHostToDevice, e->stream);
    if (ce == cudaSuccess)
        ce = cudaMemcpyAsync(e->d_raw_off, in_off.data(), (size_t)(n_utt + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);   // in_off / pageable sources are the caller's
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("H2D raw pcm: ") + cudaGetErrorString(ce));
    return PK_OK;
}

pk_status pk_stage_pcm_rate(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, int32_t src_rate) {
    if (!e || !pcm || !offsets || src_rate <= 0) return PK_ERR_INVALID;
    if (src_rate == 16000) return pk_stage_pcm(e, pcm, offsets, n_utt);
    cudaSetDevice(e->device);
    if (n_utt < 1 || n_utt > e->Bmax) return e->fail(PK_ERR_CAPACITY, "bad batch size");
    std::vector<int64_t> in_off, out_off(n_utt + 1, 0);
    pk_status s = stage_raw(e, pcm, offsets, n_utt, in_off);
    if (s) return s;
    int64_t max_out = 0;
    for (int i = 0; i < n_utt; ++i) {
        const int64_t m = pk_resample_len(in_off[i + 1] - in_off[i], src_rate, 16000);
        out_off[i + 1] = out_off[i] + m;
        max_out = std::max(max_out, m);
    }
    if ((s = e->set_batch_shapes(nullptr, out_off.data(), n_utt))) return s;     // (length checks at 16 kHz)
    e->pcm_src = nullptr;
    e->pref.valid = false;
    if ((s = e->upload_shapes())) return s;
    if (!launch_resample(e->d_raw, e->d_raw_off, e->d_pcm_off, n_utt, max_out, src_rate, 16000, e->d_pcm, e->stream))
        return e->fail(PK_ERR_CUDA, "resample launch failed");
    ++e->launches;
    e->front_done = false;
    return PK_OK;
}

pk_status pk_resample_batch(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, int32_t src_rate,
                            int32_t dst_rate, float *out, const int64_t *out_offsets) {
    if (!e || !pcm || !offsets || !out || !out_offsets || src_rate <= 0 || dst_rate <= 0 || n_utt < 1) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (n_utt > e->Bmax) return e->fail(PK_ERR_CAPACITY, "bad batch size");
    std::vector<int64_t> in_off, out_off(n_utt + 1, 0);
    pk_status s = stage_raw(e, pcm, offsets, n_utt, in_off);
    if (s) return s;
    int64_t max_out = 0;
    for (int i = 0; i < n_utt; ++i) {
        const int64_t m = pk_resample_len(in_off[i + 1] - in_off[i], src_rate, dst_rate);
        if (out_offsets[i + 1] - out_offsets[i] != m) return e->fail(PK_ERR_INVALID, "pk_resample_batch: out_offsets must be prefix sums of pk_resample_len");
        out_off[i + 1] = out_off[i] + m;
        max_out = std::max(max_out, m);
    }
    const size_t total = (size_t)out_off[n_utt];
    if (total > (size_t)e->Bmax * (size_t)e->cfg.max_samples) return e->fail(PK_ERR_CAPACITY, "pk_resample_batch: output exceeds the PCM workspace");
    cudaError_t ce = cudaMemcpyAsync(e->d_raw_off + e->Bmax + 1, out_off.data(), (size_t)(n_utt + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_resample_batch: ") + cudaGetErrorString(ce));
    float *dst = e->d_pcm_alt;                       // (the second PCM buffer: the staged batch stays intact)
    e->pref.valid = false;
    if (src_rate == dst_rate) {
        ce = cudaMemcpyAsync(dst, e->d_raw, total * sizeof(float), cudaMemcpyDeviceToDevice, e->stream);
    } else if (!launch_resample(e->d_raw, e->d_raw_off, e->d_raw_off + e->Bmax + 1, n_utt, max_out, src_rate, dst_rate, dst, e->stream)) {
        return e->fail(PK_ERR_CUDA, "resample launch failed");
    }
    ++e->launches;
    for (int i = 0; i < n_utt && ce == cudaSuccess; ++i)
        if (out_off[i + 1] > out_off[i])
            ce = cudaMemcpyAsync(out + out_offsets[i], dst + out_off[i], (size_t)(out_off[i + 1] - out_off[i]) * sizeof(float),
                                 cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_resample_batch: ") + cudaGetErrorString(ce));
    return PK_OK;
}

// ===================================================================== phrase boosting (SURVEY.md section 8f row 3)
// ContextTrie (src/phrase_boost.cpp:9-66) built on the host from token-id phrases, flattened to CSR (children of a node
// sorted by token) and uploaded; the decode kernels (ctc.cu: ctc_boosted_decode_kernel, tdt.cu: boost_on) walk it.
pk_status pk_engine::boost_state_alloc() {
    if (boost_bits) return PK_OK;
    const size_t W = ((size_t)cfg.vocab + 31) / 32;
    boost_bits = dalloc<uint32_t>((size_t)Bpad * W);
    trie_active = dalloc<int32_t>((size_t)Bpad * BOOST_MAX_ACTIVE);
    trie_nact = dalloc<int32_t>(Bpad);
    if (!boost_bits || !trie_active || !trie_nact) return fail(PK_ERR_CUDA, "cudaMalloc failed (boost state)");
    // the decode reads the bitmaps of the padding rows [n_utt, Bpad) too, and no launch ever writes those: they stay zero
    PK_CUDA(cudaMemsetAsync(boost_bits, 0, (size_t)Bpad * W * sizeof(uint32_t), stream));
    return PK_OK;
}

pk_status pk_engine::boost_upload(const char *fn, BoostSlots &dst, int row0, int n, int n_clear, const int32_t *phrase_ids,
                                  const int32_t *phrase_off, const int32_t *row_off, const float *boost, bool *any) {
    const int rows = n + n_clear;
    if (rows <= 0) return PK_OK;
    if (rows > Bmax) return fail(PK_ERR_CAPACITY, std::string(fn) + ": more rows than pk_config.max_batch");
    for (int k = 0; k < 2; ++k)                        // first use (a buffer or event that exists is kept: a failed attempt leaks nothing)
        if ((!ev_bstage[k] && cudaEventCreateWithFlags(&ev_bstage[k], cudaEventDisableTiming) != cudaSuccess) ||
            (!h_bstage[k] && cudaMallocHost(&h_bstage[k], (size_t)Bmax * (BOOST_SLOT_INTS + 1) * sizeof(int32_t)) != cudaSuccess))
            return fail(PK_ERR_CUDA, "cudaMallocHost failed (boost staging)");
    bstage_rows = Bmax;
    const int k = bstage_next;
    cudaEventSynchronize(ev_bstage[k]);                // the upload before last has left this buffer (normally long ago)
    int32_t *hs = h_bstage[k];
    float *hv = reinterpret_cast<float *>(hs + (size_t)bstage_rows * BOOST_SLOT_INTS);
    std::vector<int32_t> first, tk, cd;
    *any = false;
    for (int i = 0; i < rows; ++i) {
        int32_t *slot = hs + (size_t)i * BOOST_SLOT_INTS;
        slot[0] = slot[1] = 0;                         // an empty slot: the row is not boosted
        hv[i] = 0.f;
        if (i >= n || row_off[i + 1] == row_off[i]) continue;
        if (!boost_trie_csr(phrase_ids, phrase_off, row_off[i], row_off[i + 1], first, tk, cd))
            return fail(PK_ERR_INVALID, std::string(fn) + ": phrase_off must be non-decreasing");
        if ((int)first.size() - 1 > BOOST_SLOT_NODES)
            return fail(PK_ERR_CAPACITY, std::string(fn) + ": the phrases of row " + std::to_string(row0 + i) + " make a trie of " +
                                             std::to_string(first.size() - 1) + " nodes; a row holds at most " + std::to_string(BOOST_SLOT_NODES));
        memcpy(slot, first.data(), first.size() * sizeof(int32_t));
        memcpy(slot + BOOST_SLOT_NODES + 1, tk.data(), tk.size() * sizeof(int32_t));
        memcpy(slot + BOOST_SLOT_NODES + 1 + BOOST_SLOT_EDGES, cd.data(), cd.size() * sizeof(int32_t));
        hv[i] = boost[i];
        *any |= !tk.empty();
    }
    PK_CUDA(cudaMemcpyAsync(dst.slots + (size_t)row0 * BOOST_SLOT_INTS, hs, (size_t)rows * BOOST_SLOT_INTS * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
    PK_CUDA(cudaMemcpyAsync(dst.val + row0, hv, (size_t)rows * sizeof(float), cudaMemcpyHostToDevice, stream));
    PK_CUDA(cudaEventRecord(ev_bstage[k], stream));
    bstage_next = 1 - k;
    return PK_OK;
}

pk_status pk_set_ctc_beam(pk_engine *e, int32_t width, const pk_lm *lm, const pk_vocab *vocab, float alpha, float beta) {
    if (!e) return PK_ERR_INVALID;
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_set_ctc_beam: a Sortformer engine has no decoder");
    if (!e->cfg.has_ctc) return e->fail(PK_ERR_INVALID, "pk_set_ctc_beam: this model has no CTC head");
    if (width < 1 || width > PK_CTC_BEAM_MAX)
        return e->fail(PK_ERR_INVALID, "pk_set_ctc_beam: width " + std::to_string(width) + " (1.." + std::to_string(PK_CTC_BEAM_MAX) + ")");
    if (lm && !vocab) return e->fail(PK_ERR_INVALID, "pk_set_ctc_beam: a language model needs the vocabulary");
    if (!std::isfinite(alpha) || !std::isfinite(beta)) return e->fail(PK_ERR_INVALID, "pk_set_ctc_beam: alpha and beta must be finite");
    cudaSetDevice(e->device);
    if (!e->beam_bp) {
        const size_t rows = (size_t)e->Bmax * e->Tmax;
        e->beam_topk_id = e->dalloc<int32_t>(rows * PK_CTC_BEAM_MAX);
        e->beam_bp = e->dalloc<int32_t>(rows * PK_CTC_BEAM_MAX);
        e->beam_topk_lp = e->dalloc<float>(rows * PK_CTC_BEAM_MAX);
        e->beam_blank = e->dalloc<float>(rows);
        if (!e->beam_topk_id || !e->beam_bp || !e->beam_topk_lp || !e->beam_blank) {
            e->beam_bp = nullptr;
            return e->fail(PK_ERR_CUDA, "cudaMalloc failed (beam-search workspace)");
        }
    }
    // The tables are uploaded only when the LM or the vocabulary changes; a call that only repeats them (one per request)
    // costs nothing and keeps the captured graphs.  A replacement first drops the graphs that read the old tables, then
    // frees them.
    const uint64_t id = ctc_beam_tables_id(lm, vocab, e->cfg.vocab);
    if (id != e->beam_tab_id) {
        cudaStreamSynchronize(e->stream);
        for (auto it = e->graphs.begin(); it != e->graphs.end();) {
            if (it->first[0] != 'B') { ++it; continue; }
            if (it->second.exec) cudaGraphExecDestroy(it->second.exec);
            it = e->graphs.erase(it);
        }
        for (void *p : e->beam_tab) cudaFree(p);
        e->beam_tab.clear();
        e->beam_lm = DeviceLM{};
        e->beam_pc = DevicePieces{};
        e->beam_tab_id = 0;
        e->beam_w = 0;
        ++e->beam_gen;
        DeviceLM dlm;
        DevicePieces dpc;
        const std::string msg = ctc_beam_tables(lm, vocab, e->cfg.vocab, [e](const void *h, size_t bytes) -> void * {
            void *d = nullptr;
            if (cudaMalloc(&d, std::max<size_t>(bytes, 1)) != cudaSuccess) return nullptr;
            e->beam_tab.push_back(d);
            if (bytes && (cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, e->stream) != cudaSuccess ||
                          cudaStreamSynchronize(e->stream) != cudaSuccess)) return nullptr;
            return d;
        }, &dlm, &dpc);
        if (!msg.empty()) {
            for (void *p : e->beam_tab) cudaFree(p);
            e->beam_tab.clear();
            return e->fail(msg.rfind("cudaMalloc", 0) == 0 ? PK_ERR_CUDA : PK_ERR_INVALID, "pk_set_ctc_beam: " + msg);
        }
        e->beam_lm = dlm;
        e->beam_pc = dpc;
        e->beam_tab_id = id;
    }
    e->beam_lm.set_weights(alpha, beta);
    e->beam_w = width;
    return PK_OK;
}

pk_status pk_set_align_targets(pk_engine *e, const int32_t *ids, const int32_t *offsets, int32_t n_rows) {
    if (!e || n_rows < 0 || (n_rows > 0 && !offsets)) return PK_ERR_INVALID;
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_set_align_targets: a Sortformer engine has no decoder");
    if (!e->cfg.has_ctc) return e->fail(PK_ERR_INVALID, "pk_set_align_targets: this model has no CTC head");
    if (n_rows > e->Bmax) return e->fail(PK_ERR_CAPACITY, "pk_set_align_targets: more rows than pk_config.max_batch");
    for (int32_t i = 0; i < n_rows; ++i) {
        if (offsets[i] < 0 || offsets[i + 1] < offsets[i]) return e->fail(PK_ERR_INVALID, "pk_set_align_targets: offsets must be non-decreasing");
        if (offsets[i + 1] - offsets[i] > PK_ALIGN_MAX_TOKENS)
            return e->fail(PK_ERR_CAPACITY, "pk_set_align_targets: row " + std::to_string(i) + " has " + std::to_string(offsets[i + 1] - offsets[i]) +
                                                " tokens; a row holds at most " + std::to_string(PK_ALIGN_MAX_TOKENS));
    }
    const int32_t n_ids = n_rows > 0 ? offsets[n_rows] - offsets[0] : 0;
    if (n_ids > 0 && !ids) return PK_ERR_INVALID;
    for (int32_t i = 0; i < n_rows; ++i)
        for (int32_t k = offsets[i]; k < offsets[i + 1]; ++k)
            if (ids[k] < 0 || ids[k] > e->cfg.vocab - 2)
                return e->fail(PK_ERR_INVALID, "pk_set_align_targets: row " + std::to_string(i) + " has token id " + std::to_string(ids[k]) +
                                                   " (ids are 0.." + std::to_string(e->cfg.vocab - 2) + "; the blank is not a target)");
    cudaSetDevice(e->device);
    if (n_rows == 0) {
        e->align_rows = 0;
        return PK_OK;
    }
    if (!e->align_ids) {
        e->align_stride = 2 * std::min(e->Tmax, PK_ALIGN_MAX_TOKENS) + 1;
        e->align_ids = e->dalloc<int32_t>((size_t)e->Bmax * PK_ALIGN_MAX_TOKENS);
        e->align_off = e->dalloc<int32_t>((size_t)e->Bmax + 1);
        e->align_bp = e->dalloc<uint8_t>((size_t)e->Bmax * e->Tmax * e->align_stride);
        e->align_score = e->dalloc<double>(e->Bmax);
        e->align_loglik = e->dalloc<double>(e->Bmax);
        if (!e->align_ids || !e->align_off || !e->align_bp || !e->align_score || !e->align_loglik) {
            e->align_ids = nullptr;
            return e->fail(PK_ERR_CUDA, "cudaMalloc failed (alignment workspace)");
        }
    }
    // Host copies (pageable): cudaMemcpyAsync has read them when it returns, and the copies are ordered after the runs
    // still queued on the stream that read the previous targets.
    std::vector<int32_t> hid(ids ? ids + offsets[0] : nullptr, ids ? ids + offsets[0] + n_ids : nullptr), hoff(n_rows + 1);
    for (int32_t i = 0; i <= n_rows; ++i) hoff[i] = offsets[i] - offsets[0];
    cudaError_t ce = n_ids > 0 ? cudaMemcpyAsync(e->align_ids, hid.data(), (size_t)n_ids * sizeof(int32_t), cudaMemcpyHostToDevice, e->stream)
                               : cudaSuccess;
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(e->align_off, hoff.data(), hoff.size() * sizeof(int32_t), cudaMemcpyHostToDevice, e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_set_align_targets: ") + cudaGetErrorString(ce));
    e->align_rows = n_rows;
    return PK_OK;
}

pk_status pk_fetch_align_scores(pk_engine *e, double *score, double *loglik) {
    if (!e) return PK_ERR_INVALID;
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_fetch_align_scores: a Sortformer engine has no decoder");
    if (!e->align_last) return e->fail(PK_ERR_INVALID, "pk_fetch_align_scores: the last run was not an alignment (PK_DECODER_CTC_ALIGN)");
    cudaSetDevice(e->device);
    cudaError_t ce = score ? cudaMemcpyAsync(score, e->align_score, (size_t)e->n_utt * sizeof(double), cudaMemcpyDeviceToHost, e->stream)
                           : cudaSuccess;
    if (ce == cudaSuccess && loglik)
        ce = cudaMemcpyAsync(loglik, e->align_loglik, (size_t)e->n_utt * sizeof(double), cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_fetch_align_scores: ") + cudaGetErrorString(ce));
    return PK_OK;
}

pk_status pk_set_boost(pk_engine *e, const int32_t *phrase_ids, const int32_t *phrase_off, int32_t n_phrases, float boost) {
    if (!e || n_phrases < 0 || (n_phrases > 0 && (!phrase_ids || !phrase_off))) return PK_ERR_INVALID;
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_set_boost: a Sortformer engine has no decoder");
    if (e->cfg.n_durations == 0 && n_phrases > 0)
        return e->fail(PK_ERR_INVALID, "pk_set_boost: phrase boosting covers CTC and TDT decodes; this is an RNN-T model");
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream);
    ++e->boost_gen;
    e->brows_on = false;
    if (n_phrases == 0) {
        e->boost_on = false;
        return PK_OK;
    }
    std::vector<int32_t> first, tk, cd;
    if (!boost_trie_csr(phrase_ids, phrase_off, 0, n_phrases, first, tk, cd)) return e->fail(PK_ERR_INVALID, "pk_set_boost: phrase_off must be non-decreasing");
    if (tk.empty()) {       // only empty phrases
        e->boost_on = false;
        return PK_OK;
    }
    int32_t *d_first = e->upload(first), *d_tok = e->upload(tk), *d_child = e->upload(cd);
    if (!d_first || !d_tok || !d_child) return e->fail(PK_ERR_CUDA, "cudaMalloc failed (trie)");
    e->trie = DeviceTrie{};
    e->trie.first = d_first; e->trie.tok = d_tok; e->trie.child = d_child; e->trie.n_nodes = (int32_t)first.size() - 1;
    e->trie.boost = boost;
    if (pk_status s = e->boost_state_alloc()) return s;
    e->boost_on = true;
    return PK_OK;
}

pk_status pk_set_boost_rows(pk_engine *e, const int32_t *phrase_ids, const int32_t *phrase_off, const int32_t *row_off, const float *boost,
                            int32_t n_rows) {
    if (!e || n_rows < 0 || (n_rows > 0 && (!row_off || !boost))) return PK_ERR_INVALID;
    if (e->diar) return e->fail(PK_ERR_INVALID, "pk_set_boost_rows: a Sortformer engine has no decoder");
    if (n_rows > e->Bmax) return e->fail(PK_ERR_CAPACITY, "pk_set_boost_rows: more rows than pk_config.max_batch");
    for (int32_t i = 0; i < n_rows; ++i)
        if (row_off[i + 1] < row_off[i] || row_off[i] < 0) return e->fail(PK_ERR_INVALID, "pk_set_boost_rows: row_off must be non-decreasing");
    const bool lists = n_rows > 0 && row_off[n_rows] > row_off[0];
    if (lists && (!phrase_ids || !phrase_off)) return PK_ERR_INVALID;
    if (e->cfg.n_durations == 0 && lists)
        return e->fail(PK_ERR_INVALID, "pk_set_boost_rows: phrase boosting covers CTC and TDT decodes; this is an RNN-T model");
    cudaSetDevice(e->device);
    if (!lists && !e->brows.slots) {                   // nothing to boost and nothing on the device to clear
        e->boost_on = e->brows_on = false;
        return PK_OK;
    }
    if (!e->brows.slots) {
        e->brows.slots = e->dalloc<int32_t>((size_t)e->Bmax * BOOST_SLOT_INTS);
        e->brows.val = e->dalloc<float>(e->Bmax);
        e->brows.rows = e->Bmax;
        if (!e->brows.slots || !e->brows.val) return e->fail(PK_ERR_CUDA, "cudaMalloc failed (boost slots)");
        // every slot starts empty (first[0] == first[1]): a row no call has named decodes unboosted
        if (cudaMemsetAsync(e->brows.slots, 0, (size_t)e->Bmax * BOOST_SLOT_INTS * sizeof(int32_t), e->stream) != cudaSuccess ||
            cudaMemsetAsync(e->brows.val, 0, (size_t)e->Bmax * sizeof(float), e->stream) != cudaSuccess)
            return e->fail(PK_ERR_CUDA, "cudaMemset failed (boost slots)");
    }
    if (pk_status s = e->boost_state_alloc()) return s;
    bool any = false;
    const int n_clear = std::max(0, e->brows_hi - n_rows);   // rows of an earlier call that this one does not name
    if (pk_status s = e->boost_upload("pk_set_boost_rows", e->brows, 0, n_rows, n_clear, phrase_ids, phrase_off, row_off, boost, &any)) return s;
    e->brows_hi = n_rows;
    e->boost_on = false;
    e->brows_on = any;
    return PK_OK;
}

// Host-only probe of the checkpoint reader (safetensors.cpp): opens `path`, converts tensor `name` to fp32.  No device.
pk_status pk_safetensors_probe(const char *path, const char *name, float *out, int64_t cap, int64_t *numel) {
    if (!path) return PK_ERR_INVALID;
    SafeTensors st;
    std::string err;
    if (!st.open(path, err)) {
        g_create_err = err;
        return PK_ERR_IO;
    }
    if (!name) return PK_OK;
    std::vector<float> v;
    if (!st.read_f32(name, v, -1, err)) {
        g_create_err = err;
        return st.find(name) ? PK_ERR_IO : PK_ERR_MISSING;
    }
    if (numel) *numel = (int64_t)v.size();
    if (out)
        for (int64_t i = 0; i < cap && i < (int64_t)v.size(); ++i) out[i] = v[i];
    return PK_OK;
}

int32_t pk_truncated_count(const pk_engine *e) { return e ? e->truncated : 0; }

pk_status pk_mel(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, float *feats_out,
                 int32_t *n_frames_out) {
    pk_status s;
    if ((s = pk_stage_pcm(e, pcm, offsets, n_utt))) return s;
    if (!e->front_done && (s = e->run_mel())) return s;     // (a pinned caller buffer: already run group by group)
    e->front_done = false;
    const size_t n = (size_t)e->frame_off[n_utt] * e->cfg.mel_bins;
    cudaError_t ce = cudaMemcpyAsync(feats_out, e->feats, n * sizeof(float), cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_mel: ") + cudaGetErrorString(ce));
    if (n_frames_out)
        for (int i = 0; i < n_utt; ++i) n_frames_out[i] = e->frame_off[i + 1] - e->frame_off[i];
    return PK_OK;
}

pk_status pk_encode(pk_engine *e, const float *feats, const int32_t *n_frames, int32_t n_utt, float *enc_out,
                    int32_t *enc_lens_out, float *sub_out, float *layers_out) {
    if (!e || !feats || !n_frames || !enc_out) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    pk_status s = e->set_batch_shapes(n_frames, nullptr, n_utt);
    if (s) return s;
    if ((s = e->upload_shapes())) return s;
    const size_t nf = (size_t)e->frame_off[n_utt] * e->cfg.mel_bins;
    cudaError_t ce = cudaMemcpyAsync(e->feats, feats, nf * sizeof(float), cudaMemcpyHostToDevice, e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("H2D feats: ") + cudaGetErrorString(ce));
    if ((s = e->run_conv1())) return s;
    if ((s = e->run_encoder(sub_out, layers_out))) return s;
    ce = cudaMemcpyAsync(enc_out, e->x, (size_t)e->M * e->cfg.d_model * sizeof(float), cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_encode: ") + cudaGetErrorString(ce));
    if (enc_lens_out)
        for (int i = 0; i < n_utt; ++i) enc_lens_out[i] = e->row_off[i + 1] - e->row_off[i];
    return PK_OK;
}

// Stage a host encoder output as the current batch (decode-only entry points).
static pk_status stage_enc(pk_engine *e, const float *enc, const int32_t *enc_lens, int32_t n_utt) {
    if (n_utt <= 0 || n_utt > e->Bmax) return e->fail(PK_ERR_CAPACITY, "bad batch size");
    e->n_utt = n_utt;
    e->row_off.assign(n_utt + 1, 0);
    e->frame_off.assign(n_utt + 1, 0);
    e->s2_off.assign(n_utt + 1, 0);
    e->t2_rows.assign(n_utt + 1, 0);
    e->pcm_off.assign(n_utt + 1, 0);
    e->maxT = 0;
    for (int i = 0; i < n_utt; ++i) {
        if (enc_lens[i] < 1 || enc_lens[i] > e->Tmax) return e->fail(PK_ERR_CAPACITY, "encoder length out of range");
        e->row_off[i + 1] = e->row_off[i] + enc_lens[i];
        e->maxT = std::max(e->maxT, enc_lens[i]);
    }
    e->M = e->row_off[n_utt];
    pk_status s = e->band_rows_ok();
    if (!s) s = e->upload_shapes();
    if (s) return s;
    cudaError_t ce = cudaMemcpyAsync(e->x, enc, (size_t)e->M * e->cfg.d_model * sizeof(float), cudaMemcpyHostToDevice, e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("H2D enc: ") + cudaGetErrorString(ce));
    if (e->cfg.math != PK_MATH_FP32) launch_split(e->x, (size_t)e->M * e->cfg.d_model, e->ln, e->stream);
    return PK_OK;
}

pk_status pk_decode(pk_engine *e, const float *enc, const int32_t *enc_lens, int32_t n_utt, pk_decoder dec,
                    pk_tokens *out) {
    if (!e || !enc || !enc_lens) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    pk_status s;
    if ((s = check_decoder(e, dec))) return s;
    e->align_last = false;
    if ((s = stage_enc(e, enc, enc_lens, n_utt))) return s;
    if ((s = check_align_rows(e, dec))) return s;
    if ((s = e->run_decoder(dec))) return s;
    e->align_last = dec == PK_DECODER_CTC_ALIGN;
    return e->fetch(out);
}

pk_status pk_ctc_logprobs(pk_engine *e, const float *enc, int32_t total_frames, float *logprobs_out) {
    if (!e || !enc || !logprobs_out || total_frames < 1) return PK_ERR_INVALID;
    if (e->diar) return e->fail(PK_ERR_INVALID, "a Sortformer engine has no CTC head");
    cudaSetDevice(e->device);
    if (total_frames > e->Tmax) return e->fail(PK_ERR_CAPACITY, "pk_ctc_logprobs: more than Tmax frames");
    pk_status s;
    int32_t len = total_frames;
    e->align_last = false;
    if ((s = stage_enc(e, enc, &len, 1))) return s;
    // the [M][V] log-prob matrix lands in the (idle) qkv workspace
    if ((size_t)e->M * e->cfg.vocab > (size_t)e->Bmax * e->Tmax * 3 * e->cfg.d_model)
        return e->fail(PK_ERR_CAPACITY, "pk_ctc_logprobs: workspace too small");
    if ((s = e->run_ctc(PK_DECODER_CTC, e->qkv))) return s;
    cudaError_t ce = cudaMemcpyAsync(logprobs_out, e->qkv, (size_t)e->M * e->cfg.vocab * sizeof(float), cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string("pk_ctc_logprobs: ") + cudaGetErrorString(ce));
    return PK_OK;
}

// ===================================================================== Sortformer diarization (sortformer.cpp:42-122)

void pk_config_sortformer_117m(pk_sortformer_config *c) {   // make_sortformer_117m_config, sortformer.hpp:43-72
    memset(c, 0, sizeof(*c));
    pk_config &e = c->enc;
    e.mel_bins = 128; e.sub_channels = 256; e.d_model = 512; e.n_layers = 17; e.n_heads = 8; e.ff = 2048; e.conv_kernel = 9;
    e.max_batch = 16; e.max_samples = 1440000; e.math = PK_MATH_BF16X3;
    c->t_hidden = 192; c->t_layers = 18; c->t_heads = 8; c->t_ff = 768; c->max_speakers = 4;
}

pk_status pk_sortformer_create(const pk_sortformer_config *sf, const char *path, int device, pk_engine **out) {
    if (!sf || !path || !out) {
        g_create_err = "null argument";
        return PK_ERR_INVALID;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        g_create_err = "no CUDA device: this engine has no CPU fallback";
        return PK_ERR_CUDA;
    }
    if (device < 0 || device >= ndev) {
        g_create_err = "bad device index";
        return PK_ERR_INVALID;
    }
    const pk_config &c = sf->enc;
    if (c.local_att_left || c.local_att_right) {
        g_create_err = "pk_sortformer_create: the NEST encoder runs full attention (local_att_left = local_att_right = 0)";
        return PK_ERR_INVALID;
    }
    if (c.d_model % 128 || c.d_model % c.n_heads || c.mel_bins % 8 || c.sub_channels % 4 || c.ff % 16 || c.conv_kernel != 9 ||
        c.max_batch < 1 || c.max_samples < 400 || c.sub_channels > 1024) {
        g_create_err = "unsupported NEST encoder shape in pk_sortformer_config.enc";
        return PK_ERR_INVALID;
    }
    // (no feature normalisation here, but conv1 + dw1 stage 19 rows of mel_bins + 4 floats in 48 KiB of shared memory)
    if (c.mel_bins < 8 || c.mel_bins > MEL_NORM_THREADS) {
        g_create_err = "mel_bins must be a multiple of 8 in 8.." + std::to_string(MEL_NORM_THREADS);
        return PK_ERR_INVALID;
    }
    if (c.math != PK_MATH_FP32 && c.math != PK_MATH_BF16X3 && c.math != PK_MATH_BF16X1) {
        g_create_err = "unknown pk_math mode";
        return PK_ERR_INVALID;
    }
    // The transformer's GEMMs take K = t_hidden and t_ff (K % 64 for the wgmma path), the attention kernel head_dim 24, the
    // speaker head t_hidden % 32 <= 256.
    if (sf->t_layers < 1 || sf->t_heads < 1 || sf->t_hidden != 24 * sf->t_heads || sf->t_hidden % 64 || sf->t_hidden > 256 ||
        sf->t_ff < 64 || sf->t_ff % 64 || sf->max_speakers < 1 || sf->max_speakers > 64) {
        g_create_err = "unsupported Sortformer transformer shape: needs head_dim 24, t_hidden a multiple of 64 up to 256, t_ff a multiple of 64";
        return PK_ERR_INVALID;
    }
    if (speaker_head_smem(sf->t_hidden, sf->max_speakers) > 227 * 1024) {
        g_create_err = "unsupported Sortformer speaker head: its weights do not fit in shared memory (t_hidden, max_speakers)";
        return PK_ERR_INVALID;
    }
    pk_config cc = c;       // no decoder: its fields are not read
    cc.vocab = 0; cc.pred_hidden = 0; cc.lstm_layers = 0; cc.joint_hidden = 0; cc.n_durations = 0; cc.has_ctc = 0; cc.max_symbols = 0;
    memset(cc.durations, 0, sizeof(cc.durations));
    return create_engine(cc, sf, path, device, out);
}

#define PK_ECUDA(expr)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) return e->fail(PK_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)

static pk_status check_diar(pk_engine *e) {
    if (!e->diar) return e->fail(PK_ERR_INVALID, "not a Sortformer engine (pk_sortformer_create)");
    return e->gemm_err;
}

pk_status pk_fetch_probs(pk_engine *e, float *probs_out, int32_t *t_out) {
    if (!e || !probs_out) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (pk_status s = check_diar(e)) return s;
    if (!e->probs_valid) return e->fail(PK_ERR_INVALID, "pk_fetch_probs: no diarization run since the batch was staged");
    const size_t n = (size_t)e->M * e->sf.max_speakers;
    PK_ECUDA(cudaMemcpyAsync(e->h_probs, e->probs, n * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    PK_ECUDA(cudaStreamSynchronize(e->stream));
    memcpy(probs_out, e->h_probs, n * sizeof(float));
    if (t_out)
        for (int i = 0; i < e->n_utt; ++i) t_out[i] = e->row_off[i + 1] - e->row_off[i];
    return PK_OK;
}

pk_status pk_sortformer_forward(pk_engine *e, const float *feats, const int32_t *n_frames, int32_t n_utt, float *probs_out, int32_t *t_out) {
    if (!e || !feats || !n_frames || !probs_out) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    pk_status s;
    if ((s = check_diar(e))) return s;
    if ((s = e->set_batch_shapes(n_frames, nullptr, n_utt))) return s;
    if ((s = e->upload_shapes())) return s;
    const size_t nf = (size_t)e->frame_off[n_utt] * e->cfg.mel_bins;
    PK_ECUDA(cudaMemcpyAsync(e->feats, feats, nf * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    if ((s = e->run_conv1())) return s;
    if ((s = e->run_encoder(nullptr, nullptr))) return s;
    if ((s = e->run_diar_head())) return s;
    e->probs_valid = true;
    return pk_fetch_probs(e, probs_out, t_out);
}

// After pk_stage_pcm: the whole model after the front end replays as one CUDA graph per batch shape.
static pk_status run_diar_graph(pk_engine *e);
pk_status pk_run_diarize_staged(pk_engine *e) {
    if (!e || e->n_utt <= 0) return PK_ERR_INVALID;
    cudaSetDevice(e->device);
    if (pk_status s = check_diar(e)) return s;
    {
        pk_status fs = run_front(e);
        e->front_done = false;
        if (fs) return fs;
    }
    return run_diar_graph(e);
}

static pk_status run_diar_graph(pk_engine *e) {
    std::string key(1, 'd');
    key.append(reinterpret_cast<const char *>(e->frame_off.data()), e->frame_off.size() * sizeof(int32_t));
    pk_status s = e->run_graphed(key, [e]() {
        pk_status s = e->run_encoder(nullptr, nullptr);
        return s ? s : e->run_diar_head();
    });
    e->probs_valid = s == PK_OK;
    return s;
}

pk_status pk_diarize_batch(pk_engine *e, const float *pcm, const int64_t *offsets, int32_t n_utt, float *probs_out, int32_t *t_out) {
    if (!e || !probs_out) return PK_ERR_INVALID;
    pk_status s;
    if ((s = check_diar(e))) return s;
    if ((s = pk_stage_pcm(e, pcm, offsets, n_utt))) return s;
    if ((s = pk_run_diarize_staged(e))) return s;
    return pk_fetch_probs(e, probs_out, t_out);
}

// Sortformer::probs_to_segments (sortformer.cpp:70-113) on the host.
int32_t pk_diar_segments(const float *probs, int32_t T, int32_t S, float threshold, int32_t *spk, float *start, float *end, int32_t cap) {
    if (!probs || T < 0 || S < 1 || cap < 0 || (cap > 0 && (!spk || !start || !end))) return -1;
    struct Seg { int32_t s, t0, t1; };
    std::vector<Seg> segs;
    for (int s = 0; s < S; ++s) {
        int t0 = -1;
        for (int t = 0; t < T; ++t) {
            const bool active = probs[(size_t)t * S + s] > threshold;   // strictly above
            if (active && t0 < 0) t0 = t;
            else if (!active && t0 >= 0) { segs.push_back({s, t0, t - 1}); t0 = -1; }
        }
        if (t0 >= 0) segs.push_back({s, t0, T - 1});
    }
    // by start; equal starts keep speaker order (what the reference's std::sort gives for <= 16 segments, DESIGN.md section 5)
    std::stable_sort(segs.begin(), segs.end(), [](const Seg &a, const Seg &b) { return a.t0 < b.t0; });
    for (size_t i = 0; i < segs.size() && (int64_t)i < cap; ++i) {
        spk[i] = segs[i].s;
        start[i] = (float)segs[i].t0 * 0.08f;   // frame_to_seconds, timestamp.hpp:31-35
        end[i] = (float)segs[i].t1 * 0.08f;
    }
    return (int32_t)segs.size();
}

// ===================================================================== speaker-attributed transcription (diarize.cpp)

// DiarizedTranscriber holds a TDT-CTC Transcriber and a Sortformer (diarize.hpp of the reference): the pair must be an ASR
// engine with a TDT joint and a Sortformer engine on one device, decoded with CTC or TDT.  Errors land on `asr`.
static pk_status check_pair(pk_engine *asr, pk_engine *diar, pk_decoder dec) {
    if (!asr || !diar) return PK_ERR_INVALID;
    if (asr == diar || asr->diar) return asr->fail(PK_ERR_INVALID, "pk_transcribe_diarize: asr must be an ASR engine (pk_engine_create)");
    if (asr->cfg.n_durations == 0) return asr->fail(PK_ERR_INVALID, "pk_transcribe_diarize: asr is an RNN-T model; a TDT-CTC or TDT model is needed");
    if (!diar->diar) return asr->fail(PK_ERR_INVALID, "pk_transcribe_diarize: diar must be a Sortformer engine (pk_sortformer_create)");
    if (asr->device != diar->device) return asr->fail(PK_ERR_INVALID, "pk_transcribe_diarize: the two engines are on different devices");
    if (dec != PK_DECODER_CTC && dec != PK_DECODER_TDT) return asr->fail(PK_ERR_INVALID, "pk_transcribe_diarize: the decoder must be CTC or TDT");
    if (asr->gemm_err) return asr->gemm_err;
    if (diar->gemm_err) return asr->fail(diar->gemm_err, diar->err);
    return PK_OK;
}

// The batch staged on `asr` (pk_stage_pcm, pk_prefetch_pcm adoption, pk_stage_pcm_rate or pk_job_select) through both
// models.  The PCM is on the device once, in asr's buffer; diar's front end reads it there (pcm_src).
//   asr stream : [front end] [ASR graph] (wait: diar's front end has read the PCM) [ev_pcm_free]
//   diar stream: (wait: the PCM has landed) [front end] (wait: the ASR graph is done) [diarization graph]
// Every later writer of asr's PCM buffers (pk_stage_pcm's copies on either stream, pk_prefetch_pcm's wait on ev_pcm_free)
// is ordered after asr's stream at the ev_pcm_free record, so it cannot overwrite or swap the buffer before diar read it.
pk_status pk_run_transcribe_diarize_staged(pk_engine *asr, pk_engine *diar, pk_decoder dec) {
    if (pk_status s = check_pair(asr, diar, dec)) return s;
    if (asr->n_utt <= 0) return asr->fail(PK_ERR_INVALID, "pk_run_transcribe_diarize_staged: no batch staged on asr");
    cudaSetDevice(asr->device);
    pk_status s;
    if ((s = check_decoder(asr, dec))) return s;
    const int n = asr->n_utt;
    if ((s = diar->set_batch_shapes(nullptr, asr->pcm_off.data(), n)) || (s = diar->upload_shapes()))
        return asr->fail(s, diar->err);
    pk_engine *e = asr;    // (PK_ECUDA reports on e)
    // The samples have landed once the staging copies have: on the copy stream when pk_stage_pcm already ran asr's front
    // end under them (pinned buffer or adopted prefetch), else on asr's stream ahead of its (not yet launched) front end.
    PK_ECUDA(cudaEventRecord(asr->ev_join, asr->front_done ? asr->copy_stream : asr->stream));
    PK_ECUDA(cudaStreamWaitEvent(diar->stream, asr->ev_join, 0));
    diar->pcm_src = asr->pcm_src ? asr->pcm_src : asr->d_pcm;
    diar->front_done = false;
    s = run_front(diar);
    diar->pcm_src = nullptr;    // diar holds no PCM of its own for this batch
    diar->front_done = false;
    if (s) return asr->fail(s, diar->err);
    PK_ECUDA(cudaEventRecord(diar->ev_join, diar->stream));
    s = run_front(asr);
    asr->front_done = false;
    if (s == PK_OK) s = run_asr_graph(asr, dec);
    // (also on failure: the buffer is not free before diar's front end has read it)
    PK_ECUDA(cudaStreamWaitEvent(asr->stream, diar->ev_join, 0));
    PK_ECUDA(cudaEventRecord(asr->ev_pcm_free[asr->pcm_cur], asr->stream));
    if (s) return s;
    // Back to back: the diarization graph starts when the ASR graph has finished (DESIGN.md section 13: running the two
    // graphs side by side measured no faster).
    PK_ECUDA(cudaEventRecord(asr->ev_join, asr->stream));
    PK_ECUDA(cudaStreamWaitEvent(diar->stream, asr->ev_join, 0));
    s = run_diar_graph(diar);
    if (s) return asr->fail(s, diar->err);
    return PK_OK;
}

pk_status pk_transcribe_diarize_batch(pk_engine *asr, pk_engine *diar, const float *pcm, const int64_t *offsets, int32_t n_utt,
                                      pk_decoder dec, pk_tokens *tokens_out, float *probs_out, int32_t *t_out) {
    if (!pcm || !offsets || !probs_out) return asr ? asr->fail(PK_ERR_INVALID, "pk_transcribe_diarize_batch: null argument") : PK_ERR_INVALID;
    pk_status s;
    if ((s = check_pair(asr, diar, dec))) return s;
    if ((s = check_decoder(asr, dec))) return s;
    // diar's capacity before anything is staged (host-side shapes only)
    if ((s = diar->set_batch_shapes(nullptr, offsets, n_utt))) return asr->fail(s, diar->err);
    if ((s = pk_stage_pcm(asr, pcm, offsets, n_utt))) return s;
    if ((s = pk_run_transcribe_diarize_staged(asr, diar, dec))) return s;
    if ((s = pk_fetch_tokens(asr, tokens_out))) return s;
    if ((s = pk_fetch_probs(diar, probs_out, t_out))) return asr->fail(s, diar->err);
    return PK_OK;
}

// diarize_transcription (diarize.cpp:10-48): per word, the overlap min(end) - max(start) with every segment in list order,
// summed per speaker when > 0 in a std::unordered_map<int, float>, and the first speaker of the map's iteration with a
// strictly larger sum wins.  The map is kept on purpose: on an exact tie the winner is whichever the container iterates
// first (DESIGN.md section 13), and only the same container reproduces that.
pk_status pk_diarize_transcription(const float *word_start, const float *word_end, int32_t n_words, const int32_t *seg_spk,
                                   const float *seg_start, const float *seg_end, int32_t n_segs, int32_t *word_spk) {
    if (n_words < 0 || n_segs < 0 || (n_words > 0 && (!word_start || !word_end || !word_spk)) ||
        (n_segs > 0 && (!seg_spk || !seg_start || !seg_end)))
        return PK_ERR_INVALID;
    for (int32_t w = 0; w < n_words; ++w) {
        std::unordered_map<int, float> overlap_by_speaker;
        for (int32_t k = 0; k < n_segs; ++k) {
            const float overlap = std::min(word_end[w], seg_end[k]) - std::max(word_start[w], seg_start[k]);
            if (overlap > 0.0f) overlap_by_speaker[seg_spk[k]] += overlap;
        }
        float best = 0.0f;
        int32_t id = -1;
        for (const auto &kv : overlap_by_speaker)
            if (kv.second > best) {
                best = kv.second;
                id = kv.first;
            }
        word_spk[w] = id;
    }
    return PK_OK;
}

// Sortformer::probs_to_segments (sortformer.cpp:70-113) in the reference's own order -- built per speaker, then sorted by
// start with std::sort, whose introsort reorders equal starts above 16 segments (pk_diar_segments keeps speaker order
// instead) -- followed by pk_diarize_transcription on those segments.
int32_t pk_diarize_words(const float *probs, int32_t T, int32_t S, float threshold, const float *word_start, const float *word_end,
                         int32_t n_words, int32_t *word_spk, int32_t *seg_spk, float *seg_start, float *seg_end, int32_t seg_cap) {
    if (!probs || T < 0 || S < 1 || seg_cap < 0 || (seg_cap > 0 && (!seg_spk || !seg_start || !seg_end))) return -1;
    struct Seg { int32_t speaker_id; float start, end; };
    std::vector<Seg> segs;
    for (int s = 0; s < S; ++s) {
        int t0 = -1;
        for (int t = 0; t < T; ++t) {
            const bool active = probs[(size_t)t * S + s] > threshold;
            if (active && t0 < 0) t0 = t;
            else if (!active && t0 >= 0) { segs.push_back({s, (float)t0 * 0.08f, (float)(t - 1) * 0.08f}); t0 = -1; }
        }
        if (t0 >= 0) segs.push_back({s, (float)t0 * 0.08f, (float)(T - 1) * 0.08f});
    }
    std::sort(segs.begin(), segs.end(), [](const Seg &a, const Seg &b) { return a.start < b.start; });
    const int32_t ns = (int32_t)segs.size();
    std::vector<int32_t> spk(ns);
    std::vector<float> st(ns), en(ns);
    for (int32_t i = 0; i < ns; ++i) {
        spk[i] = segs[i].speaker_id;
        st[i] = segs[i].start;
        en[i] = segs[i].end;
        if (i < seg_cap) { seg_spk[i] = spk[i]; seg_start[i] = st[i]; seg_end[i] = en[i]; }
    }
    if (pk_diarize_transcription(word_start, word_end, n_words, spk.data(), st.data(), en.data(), ns, word_spk) != PK_OK) return -1;
    return ns;
}

}  // extern "C"
