// include/parakeet/sortformer.hpp -- header-only C++ drop-in for the reference's Sortformer diarization API
// (include/parakeet/sortformer.hpp, include/parakeet/transformer.hpp of the reference) on top of the C-ABI
// (pk_sortformer_create, pk_sortformer_forward, pk_diarize_batch, pk_diar_segments).  Offline only: the streaming
// diarize_chunk / AOSCCache of the reference are not provided.
//
// Features are host fp32 (n_frames, mel_bins) row-major, as preprocess_audio(normalize = false) makes them (or as
// Sortformer::features returns them); activities are (T', max_speakers) row-major.
#pragma once

#include "transcribe.hpp"

namespace parakeet {

struct TransformerConfig {                 // transformer.hpp:13-22
    int hidden_size = 192, num_layers = 18, num_heads = 8, ffn_intermediate = 768;
    float dropout = 0.1f, layer_norm_eps = 1e-5f;
    bool pre_ln = true, has_final_norm = false;
};

struct DiarizationSegment {                // sortformer.hpp:20-24
    int speaker_id;
    float start;                           // seconds
    float end;
};

struct SortformerConfig {                  // sortformer.hpp:28-41
    StreamingEncoderConfig nest_encoder;
    int encoder_hidden = 512, transformer_hidden = 192;
    TransformerConfig transformer;
    int max_speakers = 4;
    float activity_threshold = 0.5f;
};

inline SortformerConfig make_sortformer_117m_config() {   // sortformer.hpp:43-72
    SortformerConfig cfg;
    cfg.nest_encoder.mel_bins = 128;
    cfg.nest_encoder.hidden_size = 512;
    cfg.nest_encoder.num_layers = 17;
    cfg.nest_encoder.num_heads = 8;
    cfg.nest_encoder.ffn_intermediate = 2048;
    cfg.nest_encoder.subsampling_channels = 256;
    cfg.nest_encoder.conv_kernel_size = 9;
    cfg.nest_encoder.att_context_left = 70;
    cfg.nest_encoder.att_context_right = 0;
    cfg.nest_encoder.chunk_size = 20;
    cfg.nest_encoder.xscaling = true;
    cfg.encoder_hidden = 512;
    cfg.transformer_hidden = 192;
    cfg.transformer.hidden_size = 192;
    cfg.transformer.num_layers = 18;
    cfg.transformer.num_heads = 8;
    cfg.transformer.ffn_intermediate = 768;
    cfg.transformer.pre_ln = false;
    cfg.transformer.has_final_norm = false;
    cfg.max_speakers = 4;
    cfg.activity_threshold = 0.5f;
    return cfg;
}

// Sortformer (sortformer.hpp:98-129) on the device.  The model is the reference's post-norm preset: a SortformerConfig with
// pre_ln = true, a final norm or xscaling off is rejected.  max_batch / max_samples: the engine's capacity (utterances per
// call, samples per utterance; the preset's default is 16 x 90 s).
class Sortformer {
  public:
    explicit Sortformer(const std::string &weights_path, const SortformerConfig &config = make_sortformer_117m_config(), int device = 0,
                        int max_batch = 16, int max_samples = 90 * 16000, pk_math math = PK_MATH_BF16X3)
        : config_(config) {
        if (config.transformer.pre_ln || config.transformer.has_final_norm || !config.nest_encoder.xscaling ||
            config.encoder_hidden != config.nest_encoder.hidden_size || config.transformer_hidden != config.transformer.hidden_size)
            throw std::runtime_error("parakeet_b200: only the post-norm Sortformer with xscaling (make_sortformer_117m_config) is supported");
        pk_sortformer_config c;
        pk_config_sortformer_117m(&c);
        const StreamingEncoderConfig &e = config.nest_encoder;
        c.enc.mel_bins = e.mel_bins; c.enc.sub_channels = e.subsampling_channels; c.enc.d_model = e.hidden_size;
        c.enc.n_layers = e.num_layers; c.enc.n_heads = e.num_heads; c.enc.ff = e.ffn_intermediate; c.enc.conv_kernel = e.conv_kernel_size;
        c.enc.max_batch = max_batch; c.enc.max_samples = max_samples; c.enc.math = math;
        c.t_hidden = config.transformer.hidden_size; c.t_layers = config.transformer.num_layers; c.t_heads = config.transformer.num_heads;
        c.t_ff = config.transformer.ffn_intermediate; c.max_speakers = config.max_speakers;
        if (pk_sortformer_create(&c, weights_path.c_str(), device, &e_) != PK_OK)
            throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(nullptr));
    }
    Sortformer(const Sortformer &) = delete;
    Sortformer &operator=(const Sortformer &) = delete;
    ~Sortformer() { pk_engine_destroy(e_); }

    // Raw forward (sortformer.cpp:50-68): features (n_frames, mel_bins) -> sigmoid activities (T', max_speakers)
    std::vector<float> forward(const std::vector<float> &features) const {
        const int32_t nf = (int32_t)(features.size() / (size_t)config_.nest_encoder.mel_bins);
        std::vector<float> probs((size_t)pk_encoder_frames(nf) * config_.max_speakers);
        int32_t T = 0;
        if (pk_sortformer_forward(e_, features.data(), &nf, 1, probs.data(), &T) != PK_OK)
            throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(e_));
        return probs;
    }

    // Sortformer::diarize (sortformer.cpp:115-122): features -> segments sorted by start
    std::vector<DiarizationSegment> diarize(const std::vector<float> &features) const { return probs_to_segments(forward(features)); }

    // The whole path from 16 kHz PCM for a batch (which the reference lacks): log-mel without normalisation on the device.
    std::vector<std::vector<DiarizationSegment>> diarize_batch(const std::vector<std::vector<float>> &pcm) const {
        const int B = (int)pcm.size();
        std::vector<int64_t> off(B + 1, 0);
        size_t rows = 0;
        for (int i = 0; i < B; ++i) {
            off[i + 1] = off[i] + (int64_t)pcm[i].size();
            rows += (size_t)pk_encoder_frames(pk_mel_frames((int64_t)pcm[i].size()));
        }
        std::vector<float> buf((size_t)off[B]);
        for (int i = 0; i < B; ++i) std::copy(pcm[i].begin(), pcm[i].end(), buf.begin() + off[i]);
        std::vector<float> probs(rows * config_.max_speakers);
        std::vector<int32_t> T(B);
        if (pk_diarize_batch(e_, buf.data(), off.data(), B, probs.data(), T.data()) != PK_OK)
            throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(e_));
        std::vector<std::vector<DiarizationSegment>> out(B);
        size_t r = 0;
        for (int b = 0; b < B; ++b) {
            const float *p = probs.data() + r * config_.max_speakers;
            out[b] = probs_to_segments(std::vector<float>(p, p + (size_t)T[b] * config_.max_speakers));
            r += (size_t)T[b];
        }
        return out;
    }

    const SortformerConfig &config() const { return config_; }

  private:
    // Sortformer::probs_to_segments (sortformer.cpp:70-113), pk_diar_segments
    std::vector<DiarizationSegment> probs_to_segments(const std::vector<float> &probs) const {
        const int32_t S = config_.max_speakers, T = (int32_t)(probs.size() / (size_t)S);
        const int32_t n = pk_diar_segments(probs.data(), T, S, config_.activity_threshold, nullptr, nullptr, nullptr, 0);
        std::vector<int32_t> spk(n > 0 ? n : 1);
        std::vector<float> st(spk.size()), en(spk.size());
        pk_diar_segments(probs.data(), T, S, config_.activity_threshold, spk.data(), st.data(), en.data(), n);
        std::vector<DiarizationSegment> out;
        for (int32_t i = 0; i < n; ++i) out.push_back({spk[i], st[i], en[i]});
        return out;
    }

    SortformerConfig config_;
    pk_engine *e_ = nullptr;
};

}  // namespace parakeet
