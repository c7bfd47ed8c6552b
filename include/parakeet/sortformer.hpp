// include/parakeet/sortformer.hpp -- header-only C++ drop-in for the reference's Sortformer diarization API
// (include/parakeet/sortformer.hpp, include/parakeet/transformer.hpp of the reference) on top of the C-ABI
// (pk_sortformer_create, pk_sortformer_forward, pk_diarize_batch, pk_diar_segments) and, for streaming diarization, the
// reference's EncoderCache / AOSCCache / Sortformer::diarize_chunk plus a lock-step batch of streams
// (DiarizationStreamingBatch, pk_diar_stream_*).
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

// AOSCCache (sortformer.hpp:76-94, sortformer.cpp:9-38): arrival-order speaker tracking on the host.  A speaker arrives the
// first time its probability is > 0.5 (fixed, not activity_threshold); within a frame speakers arrive in index order; a
// speaker is never forgotten until reset().  probs: (T, n_speakers) row-major; columns beyond max_speakers are ignored.
class AOSCCache {
  public:
    explicit AOSCCache(int max_speakers = 4) : max_speakers_(max_speakers), active_(max_speakers, false) {}
    void update(const std::vector<float> &probs, int n_speakers = -1) {
        const int S = n_speakers > 0 ? n_speakers : max_speakers_;
        const size_t T = probs.size() / (size_t)S;
        for (size_t t = 0; t < T; ++t)
            for (int s = 0; s < S && s < max_speakers_; ++s)
                if (probs[t * S + s] > 0.5f && !active_[s]) {
                    active_[s] = true;
                    order_.push_back(s);
                }
    }
    std::vector<int> speaker_order() const { return order_; }
    void reset() {
        std::fill(active_.begin(), active_.end(), false);
        order_.clear();
    }

  private:
    int max_speakers_;
    std::vector<bool> active_;
    std::vector<int> order_;
};

// EncoderCache (streaming_encoder.hpp:37-43) of the NEST encoder: a handle to one device stream slot of the Sortformer that
// first uses it (leftover mel frames, K/V rings and conv caches live on the device).  Two caches on one Sortformer are two
// independent streams; a cache is bound to one Sortformer.
struct EncoderCache {
    int frames_seen = 0;                   // encoder frames this stream has produced
    bool empty() const { return slot_ < 0; }

  private:
    friend class Sortformer;
    const void *owner_ = nullptr;
    int slot_ = -1;
};

// Sortformer (sortformer.hpp:98-129) on the device.  The model is the reference's post-norm preset: a SortformerConfig with
// pre_ln = true, a final norm or xscaling off is rejected.  max_batch / max_samples: the engine's capacity (utterances per
// call, samples per utterance; the preset's default is 16 x 90 s).
class Sortformer {
  public:
    // max_chunk_samples: the largest chunk diarize_chunk takes (its features: at most 1 + max_chunk_samples / 160 frames); the
    // streams of diarize_chunk are max_batch device slots, opened on first use.
    explicit Sortformer(const std::string &weights_path, const SortformerConfig &config = make_sortformer_117m_config(), int device = 0,
                        int max_batch = 16, int max_samples = 90 * 16000, pk_math math = PK_MATH_BF16X3, int max_chunk_samples = 16000)
        : config_(config), max_batch_(max_batch), max_chunk_(max_chunk_samples) {
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

    // Sortformer::diarize_chunk (sortformer.cpp:124-150): one chunk's features (n_frames, mel_bins), as
    // preprocess_audio(chunk, {n_mels = mel_bins, normalize = false}) makes them, through the NEST encoder's forward_chunk
    // with enc_cache, then projection_ -> transformer_ -> speaker head on this chunk's encoder frames only.  Returns {} (and
    // leaves aosc_cache alone) when fewer than 8 mel frames are available; segment times are chunk-local.
    std::vector<DiarizationSegment> diarize_chunk(const std::vector<float> &features, EncoderCache &enc_cache, AOSCCache &aosc_cache) {
        bind(enc_cache);
        const int S = max_batch_, slot = enc_cache.slot_;
        std::vector<int32_t> nf(S, 0), n_out(S, 0);
        nf[slot] = (int32_t)(features.size() / (size_t)config_.nest_encoder.mel_bins);
        std::vector<float> probs((size_t)(nf[slot] / 8 + 2) * config_.max_speakers);
        if (pk_diar_stream_step_feats(e_, features.data(), nf.data(), probs.data(), n_out.data(), nullptr, nullptr) != PK_OK)
            throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(e_));
        if (n_out[slot] == 0) return {};
        probs.resize((size_t)n_out[slot] * config_.max_speakers);
        enc_cache.frames_seen += n_out[slot];
        aosc_cache.update(probs, config_.max_speakers);
        return probs_to_segments(probs);
    }

    const SortformerConfig &config() const { return config_; }

  private:
    void bind(EncoderCache &c) {
        if (c.owner_ && c.owner_ != this) throw std::runtime_error("parakeet_b200: this EncoderCache belongs to another Sortformer");
        if (c.slot_ >= 0) return;
        if (!streams_open_) {
            if (pk_diar_stream_open(e_, max_batch_, max_chunk_, config_.nest_encoder.att_context_left) != PK_OK)
                throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(e_));
            streams_open_ = true;
        }
        if (next_slot_ >= max_batch_) throw std::runtime_error("parakeet_b200: more EncoderCaches than max_batch stream slots");
        c.owner_ = this;
        c.slot_ = next_slot_++;
        c.frames_seen = 0;
        if (pk_diar_stream_reset(e_, c.slot_) != PK_OK) throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(e_));
    }

    friend class DiarizationStreamingBatch;
    friend class DiarizedTranscriber;
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
    int max_batch_ = 16, max_chunk_ = 16000, next_slot_ = 0;
    bool streams_open_ = false;
};

// n_streams Sortformer streams in lock step (which the reference lacks; mirrors StreamingBatch): one step takes one chunk
// of 16 kHz PCM (or its features) per stream, an empty chunk meaning no input for that stream, and returns each stream's
// diarize_chunk result (chunk-local segments).  Each stream keeps its own EncoderCache and AOSCCache.
class DiarizationStreamingBatch {
  public:
    DiarizationStreamingBatch(const std::string &weights_path, int n_streams, const SortformerConfig &config = make_sortformer_117m_config(),
                              int device = 0, int max_chunk_samples = 16000, int max_samples = 30 * 16000, pk_math math = PK_MATH_BF16X3)
        : model_(weights_path, config, device, n_streams, max_samples, math, max_chunk_samples), n_(n_streams) {
        if (pk_diar_stream_open(model_.e_, n_streams, max_chunk_samples, config.nest_encoder.att_context_left) != PK_OK)
            throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(model_.e_));
        model_.streams_open_ = true;
        model_.next_slot_ = n_streams;
        base_.assign(n_streams, 0);
    }

    std::vector<std::vector<DiarizationSegment>> step(const std::vector<std::vector<float>> &pcm) {
        if ((int)pcm.size() != n_) throw std::runtime_error("parakeet_b200: one chunk per stream");
        std::vector<int64_t> off(n_ + 1, 0);
        for (int i = 0; i < n_; ++i) off[i + 1] = off[i] + (int64_t)pcm[i].size();
        std::vector<float> buf((size_t)off[n_] + 1);
        for (int i = 0; i < n_; ++i) std::copy(pcm[i].begin(), pcm[i].end(), buf.begin() + off[i]);
        std::vector<float> probs((size_t)(off[n_] / 1280 + 2 * n_ + 2) * model_.config_.max_speakers);
        std::vector<int32_t> n_out(n_);
        if (pk_diar_stream_step(model_.e_, buf.data(), off.data(), probs.data(), n_out.data(), base_.data(), nullptr) != PK_OK)
            throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(model_.e_));
        return split(probs, n_out);
    }

    // the same from features: feats[s] = (n_frames_s, mel_bins) row-major
    std::vector<std::vector<DiarizationSegment>> step_features(const std::vector<std::vector<float>> &feats) {
        if ((int)feats.size() != n_) throw std::runtime_error("parakeet_b200: one chunk per stream");
        const size_t mel = (size_t)model_.config_.nest_encoder.mel_bins;
        std::vector<int32_t> nf(n_), n_out(n_);
        std::vector<float> buf(1);
        size_t rows = 0;
        for (int i = 0; i < n_; ++i) {
            nf[i] = (int32_t)(feats[i].size() / mel);
            buf.insert(buf.end() - 1, feats[i].begin(), feats[i].end());
            rows += nf[i] / 8 + 2;
        }
        std::vector<float> probs(rows * model_.config_.max_speakers);
        if (pk_diar_stream_step_feats(model_.e_, buf.data(), nf.data(), probs.data(), n_out.data(), base_.data(), nullptr) != PK_OK)
            throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(model_.e_));
        return split(probs, n_out);
    }

    // AOSCCache::speaker_order of one stream
    std::vector<int> speaker_order(int stream) const {
        std::vector<int32_t> o(model_.config_.max_speakers > 0 ? model_.config_.max_speakers : 1);
        const int32_t n = pk_diar_stream_speakers(model_.e_, stream, o.data(), (int32_t)o.size());
        if (n < 0) throw std::runtime_error("parakeet_b200: bad stream index");
        return std::vector<int>(o.begin(), o.begin() + n);
    }
    // absolute encoder frame of the first row of the stream's last chunk (its segments are relative to it)
    int frame_base(int stream) const { return base_.at(stream); }
    void reset(int stream = -1) {
        if (pk_diar_stream_reset(model_.e_, stream) != PK_OK) throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(model_.e_));
    }
    int n_streams() const { return n_; }

  private:
    std::vector<std::vector<DiarizationSegment>> split(const std::vector<float> &probs, const std::vector<int32_t> &n_out) const {
        const int S = model_.config_.max_speakers;
        std::vector<std::vector<DiarizationSegment>> out(n_);
        size_t r = 0;
        for (int i = 0; i < n_; ++i) {
            if (n_out[i] > 0) {
                const float *p = probs.data() + r * S;
                out[i] = model_.probs_to_segments(std::vector<float>(p, p + (size_t)n_out[i] * S));
            }
            r += (size_t)n_out[i];
        }
        return out;
    }

    Sortformer model_;
    int n_;
    std::vector<int32_t> base_;
};

}  // namespace parakeet
