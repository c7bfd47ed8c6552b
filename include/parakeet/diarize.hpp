// include/parakeet/diarize.hpp -- header-only C++ drop-in for the reference's speaker-attributed transcription
// (include/parakeet/diarize.hpp, src/diarize.cpp of the reference) on top of the C-ABI (pk_transcribe_diarize_batch,
// pk_diarize_words, pk_diarize_transcription).
//
//   parakeet::DiarizedTranscriber dt("asr.safetensors", "sortformer.safetensors", "vocab.txt");
//   auto r = dt.transcribe("audio.wav");
//   for (auto &w : r.words) std::cout << "Speaker " << w.speaker_id << ": " << w.word << "\n";
//
// Same names, defaults and results as the reference.  Differences:
//   * samples are std::vector<float> or (const float*, size_t) (an axiom::Tensor overload when <axiom/axiom.hpp> is on
//     the include path), 16 kHz; transcribe(path) reads the file with read_audio (resampled to 16 kHz on the host);
//   * both models live on one CUDA device: to_gpu() is a no-op; the constructor takes the device and one capacity
//     (max_batch utterances of max_samples samples) shared by the two engines, which run bf16x3 like Transcriber;
//   * transcribe_batch() is an addition: utterances go through both models in chunks of at most max_batch, the PCM copied
//     to the device once per chunk;
//   * the ASR model is a TDT-CTC (or TDT) model; RNN-T models are refused, as the reference's Transcriber holds TDT-CTC.
// Link with libparakeet_b200.so.
#pragma once

#include "sortformer.hpp"

namespace parakeet {

struct DiarizedWord {                      // diarize.hpp:19-25
    std::string word;
    float start = 0.0f;                    // seconds
    float end = 0.0f;
    int speaker_id = -1;                   // -1 = no overlapping segment
    float confidence = 1.0f;               // from the ASR word confidence
};

struct DiarizedResult {                    // diarize.hpp:27-32
    std::string text;
    std::vector<DiarizedWord> words;
    std::vector<DiarizationSegment> segments;      // raw diarization output, in the reference's order
    std::vector<WordTimestamp> word_timestamps;    // raw ASR timestamps
};

/// Assign speaker IDs to words by maximum temporal overlap (diarize.cpp:10-48, pk_diarize_transcription).
/// Words with no overlapping segment get speaker_id = -1.
inline std::vector<DiarizedWord> diarize_transcription(const std::vector<WordTimestamp> &words, const std::vector<DiarizationSegment> &segments) {
    const size_t nw = words.size(), ns = segments.size();
    std::vector<float> ws(nw + 1), we(nw + 1), ss(ns + 1), se(ns + 1);
    std::vector<int32_t> spk(ns + 1), out(nw + 1);
    for (size_t i = 0; i < nw; ++i) { ws[i] = words[i].start; we[i] = words[i].end; }
    for (size_t i = 0; i < ns; ++i) { spk[i] = segments[i].speaker_id; ss[i] = segments[i].start; se[i] = segments[i].end; }
    if (pk_diarize_transcription(ws.data(), we.data(), (int32_t)nw, spk.data(), ss.data(), se.data(), (int32_t)ns, out.data()) != PK_OK)
        throw std::runtime_error("diarize_transcription: invalid arguments");
    std::vector<DiarizedWord> r;
    r.reserve(nw);
    for (size_t i = 0; i < nw; ++i) r.push_back({words[i].word, words[i].start, words[i].end, out[i], words[i].confidence});
    return r;
}

/// parakeet::DiarizedTranscriber (diarize.hpp:48-76 of the reference): a TDT-CTC Transcriber and a Sortformer.
class DiarizedTranscriber {
  public:
    DiarizedTranscriber(const std::string &asr_weights, const std::string &sortformer_weights, const std::string &vocab_path,
                        const TDTCTCConfig &config = make_110m_config(), const SortformerConfig &sf_config = make_sortformer_117m_config(),
                        int device = 0, int max_batch = 16, int max_samples = 30 * 16000)
        : asr_(asr_weights, vocab_path, config, device, max_batch, max_samples),
          sf_(sortformer_weights, sf_config, device, max_batch, max_samples), max_batch_(max_batch) {}

    void to_gpu() {}   // both models only ever live on the device

    DiarizedResult transcribe(const std::string &audio_path, Decoder decoder = Decoder::TDT) { return transcribe(read_audio(audio_path), decoder); }
    DiarizedResult transcribe(const std::vector<float> &samples, Decoder decoder = Decoder::TDT) { return transcribe_batch({samples}, decoder)[0]; }
    DiarizedResult transcribe(const float *samples, size_t n, Decoder decoder = Decoder::TDT) {
        return transcribe(std::vector<float>(samples, samples + n), decoder);
    }
#ifdef PARAKEET_B200_HAS_AXIOM
    DiarizedResult transcribe(const axiom::Tensor &samples, Decoder decoder = Decoder::TDT) {
        auto c = samples.cpu().ascontiguousarray();
        return transcribe(c.template typed_data<float>(), c.size(), decoder);
    }
#endif

    // Not in the reference (batch-1): many utterances, max_batch at a time, through both models in one call.
    std::vector<DiarizedResult> transcribe_batch(const std::vector<std::vector<float>> &utts, Decoder decoder = Decoder::TDT) {
        std::vector<DiarizedResult> out;
        const pk_decoder dec = asr_.pick(decoder);
        const int S = sf_.config().max_speakers;
        void *tokbuf = nullptr;
        int32_t row_ints = 0;
        pk_token_buffer(asr_.engine(), &tokbuf, nullptr, &row_ints);
        const int32_t cap = row_ints - 1;
        for (size_t i = 0; i < utts.size(); i += (size_t)max_batch_) {
            const int B = (int)std::min(utts.size() - i, (size_t)max_batch_);
            std::vector<int64_t> off(B + 1, 0);
            size_t rows = 0;
            for (int b = 0; b < B; ++b) {
                off[b + 1] = off[b] + (int64_t)utts[i + b].size();
                rows += (size_t)pk_encoder_frames(pk_mel_frames((int64_t)utts[i + b].size()));
            }
            std::vector<float> buf((size_t)off[B] + 1);
            for (int b = 0; b < B; ++b) std::copy(utts[i + b].begin(), utts[i + b].end(), buf.begin() + off[b]);
            std::vector<int32_t> ids((size_t)B * cap), st((size_t)B * cap), en((size_t)B * cap), len(B), T(B);
            std::vector<float> cf((size_t)B * cap), probs(rows * S + 1);
            pk_tokens t{cap, ids.data(), st.data(), en.data(), cf.data(), len.data()};
            if (pk_transcribe_diarize_batch(asr_.engine(), sf_.e_, buf.data(), off.data(), B, dec, &t, probs.data(), T.data()) != PK_OK)
                throw std::runtime_error(std::string("parakeet_b200: ") + pk_last_error(asr_.engine()));
            size_t r = 0;
            for (int b = 0; b < B; ++b) {
                std::vector<TimestampedToken> toks;
                std::vector<int> tid;
                for (int k = 0; k < len[b]; ++k) {
                    const size_t q = (size_t)b * cap + k;
                    toks.push_back({ids[q], st[q], en[q], cf[q]});
                    tid.push_back(ids[q]);
                }
                out.push_back(finish(asr_.tokenizer().decode(tid), asr_.tokenizer().group(toks), probs.data() + r * S, T[b], S));
                r += (size_t)T[b];
            }
        }
        return out;
    }

    Transcriber &transcriber() { return asr_; }
    Sortformer &sortformer() { return sf_; }

  private:
    // one utterance: segments in the reference's order and the speaker of every word (pk_diarize_words)
    DiarizedResult finish(std::string text, std::vector<WordTimestamp> words, const float *probs, int32_t T, int S) {
        const size_t nw = words.size();
        std::vector<float> ws(nw + 1), we(nw + 1);
        for (size_t i = 0; i < nw; ++i) { ws[i] = words[i].start; we[i] = words[i].end; }
        std::vector<int32_t> wspk(nw + 1);
        const float thr = sf_.config().activity_threshold;
        const int32_t n = pk_diarize_words(probs, T, S, thr, ws.data(), we.data(), (int32_t)nw, wspk.data(), nullptr, nullptr, nullptr, 0);
        if (n < 0) throw std::runtime_error("pk_diarize_words: invalid arguments");
        std::vector<int32_t> spk(n + 1);
        std::vector<float> ss(n + 1), se(n + 1);
        pk_diarize_words(probs, T, S, thr, ws.data(), we.data(), (int32_t)nw, wspk.data(), spk.data(), ss.data(), se.data(), n);
        DiarizedResult r;
        r.text = std::move(text);
        for (int32_t k = 0; k < n; ++k) r.segments.push_back({spk[k], ss[k], se[k]});
        for (size_t i = 0; i < nw; ++i) r.words.push_back({words[i].word, words[i].start, words[i].end, wspk[i], words[i].confidence});
        r.word_timestamps = std::move(words);
        return r;
    }

    Transcriber asr_;
    Sortformer sf_;
    int max_batch_;
};

}  // namespace parakeet
