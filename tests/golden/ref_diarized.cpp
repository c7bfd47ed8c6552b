// tests/golden/ref_diarized.cpp -- TEST INFRASTRUCTURE: a C-ABI around the UNMODIFIED reference's speaker-attributed
// transcription (src/diarize.cpp: diarize_transcription and DiarizedTranscriber), linked by make_golden_diarized.py (and by
// tests/test_diarize.py's fuzz, when the library exists) against the reference objects of oracle/Makefile into
// oracle/_ref/libpkref_diarized.so.  Only golden generators and that host-only fuzz load this library.
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include <axiom/axiom.hpp>
#include <axiom/graph/graph_registry.hpp>

#include "parakeet/diarize.hpp"

using namespace parakeet;
using axiom::Shape;
using axiom::Tensor;

namespace {
thread_local std::string g_err;
}

extern "C" {

const char *pkdz_last_error() { return g_err.c_str(); }

// diarize_transcription on a word list (times only; words are named "w") and a segment list in the given order.
int pkdz_transcription(const float *ws, const float *we, int nw, const int32_t *spk, const float *ss, const float *se, int ns,
                       int32_t *out) {
    std::vector<WordTimestamp> words(nw);
    for (int i = 0; i < nw; ++i) words[i] = {"w", ws[i], we[i], 1.0f};
    std::vector<DiarizationSegment> segs(ns);
    for (int i = 0; i < ns; ++i) segs[i] = {spk[i], ss[i], se[i]};
    auto r = diarize_transcription(words, segs);
    for (int i = 0; i < nw; ++i) out[i] = r[i].speaker_id;
    return 0;
}

// DiarizedTranscriber with the default configs (make_110m_config, make_sortformer_117m_config).
void *pkdz_new(const char *asr_weights, const char *sf_weights, const char *vocab) {
    try {
        return new DiarizedTranscriber(asr_weights, sf_weights, vocab);
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void pkdz_free(void *h) { delete static_cast<DiarizedTranscriber *>(h); }

// DiarizedTranscriber::transcribe(samples, decoder: 0 CTC, 1 TDT).  text: NUL-terminated; words: the DiarizedWord strings,
// one per line; w_*[i]: start, end, speaker, confidence of words[i]; wt_*[i]: start, end, confidence of word_timestamps[i]
// (word_timestamps has the same strings, checked here); segments in result order.  Returns 0, or -1 with pkdz_last_error().
int pkdz_run(void *h, const float *pcm, int n, int decoder, char *text, int text_cap, char *words, int words_cap, float *w_start,
             float *w_end, int32_t *w_spk, float *w_conf, float *wt_start, float *wt_end, float *wt_conf, int nw_cap, int *nw,
             int32_t *seg_spk, float *seg_start, float *seg_end, int ns_cap, int *ns) {
    try {
        auto *dt = static_cast<DiarizedTranscriber *>(h);
        axiom::graph::EagerModeScope eager;
        Tensor wav = Tensor::from_data(pcm, Shape{(size_t)n}, true);
        DiarizedResult r = dt->transcribe(wav, decoder == 0 ? Decoder::CTC : Decoder::TDT);
        if ((int)r.text.size() >= text_cap) throw std::runtime_error("text capacity");
        std::memcpy(text, r.text.c_str(), r.text.size() + 1);
        if ((int)r.words.size() > nw_cap || r.word_timestamps.size() != r.words.size()) throw std::runtime_error("word capacity");
        std::string all;
        for (size_t i = 0; i < r.words.size(); ++i) {
            const auto &w = r.words[i];
            const auto &t = r.word_timestamps[i];
            if (t.word != w.word) throw std::runtime_error("words and word_timestamps differ");
            all += w.word + "\n";
            w_start[i] = w.start; w_end[i] = w.end; w_spk[i] = w.speaker_id; w_conf[i] = w.confidence;
            wt_start[i] = t.start; wt_end[i] = t.end; wt_conf[i] = t.confidence;
        }
        if ((int)all.size() >= words_cap) throw std::runtime_error("words capacity");
        std::memcpy(words, all.c_str(), all.size() + 1);
        *nw = (int)r.words.size();
        if ((int)r.segments.size() > ns_cap) throw std::runtime_error("segment capacity");
        for (size_t i = 0; i < r.segments.size(); ++i) {
            seg_spk[i] = r.segments[i].speaker_id;
            seg_start[i] = r.segments[i].start;
            seg_end[i] = r.segments[i].end;
        }
        *ns = (int)r.segments.size();
        return 0;
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

}  // extern "C"
