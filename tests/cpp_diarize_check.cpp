// tests/cpp_diarize_check.cpp -- drives include/parakeet/diarize.hpp (tests/test_diarize.py).
//   cpp_diarize_check crafted CASES.bin
//       diarize_transcription on every case of CASES.bin (int32 n; int32 w_off[n+1], s_off[n+1]; float32 ws, we [w_off[n]];
//       int32 spk, float32 ss, se [s_off[n]]); prints one line of speaker ids per case.
//   cpp_diarize_check e2e ASR.safetensors SF.safetensors VOCAB ctc|tdt MAX_SAMPLES PCM.f32...
//       DiarizedTranscriber::transcribe_batch on the clips; per clip: TEXT <text>, WORD <word> <start> <end> <speaker> <conf>
//       lines, SEG <speaker> <start> <end> lines (floats as %a).
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>

#include "parakeet/diarize.hpp"

template <class T>
static std::vector<T> take(const char *&p, size_t n) {
    std::vector<T> v(n);
    std::memcpy(v.data(), p, n * sizeof(T));
    p += n * sizeof(T);
    return v;
}

static std::vector<float> read_f32(const std::string &path) {
    std::ifstream f(path, std::ios::binary);
    std::vector<char> d((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    std::vector<float> v(d.size() / 4);
    std::memcpy(v.data(), d.data(), v.size() * 4);
    return v;
}

int main(int argc, char **argv) {
    if (argc >= 3 && std::string(argv[1]) == "crafted") {
        std::ifstream f(argv[2], std::ios::binary);
        std::vector<char> d((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        const char *p = d.data();
        const int n = take<int32_t>(p, 1)[0];
        auto w_off = take<int32_t>(p, n + 1), s_off = take<int32_t>(p, n + 1);
        auto ws = take<float>(p, w_off[n]), we = take<float>(p, w_off[n]);
        auto spk = take<int32_t>(p, s_off[n]);
        auto ss = take<float>(p, s_off[n]), se = take<float>(p, s_off[n]);
        for (int c = 0; c < n; ++c) {
            std::vector<parakeet::WordTimestamp> words;
            for (int i = w_off[c]; i < w_off[c + 1]; ++i) words.push_back({"w", ws[i], we[i], 1.0f});
            std::vector<parakeet::DiarizationSegment> segs;
            for (int i = s_off[c]; i < s_off[c + 1]; ++i) segs.push_back({spk[i], ss[i], se[i]});
            std::string line = "CASE";
            for (const auto &w : parakeet::diarize_transcription(words, segs)) line += " " + std::to_string(w.speaker_id);
            std::printf("%s\n", line.c_str());
        }
        return 0;
    }
    if (argc >= 8 && std::string(argv[1]) == "e2e") {
        parakeet::DiarizedTranscriber dt(argv[2], argv[3], argv[4], parakeet::make_110m_config(), parakeet::make_sortformer_117m_config(), 0, 8,
                                         std::atoi(argv[6]));
        dt.to_gpu();
        const parakeet::Decoder dec = std::string(argv[5]) == "ctc" ? parakeet::Decoder::CTC : parakeet::Decoder::TDT;
        std::vector<std::vector<float>> clips;
        for (int i = 7; i < argc; ++i) clips.push_back(read_f32(argv[i]));
        auto rs = dt.transcribe_batch(clips, dec);
        rs.push_back(dt.transcribe(clips[0], dec));    // the batch-1 overload gives the same result
        for (const auto &r : rs) {
            std::printf("TEXT %s\n", r.text.c_str());
            for (const auto &w : r.words) std::printf("WORD %s %a %a %d %a\n", w.word.c_str(), w.start, w.end, w.speaker_id, w.confidence);
            for (const auto &s : r.segments) std::printf("SEG %d %a %a\n", s.speaker_id, s.start, s.end);
        }
        return 0;
    }
    std::fprintf(stderr, "usage: cpp_diarize_check crafted CASES.bin | e2e ASR SF VOCAB ctc|tdt MAX_SAMPLES PCM.f32...\n");
    return 2;
}
