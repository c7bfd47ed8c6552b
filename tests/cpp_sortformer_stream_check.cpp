// tests/cpp_sortformer_stream_check.cpp -- the C++ drop-in's streaming diarization on the tiny Sortformer test shape:
// parakeet::Sortformer::diarize_chunk with one EncoderCache + AOSCCache per stream (the reference's usage, features of each
// chunk), and parakeet::DiarizationStreamingBatch from PCM.  Prints, per step and stream, the segments and the arrival
// order of both, then runs the reference's AOSCCache known answers.  Built and run by tests/test_sortformer_stream.py.
//   argv: weights max_samples max_chunk_samples, then per stream s and step k (stream-major) feats.f32 pcm.f32
#include <fstream>
#include <iomanip>
#include <iostream>
#include <iterator>

#include "parakeet/sortformer.hpp"

namespace {

std::vector<float> read_f32(const std::string &path) {
    std::ifstream f(path, std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    const float *p = reinterpret_cast<const float *>(raw.data());
    return std::vector<float>(p, p + raw.size() / sizeof(float));
}

void print(const char *tag, int k, int s, const std::vector<parakeet::DiarizationSegment> &segs, const std::vector<int> &order) {
    std::cout << tag << " " << k << " " << s << "|";
    for (const auto &g : segs) std::cout << " " << g.speaker_id << ":" << g.start << ":" << g.end;
    std::cout << "|";
    for (int o : order) std::cout << " " << o;
    std::cout << "\n";
}

bool aosc_known_answers() {      // the reference's AOSCCache known answers (tests/test_all.cpp:299-341 of the reference)
    parakeet::AOSCCache c(4);
    bool ok = c.speaker_order().empty();
    c.update({0.1f, 0.9f, 0.2f, 0.8f});
    ok = ok && c.speaker_order() == std::vector<int>{1, 3};
    c.update({0.6f, 0.1f, 0.1f, 0.1f, 0.1f, 0.9f, 0.1f, 0.9f});
    ok = ok && c.speaker_order() == std::vector<int>{1, 3, 0};
    c.update({0.5f, 0.5f, 0.5f, 0.5f});
    ok = ok && c.speaker_order() == std::vector<int>{1, 3, 0};
    c.update({0.1f, 0.1f, 0.51f, 0.1f});
    ok = ok && c.speaker_order() == std::vector<int>{1, 3, 0, 2};
    c.reset();
    ok = ok && c.speaker_order().empty();
    c.update({0.1f, 0.1f, 0.9f, 0.1f});
    ok = ok && c.speaker_order() == std::vector<int>{2};
    parakeet::AOSCCache c2(2);
    c2.update({0.1f, 0.1f, 0.9f, 0.9f, 0.1f, 0.9f, 0.9f, 0.9f}, 4);
    return ok && c2.speaker_order() == std::vector<int>{1};
}

}  // namespace

int main(int argc, char **argv) {
    const int S = 3, K = 6;
    std::cout << std::setprecision(9);
    if (argc != 4 + 2 * S * K) return 2;
    try {
        parakeet::SortformerConfig cfg = parakeet::make_sortformer_117m_config();   // tiny shape (test_sortformer_stream.py)
        cfg.nest_encoder.subsampling_channels = 64;
        cfg.nest_encoder.hidden_size = cfg.encoder_hidden = 128;
        cfg.nest_encoder.num_layers = 2;
        cfg.nest_encoder.num_heads = 2;
        cfg.nest_encoder.ffn_intermediate = 256;
        cfg.transformer.num_layers = 2;
        cfg.transformer.ffn_intermediate = 384;
        const int max_samples = std::stoi(argv[2]), max_chunk = std::stoi(argv[3]);
        auto file = [&](int s, int k, int which) { return std::string(argv[4 + 2 * (s * K + k) + which]); };
        parakeet::Sortformer model(argv[1], cfg, 0, 8, max_samples, PK_MATH_BF16X3, max_chunk);
        parakeet::DiarizationStreamingBatch batch(argv[1], S, cfg, 0, max_chunk, max_samples);
        std::vector<parakeet::EncoderCache> enc(S);
        std::vector<parakeet::AOSCCache> aosc(S, parakeet::AOSCCache(cfg.max_speakers));
        for (int k = 0; k < K; ++k) {
            std::vector<std::vector<float>> pcm(S);
            for (int s = 0; s < S; ++s) pcm[s] = read_f32(file(s, k, 1));
            auto got = batch.step(pcm);
            for (int s = 0; s < S; ++s) {
                std::vector<parakeet::DiarizationSegment> segs;
                if (!pcm[s].empty()) segs = model.diarize_chunk(read_f32(file(s, k, 0)), enc[s], aosc[s]);
                print("CHUNK", k, s, segs, aosc[s].speaker_order());
                print("BATCH", k, s, got[s], batch.speaker_order(s));
            }
        }
        std::cout << (aosc_known_answers() ? "AOSC ok" : "AOSC FAILED") << "\n";
    } catch (const std::exception &e) {
        std::cerr << e.what() << "\n";
        return 1;
    }
    return 0;
}
