// tests/cpp_sortformer_check.cpp -- the C++ drop-in's parakeet::Sortformer (reference sortformer.hpp:98-129 usage) on the tiny
// Sortformer test shape: forward() and diarize() of a raw fp32 feature file, then diarize_batch() of raw fp32 PCM files.
// Prints the activities and every segment.  Built and run by tests/test_sortformer.py.
#include <fstream>
#include <iostream>
#include <iterator>

#include "parakeet/sortformer.hpp"

namespace {

std::vector<float> read_f32(const char *path) {
    std::ifstream f(path, std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    const float *p = reinterpret_cast<const float *>(raw.data());
    return std::vector<float>(p, p + raw.size() / sizeof(float));
}

void print_segs(const char *tag, const std::vector<parakeet::DiarizationSegment> &segs) {
    std::cout << tag;
    for (const auto &s : segs) std::cout << " " << s.speaker_id << ":" << s.start << ":" << s.end;
    std::cout << "\n";
}

}  // namespace

int main(int argc, char **argv) {
    if (argc < 4) return 2;      // weights feats.f32 pcm.f32...
    try {
        parakeet::SortformerConfig cfg = parakeet::make_sortformer_117m_config();
        // the tiny Sortformer test shape (parakeet_cpp_b200.make_tiny_sortformer_config): head_dim 24, post-norm
        cfg.nest_encoder.subsampling_channels = 64; cfg.nest_encoder.hidden_size = 128; cfg.nest_encoder.num_layers = 2;
        cfg.nest_encoder.num_heads = 2; cfg.nest_encoder.ffn_intermediate = 256; cfg.encoder_hidden = 128;
        cfg.transformer.num_layers = 2; cfg.transformer.ffn_intermediate = 384;
        parakeet::Sortformer model(argv[1], cfg, 0, 8, 64000);
        std::cout.precision(9);
        const std::vector<float> feats = read_f32(argv[2]);
        const std::vector<float> probs = model.forward(feats);
        std::cout << "PROBS";
        for (float p : probs) std::cout << " " << p;
        std::cout << "\n";
        print_segs("DIARIZE", model.diarize(feats));
        std::vector<std::vector<float>> pcm;
        for (int i = 3; i < argc; ++i) pcm.push_back(read_f32(argv[i]));
        for (const auto &segs : model.diarize_batch(pcm)) print_segs("BATCH", segs);
        // the reference's preset is post-norm; a pre-norm config is refused
        parakeet::SortformerConfig pre = cfg;
        pre.transformer.pre_ln = true;
        try {
            parakeet::Sortformer bad(argv[1], pre);
            std::cout << "PRE_LN accepted\n";
        } catch (const std::runtime_error &) {
            std::cout << "PRE_LN refused\n";
        }
    } catch (const std::exception &e) {
        std::cerr << e.what() << "\n";
        return 1;
    }
    return 0;
}
