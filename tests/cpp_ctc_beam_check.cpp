// tests/cpp_ctc_beam_check.cpp -- Decoder::CTC_BEAM and Transcriber::set_language_model of the C++ drop-in on the device.
// Built and run by tests/test_ctc_beam.py; prints token ids for comparison with the ctypes binding, then the argument checks.
#include <cuda_runtime_api.h>

#include <fstream>
#include <iostream>

#include "parakeet/transcribe.hpp"

static std::vector<float> read_f32(const char *path) {
    std::ifstream f(path, std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    const float *p = reinterpret_cast<const float *>(raw.data());
    return std::vector<float>(p, p + raw.size() / sizeof(float));
}
static void ids(const parakeet::TranscribeResult &r) {
    std::cout << "ids";
    for (int t : r.token_ids) std::cout << " " << t;
    std::cout << "\n";
}
template <class F>
static void expect(const char *tag, F f) {
    try {
        f();
        std::cout << tag << " ok\n";
    } catch (const std::invalid_argument &) {
        std::cout << tag << " invalid_argument\n";
    } catch (const std::exception &) {
        std::cout << tag << " runtime_error\n";
    }
}

int main(int argc, char **argv) {
    if (argc < 5) return 2;       // weights vocab lm.arpa clip.f32
    try {
        parakeet::TDTCTCConfig cfg = parakeet::make_110m_config();      // the tiny test shape (oracle.make_tiny_config)
        cfg.encoder.subsampling_channels = 64; cfg.encoder.hidden_size = 128; cfg.encoder.num_layers = 2;
        cfg.encoder.num_heads = 2; cfg.encoder.ffn_intermediate = 256;
        cfg.prediction.vocab_size = 33; cfg.prediction.pred_hidden = 64; cfg.prediction.num_lstm_layers = 1;
        cfg.joint.encoder_hidden = 128; cfg.joint.pred_hidden = 64; cfg.joint.joint_hidden = 64; cfg.joint.vocab_size = 33;
        cfg.ctc_vocab_size = 33;
        parakeet::Transcriber t(argv[1], argv[2], cfg, 0, 4, 64000);
        const std::vector<float> clip = read_f32(argv[4]);
        parakeet::TranscribeOptions o;
        o.decoder = parakeet::Decoder::CTC_BEAM;
        o.beam_width = 6;
        ids(t.transcribe(clip, o));
        t.set_language_model(argv[3], 0.7f, 0.3f);
        ids(t.transcribe(clip, o));
        size_t free0 = 0, free1 = 0, total = 0;
        cudaDeviceSynchronize();
        cudaMemGetInfo(&free0, &total);
        for (int k = 0; k < 30; ++k) t.transcribe(clip, o);
        cudaDeviceSynchronize();
        cudaMemGetInfo(&free1, &total);
        std::cout << "memory_growth " << (long long)free0 - (long long)free1 << "\n";
        expect("boost", [&] {
            parakeet::TranscribeOptions b = o;
            b.boost_phrases = {"a"};
            t.transcribe(clip, b);
        });
        expect("batch_width", [&] {
            std::vector<parakeet::TranscribeOptions> v(2, o);
            v[1].beam_width = 4;
            t.transcribe_batch({clip, clip}, v);
        });
        expect("cleared", [&] {
            t.clear_language_model();
            t.transcribe(clip, o);
        });
    } catch (const std::exception &ex) {
        std::cerr << ex.what() << "\n";
        return 1;
    }
    return 0;
}
