// tests/cpp_rnnt_check.cpp -- exercises parakeet::RNNTTranscriber of the header-only C++ shim
// (include/parakeet/transcribe.hpp) on a tiny RNN-T checkpoint.  Built and run by
// tests/test_rnnt.py; prints token ids:start:end, text and words for comparison.
#include <cstdio>
#include <iostream>

#include "parakeet/transcribe.hpp"

int main(int argc, char **argv) {
    if (argc < 4) return 2;
    try {
        parakeet::RNNTConfig cfg = parakeet::make_rnnt_600m_config();
        cfg.encoder.subsampling_channels = 64; cfg.encoder.hidden_size = 128; cfg.encoder.num_layers = 2;
        cfg.encoder.num_heads = 2; cfg.encoder.ffn_intermediate = 256;
        cfg.prediction.vocab_size = 33; cfg.prediction.pred_hidden = 64; cfg.prediction.num_lstm_layers = 1;
        cfg.joint.encoder_hidden = 128; cfg.joint.pred_hidden = 64; cfg.joint.joint_hidden = 64; cfg.joint.vocab_size = 33;
        parakeet::RNNTTranscriber t(argv[1], argv[2], cfg, 0, 4, 64000);
        t.to_gpu();
        auto r = t.transcribe(std::string(argv[3]), true);
        std::cout << "TOK";
        for (auto &tk : r.timestamped_tokens) std::cout << " " << tk.token_id << ":" << tk.start_frame << ":" << tk.end_frame;
        std::cout << "\nTEXT " << r.text << "\nWORDS";
        for (auto &w : r.word_timestamps) std::cout << " " << w.word;
        std::cout << "\n";
        auto batch = t.transcribe_batch({parakeet::read_audio(argv[3])}, parakeet::Decoder::TDT, true);
        if (batch.size() != 1 || batch[0].token_ids != r.token_ids) return 4;
        parakeet::TranscribeOptions o;
        o.boost_phrases = {"abc"};
        try {
            t.transcribe(std::string(argv[3]), o);
            return 3;
        } catch (const std::runtime_error &) {
            std::cout << "BOOST_THROWS\n";
        }
    } catch (const std::exception &e) {
        std::fprintf(stderr, "exception: %s\n", e.what());
        return 1;
    }
    return 0;
}
