// tests/cpp_align_check.cpp -- Transcriber::align of the C++ drop-in on the device.  Built and run by tests/test_ctc_align.py;
// prints one line per text (aligned, text, id:start:end per token, words, score, log-likelihood) for comparison with the
// ctypes binding, then whether align_batch gives the same results as align one by one.
#include <cstdio>
#include <iostream>

#include "parakeet/transcribe.hpp"

static std::string line(const parakeet::AlignResult &r) {
    std::string s = (r.aligned ? "1\t" : "0\t") + r.text + "\t";
    for (size_t i = 0; i < r.timestamped_tokens.size(); ++i) {
        const auto &t = r.timestamped_tokens[i];
        s += (i ? " " : "") + std::to_string(t.token_id) + ":" + std::to_string(t.start_frame) + ":" + std::to_string(t.end_frame);
    }
    s += "\t";
    for (size_t i = 0; i < r.word_timestamps.size(); ++i) s += (i ? " " : "") + r.word_timestamps[i].word;
    char num[80];
    std::snprintf(num, sizeof(num), "\t%.17g\t%.17g", r.log_prob, r.ctc_log_likelihood);
    return s + num;
}

int main(int argc, char **argv) {
    if (argc < 5) return 2;       // weights vocab clip.wav text...
    try {
        parakeet::TDTCTCConfig cfg = parakeet::make_110m_config();      // the tiny test shape (oracle.make_tiny_config)
        cfg.encoder.subsampling_channels = 64; cfg.encoder.hidden_size = 128; cfg.encoder.num_layers = 2;
        cfg.encoder.num_heads = 2; cfg.encoder.ffn_intermediate = 256;
        cfg.prediction.vocab_size = 33; cfg.prediction.pred_hidden = 64; cfg.prediction.num_lstm_layers = 1;
        cfg.joint.encoder_hidden = 128; cfg.joint.pred_hidden = 64; cfg.joint.joint_hidden = 64; cfg.joint.vocab_size = 33;
        cfg.ctc_vocab_size = 33;
        parakeet::Transcriber t(argv[1], argv[2], cfg, 0, 4, 64000);
        std::vector<std::string> texts(argv + 4, argv + argc), lines;
        for (const auto &text : texts) lines.push_back(line(t.align(argv[3], text)));
        for (const auto &l : lines) std::cout << l << "\n";
        const std::vector<float> clip = parakeet::read_audio(argv[3]);
        auto batch = t.align_batch(std::vector<std::vector<float>>(texts.size(), clip), texts);
        bool same = batch.size() == texts.size();
        for (size_t i = 0; same && i < batch.size(); ++i) same = line(batch[i]) == lines[i];
        std::cout << "batch " << (same ? "ok" : "differs") << "\n";
    } catch (const std::exception &ex) {
        std::cerr << ex.what() << "\n";
        return 1;
    }
    return 0;
}
