// tests/cpp_boost_rows_check.cpp -- the per-request boosting overloads of the C++ drop-in end to end on the device:
// Transcriber::transcribe_batch with one TranscribeOptions per utterance, and StreamingTranscriber::set_boost_phrases.
// Built and run by tests/test_boost_cpp.py; prints token ids for comparison with the ctypes binding.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>

#include "parakeet/transcribe.hpp"

static std::vector<float> read_f32(const char *path) {
    std::ifstream f(path, std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    const float *p = reinterpret_cast<const float *>(raw.data());
    return std::vector<float>(p, p + raw.size() / sizeof(float));
}
static void print(const char *tag, const std::vector<parakeet::TimestampedToken> &toks, size_t from = 0) {
    std::cout << tag;
    for (size_t i = from; i < toks.size(); ++i) std::cout << " " << toks[i].token_id << ":" << toks[i].start_frame << ":" << toks[i].end_frame;
    std::cout << "\n";
}

int main(int argc, char **argv) {
    if (argc < 10) return 2;      // weights vocab a.f32 b.f32 phraseA phraseB  stream_weights stream.f32 chunk,chunk,...
    try {
        parakeet::TDTCTCConfig cfg = parakeet::make_110m_config();      // the tiny test shape (oracle.make_tiny_config)
        cfg.encoder.subsampling_channels = 64; cfg.encoder.hidden_size = 128; cfg.encoder.num_layers = 2;
        cfg.encoder.num_heads = 2; cfg.encoder.ffn_intermediate = 256;
        cfg.prediction.vocab_size = 33; cfg.prediction.pred_hidden = 64; cfg.prediction.num_lstm_layers = 1;
        cfg.joint.encoder_hidden = 128; cfg.joint.pred_hidden = 64; cfg.joint.joint_hidden = 64; cfg.joint.vocab_size = 33;
        cfg.ctc_vocab_size = 33;
        parakeet::Transcriber t(argv[1], argv[2], cfg, 0, 4, 64000);
        const std::vector<std::vector<float>> utts = {read_f32(argv[3]), read_f32(argv[4]), read_f32(argv[3])};
        for (auto dec : {parakeet::Decoder::CTC, parakeet::Decoder::TDT}) {
            std::vector<parakeet::TranscribeOptions> o(3);
            for (auto &x : o) { x.decoder = dec; x.timestamps = true; }
            o[0].boost_phrases = {argv[5]}; o[0].boost_score = 6.0f;
            o[2].boost_phrases = {argv[6], argv[5]}; o[2].boost_score = 9.0f;
            const auto r = t.transcribe_batch(utts, o);
            for (auto &x : r) print("ROW", x.timestamped_tokens);
            for (auto &x : t.transcribe_batch(utts, dec, true)) print("PLAIN", x.timestamped_tokens);      // the lists are gone again
        }
        try {
            t.transcribe_batch(utts, std::vector<parakeet::TranscribeOptions>(2));
            return 3;
        } catch (const std::invalid_argument &e) {
            std::cout << "ERR " << e.what() << "\n";
        }
        // a stream with hot words: the tiny streaming shape (oracle.make_tiny_stream_config)
        parakeet::EOUConfig sc = parakeet::make_eou_120m_config();
        sc.encoder.subsampling_channels = 64; sc.encoder.hidden_size = 128; sc.encoder.num_layers = 2; sc.encoder.num_heads = 2;
        sc.encoder.ffn_intermediate = 256; sc.encoder.att_context_left = 12; sc.encoder.att_context_right = 1;
        sc.prediction.vocab_size = 33; sc.prediction.pred_hidden = 64; sc.prediction.num_lstm_layers = 1;
        sc.joint.encoder_hidden = 128; sc.joint.pred_hidden = 64; sc.joint.joint_hidden = 64; sc.joint.vocab_size = 33;
        parakeet::StreamingTranscriber st(argv[7], argv[2], sc);
        const auto pcm = read_f32(argv[8]);
        for (int pass = 0; pass < 2; ++pass) {
            if (pass == 1) { st.reset(); st.set_boost_phrases({argv[5], argv[6]}, 25.0f); }
            size_t pos = 0, emitted = 0;
            for (char *p = argv[9]; *p;) {
                const long n = std::strtol(p, &p, 10);
                if (*p == ',') ++p;
                st.transcribe_chunk(pcm.data() + pos, (size_t)n);
                pos += (size_t)n;
                print(pass ? "SBOOST" : "SPLAIN", st.get_timestamped_tokens(), emitted);
                emitted = st.get_timestamped_tokens().size();
            }
        }
        parakeet::StreamingBatch sb(argv[7], argv[2], 2, sc);
        try {
            sb.set_boost(2, {argv[5]});
            return 4;
        } catch (const std::out_of_range &e) {
            std::cout << "ERR " << e.what() << "\n";
        }
    } catch (const std::exception &e) {
        std::fprintf(stderr, "exception: %s\n", e.what());
        return 1;
    }
    return 0;
}
