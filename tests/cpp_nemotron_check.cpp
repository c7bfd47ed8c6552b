// tests/cpp_nemotron_check.cpp -- the C++ drop-in's NemotronTranscriber (reference nemotron.hpp:79-132 usage) and
// StreamingBatch(NemotronConfig) on the tiny Nemotron test shape: feed a raw fp32 PCM file chunk by chunk through each
// transcribe_chunk overload, print the tokens every chunk produced, the text, the callback count and the state after
// reset; then three streams in one batch.  Built and run by tests/test_nemotron.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>

#include "parakeet/transcribe.hpp"

namespace {

parakeet::NemotronConfig tiny_config() {
    parakeet::NemotronConfig cfg = parakeet::make_nemotron_600m_config(0);
    // the tiny Nemotron test shape (tests/nemotron_oracle.py make_tiny_nemotron_config): head_dim 128, two LSTM layers
    cfg.encoder.subsampling_channels = 64; cfg.encoder.hidden_size = 256; cfg.encoder.num_layers = 2; cfg.encoder.num_heads = 2;
    cfg.encoder.ffn_intermediate = 512; cfg.encoder.att_context_left = 12;
    cfg.prediction.vocab_size = 33; cfg.prediction.pred_hidden = 64; cfg.prediction.num_lstm_layers = 2;
    cfg.joint.encoder_hidden = 256; cfg.joint.pred_hidden = 64; cfg.joint.joint_hidden = 64; cfg.joint.vocab_size = 33;
    return cfg;
}

void print_new(const char *tag, const std::vector<parakeet::TimestampedToken> &all, size_t &emitted) {
    std::cout << tag;
    for (; emitted < all.size(); ++emitted) std::cout << " " << all[emitted].token_id << ":" << all[emitted].start_frame << ":" << all[emitted].end_frame;
    std::cout << "\n";
}

}  // namespace

int main(int argc, char **argv) {
    if (argc < 5) return 2;      // weights vocab pcm.f32 chunk,chunk,...
    try {
        std::ifstream f(argv[3], std::ios::binary);
        std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        const float *pcm = reinterpret_cast<const float *>(raw.data());
        std::vector<size_t> sched;
        for (char *p = argv[4]; *p;) {
            sched.push_back((size_t)std::strtol(p, &p, 10));
            if (*p == ',') ++p;
        }
        const auto cfg = tiny_config();
        parakeet::NemotronTranscriber t(argv[1], argv[2], cfg);
        t.to_gpu();
        int n_cb = 0;
        t.set_partial_callback([&](const std::string &) { ++n_cb; });
        for (int mode = 0; mode < 2; ++mode) {          // const float* and std::vector<float>
            n_cb = 0;
            size_t pos = 0, emitted = 0;
            for (size_t n : sched) {
                if (mode == 0) t.transcribe_chunk(pcm + pos, n);
                else t.transcribe_chunk(std::vector<float>(pcm + pos, pcm + pos + n));
                pos += n;
                print_new(mode == 0 ? "CHUNK_F32" : "CHUNK_VEC", t.get_timestamped_tokens(), emitted);
            }
            std::cout << "TEXT " << t.get_text() << "\nCALLBACKS " << n_cb << "\n";
            t.reset();
            std::cout << "AFTER_RESET " << t.get_timestamped_tokens().size() << "\n";
        }
        // int16 PCM: the overload divides by 32768 (nemotron.hpp:104-110); the same samples as floats give the same tokens
        size_t total = 0;
        for (size_t n : sched) total += n;
        std::vector<int16_t> q(total);
        std::vector<float> dq(total);
        for (size_t i = 0; i < total; ++i) {
            const float v = std::fmax(-1.f, std::fmin(pcm[i], 32767.f / 32768.f));
            q[i] = (int16_t)std::lrintf(v * 32768.f);
            dq[i] = (float)q[i] / 32768.0f;
        }
        std::vector<int> a, b;
        size_t pos = 0;
        for (size_t n : sched) { t.transcribe_chunk(q.data() + pos, n); pos += n; }
        for (const auto &x : t.get_timestamped_tokens()) a.push_back(x.token_id * 100000 + x.start_frame * 100 + x.end_frame);
        t.reset();
        pos = 0;
        for (size_t n : sched) { t.transcribe_chunk(dq.data() + pos, n); pos += n; }
        for (const auto &x : t.get_timestamped_tokens()) b.push_back(x.token_id * 100000 + x.start_frame * 100 + x.end_frame);
        std::cout << "I16 " << (a == b ? 1 : 0) << " " << a.size() << "\n";
        // StreamingBatch with a NemotronConfig: stream 0 the file, stream 1 the same one step late, stream 2 silent
        parakeet::StreamingBatch batch(argv[1], argv[2], 3, cfg);
        std::vector<size_t> cut(1, 0);
        for (size_t n : sched) cut.push_back(cut.back() + n);
        for (size_t step = 0; step <= sched.size(); ++step) {
            std::vector<std::vector<float>> chunks(3);
            if (step < sched.size()) chunks[0].assign(pcm + cut[step], pcm + cut[step + 1]);
            if (step >= 1) chunks[1].assign(pcm + cut[step - 1], pcm + cut[step]);
            batch.transcribe_chunks(chunks);
        }
        for (int s = 0; s < 3; ++s) {
            size_t e = 0;
            print_new(("BATCH" + std::to_string(s)).c_str(), batch.get_timestamped_tokens(s), e);
        }
        std::cout << "BATCH_TEXT0 " << batch.get_text(0) << "\n";
    } catch (const std::exception &e) {
        std::fprintf(stderr, "exception: %s\n", e.what());
        return 1;
    }
    return 0;
}
