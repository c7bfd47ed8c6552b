// tests/golden/ref_rnnt.cpp -- TEST INFRASTRUCTURE: the reference's RNN-T model behind a small C-ABI.
//
// Built by make_golden_rnnt.py against the reference objects that oracle/Makefile compiles (oracle/_ref/obj),
// into oracle/_ref/libpkref_rnnt.so, and used only to write tests/golden/golden_rnnt_v1*.npz.  Every entry
// point only *calls* reference functions:
//   ParakeetRNNT + load_state_dict                      src/rnnt.cpp:48-52 (keys encoder_., prediction_., joint_.)
//   make_rnnt_600m_config                               include/parakeet/config.hpp:118-135
//   preprocess_audio                                    src/audio.cpp:100-158
//   FastConformerEncoder::forward                       src/encoder.cpp:253-271
//   rnnt_greedy_decode(_with_timestamps)                src/rnnt.cpp:56-177
//   Tokenizer::decode / group_timestamps                src/vocab.cpp, src/timestamp.cpp

#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include <axiom/axiom.hpp>
#include <axiom/io/safetensors.hpp>

#include "parakeet/audio.hpp"
#include "parakeet/config.hpp"
#include "parakeet/encoder.hpp"
#include "parakeet/rnnt.hpp"
#include "parakeet/timestamp.hpp"
#include "parakeet/vocab.hpp"

using namespace parakeet;
using axiom::Shape;
using axiom::Tensor;

namespace {

struct RnntModel {
    RNNTConfig cfg;
    std::unique_ptr<ParakeetRNNT> m;
    std::map<std::string, Tensor> weights;
    Tokenizer tok;
    int blank() const { return cfg.joint.vocab_size - 1; }
};

thread_local std::string g_err;

void copy_out(const Tensor &t, float *dst) {
    auto c = t.cpu().ascontiguousarray();
    std::memcpy(dst, c.typed_data<float>(), c.size() * sizeof(float));
}

}  // namespace

extern "C" {

const char *pkrnnt_last_error() { return g_err.c_str(); }

// preset 2: make_rnnt_600m_config (dims ignored); otherwise the rnnt-600m config with the given dimensions
// (test-only tiny shapes).  dims = {mel, sub_ch, d, layers, heads, ff, vocab, pred_hidden, lstm_layers, joint_hidden}.
void *pkrnnt_load(const char *weights_path, const char *vocab_path, int preset, const int *dims) {
    try {
        auto m = std::make_unique<RnntModel>();
        m->weights = axiom::io::safetensors::load(weights_path);
        auto &c = m->cfg;
        c = make_rnnt_600m_config();
        if (preset != 2) {
            c.encoder.mel_bins = dims[0];
            c.encoder.subsampling_channels = dims[1];
            c.encoder.hidden_size = dims[2];
            c.encoder.num_layers = dims[3];
            c.encoder.num_heads = dims[4];
            c.encoder.ffn_intermediate = dims[5];
            c.prediction.vocab_size = dims[6];
            c.prediction.pred_hidden = dims[7];
            c.prediction.num_lstm_layers = dims[8];
            c.joint.encoder_hidden = dims[2];
            c.joint.pred_hidden = dims[7];
            c.joint.joint_hidden = dims[9];
            c.joint.vocab_size = dims[6];
        }
        m->m = std::make_unique<ParakeetRNNT>(c);
        m->m->load_state_dict(m->weights, "", false);
        if (vocab_path && vocab_path[0]) m->tok.load(vocab_path);
        return m.release();
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void pkrnnt_free(void *h) { delete static_cast<RnntModel *>(h); }

// PCM -> normalised log-mel (n_frames, mel) -> encoder output (T', d).  mel_out holds (1 + n/160) * mel floats,
// enc_out T' * d.  Returns T' or -1.
int pkrnnt_encode_pcm(void *h, const float *pcm, int64_t n, float *mel_out, float *enc_out) {
    try {
        auto *m = static_cast<RnntModel *>(h);
        AudioConfig acfg;
        acfg.n_mels = m->cfg.encoder.mel_bins;
        auto wav = Tensor::from_data(pcm, Shape{(size_t)n}, true);
        auto f = preprocess_audio(wav, acfg).ascontiguousarray();
        if (mel_out) copy_out(f, mel_out);
        auto y = m->m->encoder()(f);
        copy_out(y, enc_out);
        return (int)y.shape()[1];
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

// enc (T, d) -> rnnt_greedy_decode_with_timestamps; rnnt_greedy_decode runs too and must give the same ids
// (else -2).  Returns the token count (at most cap written) or -1.
int pkrnnt_greedy(void *h, const float *enc, int T, int d, int max_symbols, int cap, int *ids, int *start, int *end,
                  float *conf) {
    try {
        auto *m = static_cast<RnntModel *>(h);
        auto e = Tensor::from_data(enc, Shape{1, (size_t)T, (size_t)d}, true);
        auto r = rnnt_greedy_decode_with_timestamps(*m->m, e, m->blank(), max_symbols);
        auto plain = rnnt_greedy_decode(*m->m, e, m->blank(), max_symbols);
        const int n = (int)r[0].size();
        if (plain[0].size() != r[0].size()) {
            g_err = "rnnt_greedy_decode and rnnt_greedy_decode_with_timestamps differ in length";
            return -2;
        }
        for (int i = 0; i < n; ++i) {
            if (plain[0][i] != r[0][i].token_id) {
                g_err = "rnnt_greedy_decode and rnnt_greedy_decode_with_timestamps differ at token " + std::to_string(i);
                return -2;
            }
            if (i < cap) {
                ids[i] = r[0][i].token_id;
                start[i] = r[0][i].start_frame;
                end[i] = r[0][i].end_frame;
                conf[i] = r[0][i].confidence;
            }
        }
        return n;
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

// Tokenizer::decode -> UTF-8 text in buf (NUL-terminated); returns the full length.
int pkrnnt_detok(void *h, const int *ids, int n, char *buf, int cap) {
    try {
        auto *m = static_cast<RnntModel *>(h);
        auto s = m->tok.decode(std::vector<int>(ids, ids + n));
        int k = (int)std::min<size_t>(s.size(), (size_t)cap - 1);
        std::memcpy(buf, s.data(), k);
        buf[k] = 0;
        return (int)s.size();
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

// group_timestamps(Words): words '\n'-separated into buf; returns the number of words.
int pkrnnt_group_words(void *h, const int *ids, const int *start, const int *end, const float *conf, int n, char *buf,
                       int cap, float *w_start, float *w_end, float *w_conf) {
    try {
        auto *m = static_cast<RnntModel *>(h);
        std::vector<TimestampedToken> toks(n);
        for (int i = 0; i < n; ++i) toks[i] = {ids[i], start[i], end[i], conf[i]};
        auto words = group_timestamps(toks, m->tok.pieces());
        std::string s;
        for (size_t i = 0; i < words.size(); ++i) {
            s += words[i].word;
            s += '\n';
            w_start[i] = words[i].start;
            w_end[i] = words[i].end;
            w_conf[i] = words[i].confidence;
        }
        int k = (int)std::min<size_t>(s.size(), (size_t)cap - 1);
        std::memcpy(buf, s.data(), k);
        buf[k] = 0;
        return (int)words.size();
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

}  // extern "C"
