// tests/golden/ref_nemotron.cpp -- TEST INFRASTRUCTURE: a C-ABI around the UNMODIFIED reference's Nemotron streaming
// model (ParakeetNemotron, src/nemotron.cpp), linked by make_golden_nemotron.py against the reference objects of
// oracle/Makefile into oracle/_ref/libpkref_nemotron.so.  One handle = one stream; a chunk call runs exactly the steps of
// NemotronTranscriber::transcribe_chunk (nemotron.cpp:25-55), with the intermediate tensors copied out:
//   StreamingAudioPreprocessor::process_chunk -> encoder().forward_chunk -> rnnt_streaming_decode_chunk
// Two differences from the transcriber, both deliberate:
//   * blank = vocab - 1 is passed to rnnt_streaming_decode_chunk.  The transcriber passes none and gets the default 1024
//     (eou.hpp:94), a real subword of the 8193-label vocabulary and past the embedding table of a small test vocabulary;
//     the engine decodes with vocab - 1 (DESIGN.md section 5).
//   * the preprocessor makes config mel_bins mels (the transcriber's is default-constructed: 80, equal for the preset).
// As in oracle/ref_harness_stream.cpp, the calls run under axiom::graph::EagerModeScope (forward_cached crashes under lazy
// evaluation on the CPU path).  Only golden generators load this library.
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include <axiom/axiom.hpp>
#include <axiom/graph/graph_registry.hpp>
#include <axiom/io/safetensors.hpp>

#include "parakeet/audio.hpp"
#include "parakeet/nemotron.hpp"

using namespace parakeet;
using axiom::Shape;
using axiom::Tensor;

namespace {
struct NemoStream {
    NemotronConfig cfg;
    std::unique_ptr<ParakeetNemotron> model;
    std::map<std::string, Tensor> weights;
    StreamingAudioPreprocessor pre;
    EncoderCache cache;
    StreamingDecodeState st;
};
thread_local std::string g_err;
}  // namespace

extern "C" {

const char *pknemo_last_error() { return g_err.c_str(); }

// make_nemotron_600m_config(latency_frames) with overrides; dims <= 0 keep the preset's values
// dims = mel, sub_channels, d, layers, heads, ff, vocab, pred_hidden, lstm_layers, joint_hidden, att_context_left
void *pknemo_new(const char *weights_path, int latency_frames, const int32_t *dims) {
    try {
        auto s = std::make_unique<NemoStream>();
        NemotronConfig &c = s->cfg;
        c = make_nemotron_600m_config(latency_frames);
        if (dims[0] > 0) c.encoder.mel_bins = dims[0];
        if (dims[1] > 0) c.encoder.subsampling_channels = dims[1];
        if (dims[2] > 0) { c.encoder.hidden_size = dims[2]; c.joint.encoder_hidden = dims[2]; }
        if (dims[3] > 0) c.encoder.num_layers = dims[3];
        if (dims[4] > 0) c.encoder.num_heads = dims[4];
        if (dims[5] > 0) c.encoder.ffn_intermediate = dims[5];
        if (dims[6] > 0) { c.prediction.vocab_size = dims[6]; c.joint.vocab_size = dims[6]; }
        if (dims[7] > 0) { c.prediction.pred_hidden = dims[7]; c.joint.pred_hidden = dims[7]; }
        if (dims[8] > 0) c.prediction.num_lstm_layers = dims[8];
        if (dims[9] > 0) c.joint.joint_hidden = dims[9];
        if (dims[10] > 0) c.encoder.att_context_left = dims[10];
        AudioConfig ac;
        ac.n_mels = c.encoder.mel_bins;
        s->pre = StreamingAudioPreprocessor(ac);
        s->weights = axiom::io::safetensors::load(weights_path);
        s->model = std::make_unique<ParakeetNemotron>(c);
        s->model->load_state_dict(s->weights, "", false);
        return s.release();
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void pknemo_free(void *h) { delete static_cast<NemoStream *>(h); }

// One chunk of PCM.  Outputs (each may be empty): log-mel frames [n_frames][mel], encoder rows [n_enc][d], new tokens
// (id, start, end) + confidences.  Returns 0, or -1 (see pknemo_last_error).
int pknemo_chunk(void *h, const float *pcm, int n, float *feats_out, int feats_cap, int *n_frames, float *enc_out, int enc_cap,
                 int *n_enc, int32_t *tok_out, float *conf_out, int tok_cap, int *n_tok) {
    auto *s = static_cast<NemoStream *>(h);
    *n_frames = *n_enc = *n_tok = 0;
    try {
        axiom::graph::EagerModeScope eager;
        auto samples = Tensor::from_data(pcm, Shape{(size_t)n}, true);
        auto feats = s->pre.process_chunk(samples);
        if (!feats.storage()) return 0;
        const int nf = (int)feats.shape()[1], nm = (int)feats.shape()[2];
        if (nf > feats_cap) { g_err = "feats capacity"; return -1; }
        *n_frames = nf;
        auto fc = feats.cpu().ascontiguousarray();
        std::memcpy(feats_out, fc.typed_data<float>(), (size_t)nf * nm * sizeof(float));
        auto enc = s->model->encoder().forward_chunk(feats, s->cache);
        if (!enc.storage() || enc.shape().size() == 0) return 0;
        const int ne = (int)enc.shape()[1], d = (int)enc.shape()[2];
        if (ne > enc_cap) { g_err = "enc capacity"; return -1; }
        *n_enc = ne;
        auto ec = enc.cpu().ascontiguousarray();
        std::memcpy(enc_out, ec.typed_data<float>(), (size_t)ne * d * sizeof(float));
        const size_t before = s->st.timestamped_tokens.size();
        rnnt_streaming_decode_chunk(s->model->prediction(), s->model->joint(), enc, s->cfg.durations, s->st,
                                    s->cfg.joint.vocab_size - 1);
        const size_t after = s->st.timestamped_tokens.size();
        if ((int)(after - before) > tok_cap) { g_err = "token capacity"; return -1; }
        for (size_t i = before; i < after; ++i) {
            const auto &t = s->st.timestamped_tokens[i];
            tok_out[3 * (i - before) + 0] = t.token_id;
            tok_out[3 * (i - before) + 1] = t.start_frame;
            tok_out[3 * (i - before) + 2] = t.end_frame;
            conf_out[i - before] = t.confidence;
        }
        *n_tok = (int)(after - before);
        return 0;
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

}  // extern "C"
