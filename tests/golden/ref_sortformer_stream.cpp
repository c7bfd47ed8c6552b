// tests/golden/ref_sortformer_stream.cpp -- TEST INFRASTRUCTURE: a C-ABI around the UNMODIFIED reference's streaming
// Sortformer diarization (Sortformer::diarize_chunk, AOSCCache; src/sortformer.cpp), linked by make_golden_sortformer_stream.py
// against the reference objects of oracle/Makefile into oracle/_ref/libpkref_sortformer_stream.so.  One stream = one
// EncoderCache + one AOSCCache; one chunk call = preprocess_audio(chunk, {n_mels = mel_bins, normalize = false}) (as
// diarize.cpp:82-85 makes a chunk's features) and Sortformer::diarize_chunk.
//
// Every module is loaded with strict = true.  The encoder rows come from a stand-alone StreamingFastConformerEncoder loaded
// from the same state dict under "nest_encoder_." and run on its own EncoderCache with the same chunks: the same module,
// weights and forward_chunk calls that diarize_chunk makes (sortformer.cpp:128).  The speaker activities come from a
// stand-alone Linear / TransformerEncoder / Linear x 2 head on those rows (sortformer.cpp:134-142).  Only golden
// generators load this library.
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
#include "parakeet/sortformer.hpp"

using namespace parakeet;
using axiom::Shape;
using axiom::Tensor;

namespace {
struct SfModel {
    SortformerConfig cfg;
    std::map<std::string, Tensor> weights;
    std::unique_ptr<Sortformer> model;
    std::unique_ptr<StreamingFastConformerEncoder> enc;
    std::unique_ptr<Linear> proj, first_hidden, output_proj;
    std::unique_ptr<TransformerEncoder> trans;
};
struct SfStream {
    EncoderCache cache, tap_cache;
    std::unique_ptr<AOSCCache> aosc;
};
thread_local std::string g_err;

int copy_out(const Tensor &t, float *dst, int cap_rows, int cols, int *rows) {
    auto c = t.cpu().ascontiguousarray();
    const size_t n = c.size();
    const int r = (int)(n / (size_t)cols);
    if (r > cap_rows) return -1;
    std::memcpy(dst, c.typed_data<float>(), n * sizeof(float));
    *rows = r;
    return 0;
}
}  // namespace

extern "C" {

const char *pkss_last_error() { return g_err.c_str(); }

// make_sortformer_117m_config() with overrides; dims <= 0 keep the preset's values
// dims = mel, sub_channels, d, layers, heads, ff, t_hidden, t_layers, t_heads, t_ff, max_speakers, att_context_left
void *pkss_new(const char *weights_path, const int32_t *dims) {
    try {
        auto s = std::make_unique<SfModel>();
        SortformerConfig &c = s->cfg;
        c = make_sortformer_117m_config();
        if (dims[0] > 0) c.nest_encoder.mel_bins = dims[0];
        if (dims[1] > 0) c.nest_encoder.subsampling_channels = dims[1];
        if (dims[2] > 0) { c.nest_encoder.hidden_size = dims[2]; c.encoder_hidden = dims[2]; }
        if (dims[3] > 0) c.nest_encoder.num_layers = dims[3];
        if (dims[4] > 0) c.nest_encoder.num_heads = dims[4];
        if (dims[5] > 0) c.nest_encoder.ffn_intermediate = dims[5];
        if (dims[6] > 0) { c.transformer_hidden = dims[6]; c.transformer.hidden_size = dims[6]; }
        if (dims[7] > 0) c.transformer.num_layers = dims[7];
        if (dims[8] > 0) c.transformer.num_heads = dims[8];
        if (dims[9] > 0) c.transformer.ffn_intermediate = dims[9];
        if (dims[10] > 0) c.max_speakers = dims[10];
        if (dims[11] > 0) c.nest_encoder.att_context_left = dims[11];
        s->weights = axiom::io::safetensors::load(weights_path);
        s->model = std::make_unique<Sortformer>(c);
        s->model->load_state_dict(s->weights, "", true);
        s->enc = std::make_unique<StreamingFastConformerEncoder>(c.nest_encoder);
        s->enc->load_state_dict(s->weights, "nest_encoder_.", true);
        s->proj = std::make_unique<Linear>(true);
        s->proj->load_state_dict(s->weights, "projection_.", true);
        s->trans = std::make_unique<TransformerEncoder>(c.transformer);
        s->trans->load_state_dict(s->weights, "transformer_.", true);
        s->first_hidden = std::make_unique<Linear>(true);
        s->first_hidden->load_state_dict(s->weights, "first_hidden_.", true);
        s->output_proj = std::make_unique<Linear>(true);
        s->output_proj->load_state_dict(s->weights, "output_proj_.", true);
        return s.release();
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void pkss_free(void *h) { delete static_cast<SfModel *>(h); }

void *pkss_stream_new(void *h) {
    auto st = new SfStream;
    st->aosc = std::make_unique<AOSCCache>(static_cast<SfModel *>(h)->cfg.max_speakers);
    return st;
}
void pkss_stream_free(void *st) { delete static_cast<SfStream *>(st); }

// One diarize_chunk on stream `st` with the chunk pcm[0..n).  enc [C][d] (stand-alone encoder on its own cache), probs
// [C][S] (ops::sigmoid of the same head as diarize_chunk; C = 0 when forward_chunk returns nothing), the segments
// diarize_chunk returns, and the AOSC order after the call.  Returns 0, or -1 with pkss_last_error().
int pkss_chunk(void *h, void *stp, const float *pcm, int n, float *enc, float *probs, int cap_t, int *nt, int32_t *spk, float *seg_start,
               float *seg_end, int cap_s, int *ns, int32_t *order, int *n_order) {
    try {
        auto *s = static_cast<SfModel *>(h);
        auto *st = static_cast<SfStream *>(stp);
        const SortformerConfig &c = s->cfg;
        axiom::graph::EagerModeScope eager;
        Tensor wav = Tensor::from_data(pcm, Shape{(size_t)n}, true);
        AudioConfig ac;
        ac.n_mels = c.nest_encoder.mel_bins;
        ac.normalize = false;
        Tensor f = preprocess_audio(wav, ac);           // (1, frames, mel)
        Tensor e = s->enc->forward_chunk(f, st->tap_cache);
        *nt = 0;
        if (e.storage() && e.shape().size() != 0) {
            int r = 0;
            if (copy_out(e, enc, cap_t, c.nest_encoder.hidden_size, &r)) throw std::runtime_error("enc capacity");
            *nt = r;
            Tensor hh = axiom::ops::relu((*s->trans)((*s->proj)(e)));
            hh = axiom::ops::relu((*s->first_hidden)(hh));
            Tensor p = axiom::ops::sigmoid((*s->output_proj)(hh));
            if (copy_out(p, probs, cap_t, c.max_speakers, &r)) throw std::runtime_error("probs capacity");
        }
        auto segs = s->model->diarize_chunk(f, st->cache, *st->aosc);
        if ((int)segs.size() > cap_s) throw std::runtime_error("segment capacity");
        for (size_t i = 0; i < segs.size(); ++i) {
            spk[i] = segs[i].speaker_id;
            seg_start[i] = segs[i].start;
            seg_end[i] = segs[i].end;
        }
        *ns = (int)segs.size();
        auto ord = st->aosc->speaker_order();
        for (size_t i = 0; i < ord.size(); ++i) order[i] = ord[i];
        *n_order = (int)ord.size();
        return 0;
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

}  // extern "C"
