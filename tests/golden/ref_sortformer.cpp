// tests/golden/ref_sortformer.cpp -- TEST INFRASTRUCTURE: a C-ABI around the UNMODIFIED reference's Sortformer diarization
// model (src/sortformer.cpp, src/transformer.cpp), linked by make_golden_sortformer.py against the reference objects of
// oracle/Makefile into oracle/_ref/libpkref_sortformer.so.  One call = the reference CLI's `sortformer` mode (main.cpp:500-530)
// on one utterance: preprocess_audio with n_mels = nest_encoder.mel_bins and normalize = false, then Sortformer::forward
// and Sortformer::diarize, with the intermediate tensors copied out.
//
// Every module is loaded with strict = true, so a key the reference registers but the checkpoint lacks is an error here
// (the reference's CLI loads with strict = false and would silently keep it uninitialised).  The NEST encoder output and the
// transformer output come from a stand-alone StreamingFastConformerEncoder / Linear / TransformerEncoder loaded from the same
// state dict under "nest_encoder_." / "projection_." / "transformer_." (Module::load_state_dict, axiom module.cpp:24-38): the
// same modules, weights and forward calls that Sortformer::forward makes (sortformer.cpp:50-68).  Only golden generators
// load this library.
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
    std::unique_ptr<Linear> proj;
    std::unique_ptr<TransformerEncoder> trans;
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

const char *pksf_last_error() { return g_err.c_str(); }

// make_sortformer_117m_config() with overrides; dims <= 0 keep the preset's values
// dims = mel, sub_channels, d, layers, heads, ff, t_hidden, t_layers, t_heads, t_ff, max_speakers
void *pksf_new(const char *weights_path, const int32_t *dims) {
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
        s->weights = axiom::io::safetensors::load(weights_path);
        s->model = std::make_unique<Sortformer>(c);
        s->model->load_state_dict(s->weights, "", true);
        s->enc = std::make_unique<StreamingFastConformerEncoder>(c.nest_encoder);
        s->enc->load_state_dict(s->weights, "nest_encoder_.", true);
        s->proj = std::make_unique<Linear>(true);
        s->proj->load_state_dict(s->weights, "projection_.", true);
        s->trans = std::make_unique<TransformerEncoder>(c.transformer);
        s->trans->load_state_dict(s->weights, "transformer_.", true);
        return s.release();
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void pksf_free(void *h) { delete static_cast<SfModel *>(h); }

// feats [n_frames][mel], enc [T'][d], trans [T'][t_hidden], probs [T'][S]; segments (speaker, start s, end s) as diarize()
// returns them.  Returns 0, or -1 with pksf_last_error().
int pksf_run(void *h, const float *pcm, int n, float *feats, int cap_f, int *nf, float *enc, float *trans, float *probs, int cap_t, int *nt,
             int32_t *spk, float *seg_start, float *seg_end, int cap_s, int *ns) {
    try {
        auto *s = static_cast<SfModel *>(h);
        const SortformerConfig &c = s->cfg;
        axiom::graph::EagerModeScope eager;
        Tensor wav = Tensor::from_data(pcm, Shape{(size_t)n}, true);
        AudioConfig ac;
        ac.n_mels = c.nest_encoder.mel_bins;
        ac.normalize = false;                           // main.cpp:514-517
        Tensor f = preprocess_audio(wav, ac);           // (1, frames, mel)
        if (copy_out(f, feats, cap_f, c.nest_encoder.mel_bins, nf)) throw std::runtime_error("feats capacity");
        Tensor e = (*s->enc)(f);
        int r = 0;
        if (copy_out(e, enc, cap_t, c.nest_encoder.hidden_size, &r)) throw std::runtime_error("enc capacity");
        Tensor t = (*s->trans)((*s->proj)(e));
        if (copy_out(t, trans, cap_t, c.transformer.hidden_size, &r)) throw std::runtime_error("trans capacity");
        Tensor p = s->model->forward(f);
        if (copy_out(p, probs, cap_t, c.max_speakers, nt)) throw std::runtime_error("probs capacity");
        auto segs = s->model->diarize(f);
        if ((int)segs.size() > cap_s) throw std::runtime_error("segment capacity");
        for (size_t i = 0; i < segs.size(); ++i) {
            spk[i] = segs[i].speaker_id;
            seg_start[i] = segs[i].start;
            seg_end[i] = segs[i].end;
        }
        *ns = (int)segs.size();
        return 0;
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

}  // extern "C"
