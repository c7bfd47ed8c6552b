// lm.h -- the word n-gram language model behind pk_lm (lm.cpp): the parsed ARPA file, its host scoring (which the
// device scoring in ctc_beam.cu restates), and the open-addressing tables that pk_set_ctc_beam copies to the device.
#pragma once
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/parakeet_b200.h"

#ifdef __CUDACC__
#define PK_LM_HD __host__ __device__ __forceinline__
#else
#define PK_LM_HD inline
#endif

namespace pk {

// (shared by the host tables and the device lookups of ctc_beam.cu)
constexpr uint64_t kFnvBasis = 14695981039346656037ull, kFnvPrime = 1099511628211ull;
PK_LM_HD uint64_t fnv1a(uint64_t h, const uint8_t *p, size_t n) {
    for (size_t i = 0; i < n; ++i) h = (h ^ p[i]) * kFnvPrime;
    return h;
}
PK_LM_HD uint64_t lm_ngram_key(int32_t ctx, int32_t wid) { return ((uint64_t)(uint32_t)(ctx + 1) << 32) | (uint32_t)wid; }
// slot of a key in a table of mask + 1 (a power of two) slots; probing is linear from there
PK_LM_HD uint32_t lm_slot(uint64_t key, uint32_t mask) {
    key ^= key >> 33;
    key *= 0xff51afd7ed558ccdull;
    key ^= key >> 33;
    return (uint32_t)key & mask;
}

// The pieces of a vocabulary (text.cpp); nullptr for a null vocabulary.
const std::vector<std::string> *vocab_pieces(const pk_vocab *v);

// Host tables in the device layout of DeviceLM (kernels.h).
struct LmTables {
    std::vector<unsigned long long> word_key, ng_key;
    std::vector<int32_t> word_id, ng_val, suffix, order;
    std::vector<double> prob, backoff;
    uint32_t word_mask = 0, ng_mask = 0;
};

}  // namespace pk

struct pk_lm {
    uint64_t serial = 0;                                 // unique per pk_lm_load in this process
    int32_t max_order = 0;
    std::vector<int64_t> counts;                         // [order] n-grams per order (counts[0] unused)
    std::vector<std::string> words;                      // word id -> bytes
    std::unordered_map<std::string, int32_t> word_ids;
    // entry 0 = the empty context; every other entry is one n-gram
    std::vector<double> prob, backoff;
    std::vector<int32_t> suffix, order;
    std::unordered_map<uint64_t, int32_t> next;         // lm_ngram_key(context entry, word) -> entry
    int32_t start = 0, unk = 0, eos = -1;
    pk::LmTables tables;

    int32_t find(int32_t ctx, int32_t wid) const {
        auto it = next.find(pk::lm_ngram_key(ctx, wid));
        return it == next.end() ? -1 : it->second;
    }
    int32_t word(const std::string &w) const {
        auto it = word_ids.find(w);
        return it == word_ids.end() ? unk : it->second;
    }
    // log10 p(wid | state) by back-off; moves the state on
    double score(int32_t &state, int32_t wid) const {
        double acc = 0.0;
        int32_t ctx = state;
        for (;;) {
            const int32_t e = find(ctx, wid);
            if (e >= 0) {
                state = order[e] == max_order ? suffix[e] : e;
                return acc + prob[e];
            }
            acc += backoff[ctx];
            ctx = suffix[ctx];
        }
    }
};
