// text.cpp -- host-side text helpers behind the C-ABI (no device work).
//
// Behavioural parity targets (reference):
//   Tokenizer::load   src/vocab.cpp:10-27   "piece<TAB>score" lines; a line without a tab is
//                                            taken whole; empty lines are skipped.
//   Tokenizer::decode src/vocab.cpp:29-64   concatenate pieces, out-of-range id -> "[id]",
//                                            U+2581 -> ' ', strip exactly one leading space.
//   group_timestamps  src/timestamp.cpp:24-75 (Words mode) a piece starting with U+2581
//                                            opens a new word; word conf = min token conf;
//                                            seconds = frame * 0.08f (timestamp.hpp:31-35).
//   Tokenizer::encode src/vocab.cpp:76-117  greedy longest piece match on bytes (pk_tokenize).
//   ContextTrie + ctc_greedy_decode(_with_timestamps)_boosted  src/phrase_boost.cpp:9-176 (pk_ctc_decode_boosted).
//   resample / sinc_resample src/audio_io.cpp:101-195, :238-251 (pk_resample): same double arithmetic, bit-exact.
#include <algorithm>
#include <cstring>
#include <fstream>
#include <cmath>
#include <numeric>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/parakeet_b200.h"
#include "lm.h"

struct pk_vocab {
    std::vector<std::string> pieces;
};

namespace pk {
const std::vector<std::string> *vocab_pieces(const pk_vocab *v) { return v ? &v->pieces : nullptr; }
}  // namespace pk

namespace {
const char kMark[] = "\xe2\x96\x81";  // U+2581
bool has_mark(const std::string &s) { return s.size() >= 3 && s.compare(0, 3, kMark) == 0; }

int32_t emit(const std::string &s, char *buf, int32_t cap) {
    if (buf && cap > 0) {
        size_t k = std::min(s.size(), (size_t)cap - 1);
        memcpy(buf, s.data(), k);
        buf[k] = 0;
    }
    return (int32_t)s.size();
}
}  // namespace

extern "C" {

pk_status pk_vocab_load(const char *vocab_path, pk_vocab **out) {
    if (!vocab_path || !out) return PK_ERR_INVALID;
    std::ifstream f(vocab_path);
    if (!f) return PK_ERR_IO;
    auto *v = new pk_vocab();
    std::string line;
    while (std::getline(f, line)) {
        size_t tab = line.find('\t');
        if (tab != std::string::npos)
            v->pieces.emplace_back(line, 0, tab);
        else if (!line.empty())
            v->pieces.push_back(line);
    }
    *out = v;
    return PK_OK;
}

void pk_vocab_free(pk_vocab *v) { delete v; }

int32_t pk_vocab_size(const pk_vocab *v) { return v ? (int32_t)v->pieces.size() : 0; }

int32_t pk_vocab_max_piece_bytes(const pk_vocab *v) {
    size_t m = 16;                                  // "[id]" placeholders of out-of-range ids (vocab.cpp:57-60)
    if (v)
        for (const auto &p : v->pieces) m = std::max(m, p.size());
    return (int32_t)m;
}

int32_t pk_detokenize(const pk_vocab *v, const int32_t *ids, int32_t n, char *buf, int32_t cap) {
    if (!v) return -1;
    std::string joined;
    for (int32_t i = 0; i < n; ++i) {
        const int32_t id = ids[i];
        if (id < 0 || id >= (int32_t)v->pieces.size())
            joined += "[" + std::to_string(id) + "]";
        else
            joined += v->pieces[id];
    }
    std::string text;
    text.reserve(joined.size());
    for (size_t pos = 0; pos < joined.size();) {
        if (joined.compare(pos, 3, kMark) == 0 && pos + 3 <= joined.size()) {
            text += ' ';
            pos += 3;
        } else {
            text += joined[pos++];
        }
    }
    if (!text.empty() && text[0] == ' ') text.erase(0, 1);
    return emit(text, buf, cap);
}

int32_t pk_group_words(const pk_vocab *v, const int32_t *ids, const int32_t *start, const int32_t *end,
                       const float *conf, int32_t n, char *buf, int32_t cap, float *w_start, float *w_end,
                       float *w_conf) {
    if (!v) return -1;
    if (n <= 0) {
        emit("", buf, cap);
        return 0;
    }
    const float kFrame = 0.08f;
    std::string all, word;
    int32_t n_words = 0;
    int ws = start[0], we = end[0];
    float wc = 1.0f;
    auto flush = [&]() {
        all += word;
        all += '\n';
        w_start[n_words] = (float)ws * kFrame;
        w_end[n_words] = (float)we * kFrame;
        w_conf[n_words] = wc;
        ++n_words;
        word.clear();
    };
    for (int32_t i = 0; i < n; ++i) {
        if (ids[i] < 0 || ids[i] >= (int32_t)v->pieces.size()) continue;
        const std::string &piece = v->pieces[ids[i]];
        const bool opens = has_mark(piece);
        if (opens && !word.empty()) {
            flush();
            ws = start[i];
            wc = 1.0f;
        }
        word += opens ? piece.substr(3) : piece;
        we = end[i];
        wc = std::min(wc, conf ? conf[i] : 1.0f);
    }
    if (!word.empty()) flush();
    emit(all, buf, cap);
    return n_words;
}

int32_t pk_tokenize(const pk_vocab *v, const char *text, int32_t *ids, int32_t cap) {
    if (!v || !text || v->pieces.empty() || !text[0]) return 0;
    std::unordered_map<std::string, int32_t> table;             // later duplicates win, like operator[] in the reference
    size_t max_len = 0;
    for (size_t i = 0; i < v->pieces.size(); ++i) {
        table[v->pieces[i]] = (int32_t)i;
        max_len = std::max(max_len, v->pieces[i].size());
    }
    std::string input = kMark;
    for (const char *c = text; *c; ++c) {
        if (*c == ' ') input += kMark;
        else input += *c;
    }
    int32_t n = 0;
    size_t pos = 0;
    while (pos < input.size()) {
        size_t len = std::min(max_len, input.size() - pos);
        int32_t id = -1;
        for (; len >= 1; --len) {
            auto it = table.find(input.substr(pos, len));
            if (it != table.end()) {
                id = it->second;
                break;
            }
        }
        if (id >= 0) {
            if (ids && n < cap) ids[n] = id;
            ++n;
            pos += len;
        } else {
            ++pos;                                               // unknown byte: skipped
        }
    }
    return n;
}

namespace {
// ContextTrie (phrase_boost.cpp:9-66): node 0 = root; the active set always contains the root.
struct Trie {
    std::vector<std::unordered_map<int32_t, int32_t>> children{1};
    void insert(const int32_t *ids, int32_t n) {
        int32_t node = 0;
        for (int32_t i = 0; i < n; ++i) {
            auto it = children[node].find(ids[i]);
            if (it == children[node].end()) {
                const int32_t next = (int32_t)children.size();
                children[node][ids[i]] = next;
                children.emplace_back();
                node = next;
            } else {
                node = it->second;
            }
        }
    }
};
}  // namespace

int32_t pk_ctc_decode_boosted(const float *lp, int32_t T, int32_t V, int32_t blank, const int32_t *ph_ids,
                              const int32_t *ph_off, int32_t n_phrases, float boost, int32_t *ids, int32_t *start,
                              int32_t *end, float *conf, int32_t cap) {
    if (!lp || T < 0 || V <= 0 || n_phrases < 0 || (n_phrases > 0 && (!ph_ids || !ph_off)) || !ids || cap < 0) return -1;
    Trie trie;
    for (int32_t p = 0; p < n_phrases; ++p) trie.insert(ph_ids + ph_off[p], ph_off[p + 1] - ph_off[p]);
    std::vector<int32_t> active{0}, next;
    std::vector<uint8_t> boosted((size_t)V, 0);
    std::vector<int32_t> marked;
    int32_t n = 0, prev = -1, last = -1;                         // last = slot of the most recent token (for end frames)
    for (int32_t t = 0; t < T; ++t) {
        const float *row = lp + (size_t)t * V;
        for (int32_t m : marked) boosted[m] = 0;
        marked.clear();
        for (int32_t st : active)
            for (const auto &kv : trie.children[st])
                if (kv.first >= 0 && kv.first < V && !boosted[kv.first]) {
                    boosted[kv.first] = 1;
                    marked.push_back(kv.first);
                }
        int32_t best = 0;
        float best_val = row[0] + (boosted[0] ? boost : 0.0f);
        for (int32_t v2 = 1; v2 < V; ++v2) {                     // strict '>': the first maximum wins
            const float val = row[v2] + (boosted[v2] ? boost : 0.0f);
            if (val > best_val) {
                best_val = val;
                best = v2;
            }
        }
        if (best != prev) {
            if (prev != -1 && prev != blank && last >= 0 && end && last < cap) end[last] = t - 1;
            if (best != blank) {
                if (n < cap) {
                    ids[n] = best;
                    if (start) start[n] = t;
                    if (end) end[n] = t;
                    if (conf) conf[n] = std::exp(row[best]);     // raw (unboosted) log-prob
                }
                last = n++;
                next.assign(1, 0);                               // advance: the root plus every continued phrase
                for (int32_t st : active) {
                    auto it = trie.children[st].find(best);
                    if (it != trie.children[st].end() && std::find(next.begin(), next.end(), it->second) == next.end())
                        next.push_back(it->second);
                }
                active.swap(next);
            }
        }
        prev = best;
    }
    if (last >= 0 && end && last < cap) end[last] = T - 1;
    return n;
}

}  // extern "C"
