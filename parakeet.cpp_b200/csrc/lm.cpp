// lm.cpp -- ARPA word n-gram language models for the CTC beam search (pk_lm_*; DESIGN.md section 14).
//
// The file is read once into entries (one per n-gram, entry 0 = the empty context) linked by (context entry, word) ->
// entry, which is both the host scorer (pk_lm::score) and, flattened into open-addressing tables, the device one.
#include <atomic>
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "lm.h"

namespace pk_detail {
std::string &create_err();   // pk_last_error(NULL) (engine.cu)
}

namespace {

using pk::LmTables;

bool parse_double(const std::string &s, double *out) {
    if (s.empty()) return false;
    errno = 0;
    char *end = nullptr;
    const double v = std::strtod(s.c_str(), &end);
    if (end != s.c_str() + s.size() || errno == ERANGE || !std::isfinite(v)) return false;
    *out = v;
    return true;
}

std::vector<std::string> split_ws(const std::string &line) {
    std::vector<std::string> f;
    std::istringstream is(line);
    std::string t;
    while (is >> t) f.push_back(t);
    return f;
}

bool blank_line(const std::string &s) { return s.find_first_not_of(" \t\r") == std::string::npos; }

uint32_t pow2_mask(size_t n) {
    size_t c = 16;
    while (c < 2 * n) c <<= 1;
    return (uint32_t)(c - 1);
}

// Open-addressing tables of the device layout; false: two words share a hash (named in *msg).
bool build_tables(const pk_lm &lm, LmTables &t, std::string *msg) {
    t.word_mask = pow2_mask(lm.words.size());
    t.word_key.assign((size_t)t.word_mask + 1, 0ull);
    t.word_id.assign((size_t)t.word_mask + 1, -1);
    for (int32_t w = 0; w < (int32_t)lm.words.size(); ++w) {
        const std::string &s = lm.words[w];
        uint64_t h = pk::fnv1a(pk::kFnvBasis, reinterpret_cast<const uint8_t *>(s.data()), s.size());
        if (h == 0) h = 1;                                   // (0 marks an empty slot; a word hashing to 0 is looked up as 1)
        uint32_t i = pk::lm_slot(h, t.word_mask);
        while (t.word_key[i] != 0 && t.word_key[i] != h) i = (i + 1) & t.word_mask;
        if (t.word_key[i] == h) {
            *msg = "words \"" + lm.words[t.word_id[i]] + "\" and \"" + s + "\" have the same 64-bit FNV-1a hash";
            return false;
        }
        t.word_key[i] = h;
        t.word_id[i] = w;
    }
    t.ng_mask = pow2_mask(lm.next.size());
    t.ng_key.assign((size_t)t.ng_mask + 1, 0ull);
    t.ng_val.assign((size_t)t.ng_mask + 1, -1);
    for (const auto &kv : lm.next) {
        uint32_t i = pk::lm_slot(kv.first, t.ng_mask);
        while (t.ng_key[i] != 0) i = (i + 1) & t.ng_mask;
        t.ng_key[i] = kv.first;
        t.ng_val[i] = kv.second;
    }
    t.prob = lm.prob;
    t.backoff = lm.backoff;
    t.suffix = lm.suffix;
    t.order = lm.order;
    return true;
}

pk_status load(const char *path, pk_lm *lm, std::string *msg) {
    std::ifstream f(path);
    if (!f) {
        *msg = std::string("cannot open ") + path;
        return PK_ERR_IO;
    }
    std::string line;
    int64_t ln = 0;
    auto err = [&](const std::string &m) {
        *msg = std::string(path) + ":" + std::to_string(ln) + ": " + m;
        return PK_ERR_IO;
    };
    bool got = false;
    while (std::getline(f, line)) {
        ++ln;
        if (line.rfind("\\data\\", 0) == 0) { got = true; break; }
    }
    if (!got) return err("no \\data\\ section");
    std::vector<int64_t> counts(1, 0);
    std::string pending;                                     // the first line after the counts
    bool have_pending = false;
    while (std::getline(f, line)) {
        ++ln;
        if (blank_line(line)) {
            if (counts.size() > 1) break;
            continue;
        }
        if (line.rfind("ngram ", 0) != 0) { pending = line; have_pending = true; break; }
        const size_t eq = line.find('=');
        double k = 0, c = 0;
        if (eq == std::string::npos || !parse_double(line.substr(6, eq - 6), &k) || !parse_double(line.substr(eq + 1), &c) ||
            k != std::floor(k) || c != std::floor(c) || c < 0)
            return err("field does not parse: \"" + line + "\"");
        if ((int64_t)k != (int64_t)counts.size()) return err("ngram counts must be listed in order 1, 2, ...");
        counts.push_back((int64_t)c);
    }
    const int N = (int)counts.size() - 1;
    if (N < 1 || N > 6) return err("order " + std::to_string(N) + " (1..6 supported)");
    lm->max_order = N;
    lm->counts = counts;
    lm->prob.assign(1, 0.0);
    lm->backoff.assign(1, 0.0);
    lm->suffix.assign(1, -1);
    lm->order.assign(1, 0);
    auto next_line = [&](std::string &out) {
        if (have_pending) { out = pending; have_pending = false; return true; }
        if (!std::getline(f, out)) return false;
        ++ln;
        return true;
    };
    for (int k = 1; k <= N; ++k) {
        const std::string head = "\\" + std::to_string(k) + "-grams:";
        bool found = false;
        while (next_line(line)) {
            if (blank_line(line)) continue;
            if (line.rfind(head, 0) != 0) return err("expected " + head);
            found = true;
            break;
        }
        if (!found) return err("truncated file: " + head + " missing");
        int64_t n = 0;
        while (next_line(line)) {
            if (blank_line(line)) {
                if (n == counts[k]) break;
                continue;
            }
            if (line[0] == '\\') {
                have_pending = true;
                pending = line;
                break;
            }
            if (n == counts[k]) return err(std::to_string(k) + "-grams: more entries than the count " + std::to_string(counts[k]));
            const std::vector<std::string> fld = split_ws(line);
            double p = 0, b = 0;
            if ((fld.size() != (size_t)k + 1 && fld.size() != (size_t)k + 2) || !parse_double(fld[0], &p) ||
                (fld.size() == (size_t)k + 2 && !parse_double(fld[k + 1], &b)))
                return err("field does not parse: \"" + line + "\"");
            int32_t ctx = 0;
            for (int j = 1; j < k && ctx >= 0; ++j) {
                auto it = lm->word_ids.find(fld[j]);
                ctx = it == lm->word_ids.end() ? -1 : lm->find(ctx, it->second);
            }
            if (ctx < 0) return err("the context of \"" + line + "\" is not in the file");
            int32_t wid;
            if (k == 1) {
                if (lm->word_ids.count(fld[1])) return err("duplicate 1-gram \"" + fld[1] + "\"");
                wid = (int32_t)lm->words.size();
                lm->words.push_back(fld[1]);
                lm->word_ids.emplace(fld[1], wid);
            } else {
                auto it = lm->word_ids.find(fld[k]);
                if (it == lm->word_ids.end()) return err("word \"" + fld[k] + "\" is not a 1-gram");
                wid = it->second;
            }
            const uint64_t key = pk::lm_ngram_key(ctx, wid);
            if (lm->next.count(key)) return err("duplicate n-gram \"" + line + "\"");
            lm->next.emplace(key, (int32_t)lm->prob.size());
            lm->prob.push_back(p);
            lm->backoff.push_back(b);
            lm->order.push_back(k);
            ++n;
        }
        if (n != counts[k])
            return err(std::to_string(k) + "-grams: " + std::to_string(n) + " entries, the count says " + std::to_string(counts[k]));
    }
    got = false;
    while (next_line(line)) {
        if (blank_line(line)) continue;
        if (line.rfind("\\end\\", 0) != 0) return err("expected \\end\\");
        got = true;
        break;
    }
    if (!got) return err("truncated file: \\end\\ missing");
    if (!lm->word_ids.count("<unk>")) {
        const int32_t wid = (int32_t)lm->words.size();
        lm->words.push_back("<unk>");
        lm->word_ids.emplace("<unk>", wid);
        lm->next.emplace(pk::lm_ngram_key(0, wid), (int32_t)lm->prob.size());
        lm->prob.push_back(-10.0);
        lm->backoff.push_back(0.0);
        lm->order.push_back(1);
        ++lm->counts[1];
    }
    lm->unk = lm->word_ids.at("<unk>");
    // suffix of an entry = its longest present proper suffix; the words of each entry are recovered from the links
    std::vector<int32_t> parent(lm->prob.size(), -1), last(lm->prob.size(), -1);
    for (const auto &kv : lm->next) {
        parent[kv.second] = (int32_t)(kv.first >> 32) - 1;
        last[kv.second] = (int32_t)(kv.first & 0xffffffffu);
    }
    lm->suffix.resize(lm->prob.size(), 0);
    std::vector<int32_t> ws;
    for (int32_t e = 1; e < (int32_t)lm->prob.size(); ++e) {
        ws.clear();
        for (int32_t x = e; x > 0; x = parent[x]) ws.push_back(last[x]);   // reversed words
        int32_t suf = 0;
        for (size_t s = 1; s < ws.size(); ++s) {                           // drop the s oldest words
            int32_t x = 0;
            for (size_t j = ws.size() - s; j-- > 0 && x >= 0;) x = lm->find(x, ws[j]);
            if (x >= 0) { suf = x; break; }
        }
        lm->suffix[e] = suf;
    }
    auto bos = lm->word_ids.find("<s>");
    lm->start = 0;
    if (bos != lm->word_ids.end()) {
        const int32_t e = lm->find(0, bos->second);
        lm->start = lm->order[e] == N ? lm->suffix[e] : e;
    }
    lm->eos = lm->word("</s>");
    if (!build_tables(*lm, lm->tables, msg)) return err(*msg);
    return PK_OK;
}

}  // namespace

extern "C" {

pk_status pk_lm_load(const char *arpa_path, pk_lm **out) {
    if (!arpa_path || !out) return PK_ERR_INVALID;
    *out = nullptr;
    static std::atomic<uint64_t> next_serial{1};
    auto *lm = new pk_lm();
    lm->serial = next_serial++;
    std::string msg;
    const pk_status s = load(arpa_path, lm, &msg);
    if (s != PK_OK) {
        pk_detail::create_err() = msg;
        delete lm;
        return s;
    }
    *out = lm;
    return PK_OK;
}

void pk_lm_free(pk_lm *lm) { delete lm; }

int32_t pk_lm_order(const pk_lm *lm) { return lm ? lm->max_order : 0; }

int64_t pk_lm_count(const pk_lm *lm, int32_t order) {
    return lm && order >= 1 && order <= lm->max_order ? lm->counts[order] : -1;
}

double pk_lm_sentence_log10(const pk_lm *lm, const char *words) {
    if (!lm || !words) return NAN;
    int32_t state = lm->start;
    double acc = 0.0;
    for (const std::string &w : split_ws(words)) acc += lm->score(state, lm->word(w));
    return acc + lm->score(state, lm->eos);
}

}  // extern "C"
