// Host-only part of the per-utterance boosting overloads of the C++ shim (include/parakeet/transcribe.hpp): the argument
// checking of transcribe_batch(utts, options) and the packing of the phrase lists into the layout of pk_set_boost_rows,
// exercised WITHOUT a device (tests/test_boost_cpp.py builds and runs this on the CPU).
#include <cstdio>
#include <string>
#include <vector>

#include <parakeet/transcribe.hpp>

template <class F>
static const char *thrown(F f) {
    try {
        f();
    } catch (const std::invalid_argument &) {
        return "invalid_argument";
    } catch (const std::runtime_error &) {
        return "runtime_error";
    }
    return "none";
}

int main(int argc, char **argv) {
    if (argc < 4) return 2;      // vocab phraseA phraseB
    using namespace parakeet;
    Tokenizer tok;
    tok.load(argv[1]);
    std::vector<TranscribeOptions> o(3);
    o[0].boost_phrases = {argv[2], argv[3]};
    o[0].boost_score = 4.0f;
    o[2].boost_phrases = {argv[3], ""};
    o[2].boost_score = 7.5f;
    std::printf("ok %s\n", thrown([&] { detail::check_batch_options(o, 3, false); }));
    std::printf("count %s\n", thrown([&] { detail::check_batch_options(o, 2, false); }));
    std::printf("rnnt %s\n", thrown([&] { detail::check_batch_options(o, 3, true); }));
    std::printf("rnnt_plain %s\n", thrown([&] { detail::check_batch_options(std::vector<TranscribeOptions>(2), 2, true); }));
    auto d = o;
    d[1].decoder = Decoder::CTC;
    std::printf("decoder %s\n", thrown([&] { detail::check_batch_options(d, 3, false); }));
    auto t = o;
    t[2].timestamps = true;
    std::printf("timestamps %s\n", thrown([&] { detail::check_batch_options(t, 3, false); }));
    std::printf("empty %s\n", thrown([&] { detail::check_batch_options({}, 0, false); }));
    const auto r = detail::pack_boost_rows(o, 0, 3, tok);
    std::printf("ids");
    for (int v : r.ids) std::printf(" %d", v);
    std::printf("\noff");
    for (int v : r.off) std::printf(" %d", v);
    std::printf("\nrow");
    for (int v : r.row) std::printf(" %d", v);
    std::printf("\nscore");
    for (float v : r.score) std::printf(" %g", v);
    std::printf("\nany %d %d\n", (int)r.any, (int)detail::pack_boost_rows(o, 1, 1, tok).any);
    return 0;
}
