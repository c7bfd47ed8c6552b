"""CTC prefix beam search with word n-gram fusion (PK_DECODER_CTC_BEAM, DESIGN.md section 14).

CPU: the float64 oracle (tests/ctc_beam_oracle.py) against brute-force enumeration, the ARPA parser (pk_lm_*) against the
oracle's independent reader, and the parser's errors.  GPU: the kernels through pk_kernel_ctc_beam against the oracle, the
LM's effect, the engine path end to end, batching and graph replay, and the rejections.  Every GPU comparison first
requires each decision of the oracle to be wider than its rounding bound, so a near tie fails loudly instead of flipping."""
from __future__ import annotations

import ctypes as C
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_beam_oracle as CB  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
PK_ERR_INVALID, PK_ERR_IO = 1, 2


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def _lm_words(pieces, rng, n):
    """LM words spelled from the vocabulary: a word-starting piece, then 0-2 continuation pieces."""
    starts = [p[1:] for p in pieces if p.startswith(CB.SP_MARK) and len(p) > 1]
    conts = [p for p in pieces if not p.startswith(CB.SP_MARK)]
    out = set()
    while len(out) < n:
        w = starts[int(rng.integers(len(starts)))] + "".join(conts[int(rng.integers(len(conts)))] for _ in range(int(rng.integers(0, 3))))
        out.add(w)
    return sorted(out)


# ------------------------------------------------------------------ CPU: the oracle and the parser
@pytest.mark.parametrize("T", [1, 2, 3, 4, 5, 6])
def test_oracle_equals_brute_force(T):
    for seed in range(4):
        rng = np.random.default_rng(100 * T + seed)
        lp = CB.make_logprobs(rng, T, 4, sigma=1.0, peak=float(rng.uniform(0, 2)))
        prefix, score, tot = CB.brute_force(lp)
        res = CB.beam_search(lp, 10 ** 6, extend_all=True, keep_all=True)
        assert res["prefix"] == prefix
        assert math.isclose(res["score"], score, rel_tol=1e-12, abs_tol=1e-12)
        # with no pruning every prefix keeps its exact probability
        for b in res["beams"]:
            assert math.isclose(CB.lse(b["pb"], b["pnb"]), tot[b["p"]], rel_tol=1e-12, abs_tol=1e-12)


def _arpa_cases(tmp_path):
    words = ["alpha", "beta", "gamma", "delta", "héllo", "日本", "straße", "x"]
    for order in (1, 2, 3, 4):
        for unk in (True, False):
            path = str(tmp_path / f"lm{order}{int(unk)}.arpa")
            CB.make_arpa(path, words, order, seed=order * 10 + unk, per_order=60, unk=unk)
            yield path, words


def test_lm_sentence_scores_match_the_python_reader(pkg, tmp_path):
    rng = np.random.default_rng(7)
    n = 0
    for path, words in _arpa_cases(tmp_path):
        ref = CB.Arpa(path)
        lm = pkg.LanguageModel(path)
        assert lm.order == ref.order
        for k in range(1, ref.order + 1):
            assert lm.count(k) == sum(1 for g in ref.prob if len(g) == k)
        for _ in range(40):
            sent = [words[int(i)] if rng.random() < 0.9 else "zzz" for i in rng.integers(0, len(words), int(rng.integers(0, 9)))]
            got = lm.sentence_log10(" ".join(sent))
            assert abs(got - ref.sentence_log10(sent)) < 1e-9, (path, sent)
            n += 1
        lm.close()
    assert n == 320


def _bad(tmp_path, name, text):
    p = str(tmp_path / name)
    with open(p, "w", encoding="utf-8") as f:
        f.write(text)
    return p


GOOD = "\\data\\\nngram 1=3\nngram 2=1\n\n\\1-grams:\n-1.0\t<s>\t-0.5\n-0.5\ta\t-0.2\n-0.7\t</s>\n\n\\2-grams:\n-0.1\t<s> a\n\n\\end\\\n"


@pytest.mark.parametrize("name,text,line", [
    ("counts", GOOD.replace("ngram 1=3", "ngram 1=4"), 10),                 # the 1-grams end early
    ("prefix", GOOD.replace("-0.1\t<s> a", "-0.1\ta a\n-0.1\tb a").replace("ngram 2=1", "ngram 2=2"), 12),
    ("truncated", GOOD[:GOOD.index("\\2-grams:")], 9),
    ("field", GOOD.replace("-0.5\ta\t-0.2", "-0.5x\ta\t-0.2"), 7),
])
def test_malformed_arpa_is_an_io_error_naming_the_line(pkg, tmp_path, name, text, line):
    L = pkg.load_library()
    h = C.c_void_p()
    p = _bad(tmp_path, name + ".arpa", text)
    assert L.pk_lm_load(p.encode(), C.byref(h)) == PK_ERR_IO
    msg = L.pk_last_error(None).decode()
    assert f"{p}:{line}:" in msg, msg
    assert L.pk_lm_load(_bad(tmp_path, "good.arpa", GOOD).encode(), C.byref(h)) == 0
    L.pk_lm_free(h)


# ------------------------------------------------------------------ GPU: the kernels against the oracle
def hook(pkg, lps, W, lm=None, vocab=None, alpha=0.5, beta=1.0, cap=None):
    """pk_kernel_ctc_beam on a list of [T][V] log-prob matrices -> (tokens per row, topk ids, bp)."""
    L = pkg.load_library()
    V = lps[0].shape[1]
    off = np.zeros(len(lps) + 1, np.int32)
    off[1:] = np.cumsum([x.shape[0] for x in lps])
    rows = int(off[-1])
    lp = np.ascontiguousarray(np.concatenate(lps) if rows else np.zeros((1, V), np.float32), np.float32)
    cap = cap or max(1, max(x.shape[0] for x in lps) + 8)
    n = len(lps)
    tok = np.zeros((n, 1 + cap), np.int32)
    st, en = np.zeros((n, cap), np.int32), np.zeros((n, cap), np.int32)
    cf = np.zeros((n, cap), np.float32)
    R = max(rows, 1)
    tid, tlp, blp, bp = np.zeros((R, W), np.int32), np.zeros((R, W), np.float32), np.zeros(R, np.float32), np.zeros((R, W), np.int32)
    gb = C.c_int64(-1)
    i32, f32 = C.c_int32, C.c_float
    s = L.pk_kernel_ctc_beam(0, n, _p(off, i32), rows, V, _p(lp, f32), W, lm.h if lm else None, vocab.h if vocab else None, alpha, beta,
                             cap, _p(tok, i32), _p(st, i32), _p(en, i32), _p(cf, f32), _p(tid, i32), _p(tlp, f32), _p(blp, f32), _p(bp, i32),
                             C.byref(gb))
    assert s == 0, f"pk_kernel_ctc_beam -> {s}"
    assert gb.value == 0, "a guard band was written"
    out = []
    for b in range(n):
        k = int(tok[b, 0])
        out.append([(int(tok[b, 1 + i]), int(st[b, i]), int(en[b, i]), float(cf[b, i])) for i in range(k)])
    return out, tid[:rows], bp[:rows]


def _check_rows(got, lps, W, **kw):
    merges, differ = 0, 0
    for g, lp in zip(got, lps):
        ref = CB.beam_search(lp, W, **kw)
        assert CB.min_margin_ratio(ref, lp.shape[0]) > 4.0, "a decision of the oracle is within 4x its rounding bound"
        assert [t[:3] for t in g] == [t[:3] for t in ref["tokens"]]
        assert np.allclose([t[3] for t in g], [t[3] for t in ref["tokens"]], rtol=1e-6, atol=0)
        merges += ref["merges"]
        differ += list(ref["prefix"]) != CB.greedy(lp)
    return merges, differ


def _batch(V, seed):
    rng = np.random.default_rng(seed)
    lps = [CB.make_logprobs(rng, T, V, sigma=float(rng.uniform(0.5, 2.0)), peak=float(rng.uniform(1.0, 5.0)))
           for T in (0, 1, 2, 126, 400, 126, 126)]
    lps[6][:, 3:V - 1] = -np.inf                            # three tokens and the blank: prefixes meet and merge
    lps[5][60:] = -np.inf                                   # every log-prob -inf past a frame: no hypothesis survives
    mask = rng.random(lps[3].shape) < 0.6                   # most tokens impossible: absent top-W entries
    mask[:, -1] = False
    lps[3][mask] = -np.inf
    return lps


@gpu
@pytest.mark.parametrize("V", [33, 1025, 8193])
@pytest.mark.parametrize("W", [1, 2, 8, 32])
def test_kernel_hook_matches_the_oracle(pkg, V, W):
    lps = _batch(V, 1000 * V + W)
    got, tid, _ = hook(pkg, lps, W)
    # the frame pass: the W best non-blank ids, ties to the lower id, -1 where fewer are finite
    flat = np.concatenate(lps)
    for r in range(0, flat.shape[0], 37):
        ids = sorted((v for v in range(V - 1) if flat[r, v] > -np.inf), key=lambda v: (-flat[r, v], v))[:W]
        assert tid[r].tolist() == ids + [-1] * (W - len(ids))
    merges, differ = _check_rows(got, lps, W)
    assert got[0] == [] and got[5] == []
    if W > 1:
        assert merges > 0 and differ > 0, "the comparison would not exercise merging or differ from greedy"


@gpu
@pytest.mark.parametrize("V,W", [(33, 8), (1025, 4), (1025, 32)])
def test_kernel_hook_with_a_language_model(pkg, synth, tmp_path, V, W):
    pieces = synth.make_vocab(V - 1, seed=V)
    vp = str(tmp_path / "v.txt")
    synth.save_vocab(vp, pieces)
    rng = np.random.default_rng(V + W)
    words = _lm_words(pieces, rng, 60)
    arpa = str(tmp_path / "lm.arpa")
    CB.make_arpa(arpa, words, 3, seed=V, per_order=300)
    lm, voc = pkg.LanguageModel(arpa), pkg.engine.Tokenizer(vp)
    lps = _batch(V, 7 * V + W + (3 if (V, W) == (1025, 32) else 0))     # (a seed whose decisions all clear the margin guard)
    for alpha, beta in ((0.5, 1.0), (1.5, -0.5)):
        got, _, _ = hook(pkg, lps, W, lm, voc, alpha, beta)
        _check_rows(got, lps, W, lm=CB.Arpa(arpa), pieces=pieces, alpha=alpha, beta=beta)
    # zero weights: the bytes of the decode without a language model
    assert hook(pkg, lps, W, lm, voc, 0.0, 0.0)[0] == hook(pkg, lps, W)[0]


@gpu
def test_language_model_changes_the_answer_for_the_right_reason(pkg, tmp_path):
    pieces = ["▁cat", "▁kat", "▁sat", "s"] + [f"▁w{i}" for i in range(28)]
    V = len(pieces) + 1
    vp = str(tmp_path / "v.txt")
    with open(vp, "w", encoding="utf-8") as f:
        f.write("".join(f"{p}\t0\n" for p in pieces))
    arpa = str(tmp_path / "lm.arpa")
    CB.write_arpa(arpa, {("<s>",): (-99.0, -0.3), ("</s>",): (-1.0, None), ("cat",): (-3.0, -0.2), ("kat",): (-0.5, -0.2),
                         ("sat",): (-1.0, -0.1)}, 1)
    lp = np.full((6, V), -12.0, np.float64)
    lp[0, 0], lp[0, 1], lp[0, V - 1] = math.log(0.50), math.log(0.46), math.log(0.04)   # "cat" and "kat" nearly tied
    lp[1, V - 1] = 0.0
    lp[2, 2] = 0.0                                                                        # "sat"
    lp[3:, V - 1] = 0.0
    lp = (lp - np.log(np.exp(lp).sum(1, keepdims=True))).astype(np.float32)
    lm, voc = pkg.LanguageModel(arpa), pkg.engine.Tokenizer(vp)
    plain = hook(pkg, [lp], 4)[0][0]
    fused = hook(pkg, [lp], 4, lm, voc, 1.0, 0.0)[0][0]
    assert [t[0] for t in plain] == [0, 2]                  # acoustics alone: "cat sat"
    assert [t[0] for t in fused] == [1, 2]                  # the LM's word: "kat sat"
    ref = CB.beam_search(lp, 4, lm=CB.Arpa(arpa), pieces=pieces, alpha=1.0, beta=0.0)
    assert [t[:3] for t in fused] == [t[:3] for t in ref["tokens"]]


# ------------------------------------------------------------------ GPU: the engine
# clips whose oracle decisions are wide enough for the device log-probs (checked on the CPU by
# test_end_to_end_clips_have_wide_margins)
E2E = {"tiny": [(43, 20517), (55, 19545)], "110m": [(164, 18716)]}
E2E_LP_ERR = 3e-4           # the per-log-prob error |device - oracle| these clips allow (measured on an H100: 2.2e-4); the GPU test measures it


def _oracle_lp(O, mdl, pcm):
    return O.ctc_log_probs(mdl.W, O.encoder_forward(mdl.W, O.preprocess_audio(pcm, mdl.ocfg.mel_bins), mdl.ocfg))


@pytest.mark.parametrize("kind", ["tiny", "110m"])
def test_end_to_end_clips_have_wide_margins(O, synth, tiny, m110, kind):
    mdl = tiny if kind == "tiny" else m110
    for seed, n in E2E[kind]:
        lp = _oracle_lp(O, mdl, synth.make_audio(n, seed))
        for W in (4, 8):
            assert CB.margins_clear(CB.beam_search(lp, W), lp.shape[0], E2E_LP_ERR)


@gpu
@pytest.mark.parametrize("kind", ["tiny", "110m"])
def test_engine_end_to_end_against_the_oracle(pkg, O, synth, tiny, m110, kind):
    mdl = tiny if kind == "tiny" else m110
    eng = pkg.Engine(mdl.cfg, mdl.weights_path, 0)
    pcms = [synth.make_audio(n, seed) for seed, n in E2E[kind]]
    for W in (4, 8):
        eng.set_ctc_beam(W)
        got = eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM)
        for pcm, g in zip(pcms, got):
            lp = _oracle_lp(O, mdl, pcm)
            err = float(np.abs(eng.ctc_logprobs(eng.encode(eng.mel([pcm]))[0]) - lp).max())
            ref = CB.beam_search(lp, W)
            assert CB.margins_clear(ref, lp.shape[0], err), f"a decision is within 4x its bound (log-prob error {err:.3g})"
            assert [(t.token_id, t.start_frame, t.end_frame) for t in g] == [t[:3] for t in ref["tokens"]]
            assert np.allclose([t.confidence for t in g], [t[3] for t in ref["tokens"]], rtol=1e-3)
    eng.close()


@gpu
def test_engine_rows_are_independent_and_graph_replay_is_stable(pkg, synth, tiny, tmp_path):
    eng = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    rng = np.random.default_rng(3)
    arpa = str(tmp_path / "lm.arpa")
    CB.make_arpa(arpa, _lm_words(tiny.pieces, rng, 40), 3, seed=5, per_order=100)
    lm = pkg.LanguageModel(arpa)
    pcms = [synth.make_audio(n, s) for s, n in ((31, 30000), (32, 16000), (33, 41000))]
    greedy = eng.transcribe_batch(pcms, pkg.Decoder.CTC)
    eng.set_ctc_beam(8, lm, tiny.vocab_path, 0.8, 0.5)
    lm.close()                                              # the engine holds its own copy of the tables
    runs = [eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM) for _ in range(3)]
    assert runs[0] == runs[1] == runs[2]
    assert eng.transcribe_batch([pcms[1]], pkg.Decoder.CTC_BEAM)[0] == runs[0][1]
    encs = eng.encode(eng.mel(pcms))
    assert eng.decode(encs, pkg.Decoder.CTC_BEAM) == runs[0]
    # the greedy decode is unchanged by a beam setting
    assert eng.transcribe_batch(pcms, pkg.Decoder.CTC) == greedy
    eng.close()


@gpu
def test_rejections(pkg, O, synth, tiny, tmp_path):
    L = pkg.load_library()
    eng = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    pcms = [synth.make_audio(20000, 5)]
    with pytest.raises(RuntimeError, match="pk_set_ctc_beam first"):
        eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM)
    for w in (0, 33):
        assert L.pk_set_ctc_beam(eng.h, w, None, None, 0.5, 1.0) == PK_ERR_INVALID
    eng.set_ctc_beam(4)
    eng.set_boost([[3, 4]], 2.0)
    with pytest.raises(RuntimeError, match="boosting"):
        eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM)
    eng.set_boost([], 0.0)
    assert len(eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM)) == 1
    eng.close()
    rcfg = pkg.make_tiny_rnnt_config()
    wp = str(tmp_path / "r.safetensors")
    synth.save_safetensors(wp, synth.make_weights(rcfg, seed=3, blank_bias=-1.0))
    er = pkg.Engine(rcfg, wp, 0)
    assert L.pk_set_ctc_beam(er.h, 4, None, None, 0.5, 1.0) == PK_ERR_INVALID
    with pytest.raises(RuntimeError, match="no CTC head"):
        er.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM)
    er.close()


def _big_arpa(tiny, tmp_path, seed):
    """A 3-gram of about 8 10^4 n-grams over words spelled from the tiny vocabulary: its device tables take ~5 MB."""
    path = str(tmp_path / f"big{seed}.arpa")
    CB.make_arpa(path, _lm_words(tiny.pieces, np.random.default_rng(seed), 2000), 3, seed=seed, per_order=40000)
    return path


@gpu
def test_repeated_and_replaced_language_models_keep_device_memory_flat(pkg, synth, tiny, tmp_path):
    import torch
    eng = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    lms = [pkg.LanguageModel(_big_arpa(tiny, tmp_path, s)) for s in (1, 2)]
    voc = pkg.engine.Tokenizer(tiny.vocab_path)
    pcms = [synth.make_audio(n, s) for s, n in ((41, 24000), (42, 18000))]
    eng.set_ctc_beam(8, lms[0], voc)
    want = [eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM) for _ in range(3)][-1]

    def free():
        eng.sync()
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]

    f0 = free()
    for _ in range(30):                                     # one call per request, as a server makes it
        eng.set_ctc_beam(8, lms[0], voc)
        assert eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM) == want
    assert f0 - free() < (4 << 20), "repeating pk_set_ctc_beam with the same LM grew device memory"
    for k in range(10):                                     # replacing the LM frees the tables it replaces
        eng.set_ctc_beam(8, lms[(k + 1) % 2], voc)
        eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM)
    eng.set_ctc_beam(8, lms[0], voc)
    assert eng.transcribe_batch(pcms, pkg.Decoder.CTC_BEAM) == want
    assert f0 - free() < (4 << 20), "replacing the LM did not free the previous tables"
    eng.close()


# ------------------------------------------------------------------ the C++ drop-in
def _build_cpp(pkg, tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path / "cpp_ctc_beam_check")
    libdir = os.path.dirname(pkg.lib_path())
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"),
                    os.path.join(ROOT, "tests", "cpp_ctc_beam_check.cpp"), "-L" + libdir, "-lparakeet_b200", "-L" + os.path.join(cuda, "lib64"),
                    "-lcudart", "-Wl,-rpath," + libdir, "-o", exe], check=True)
    return exe


@gpu
def test_cpp_transcriber_beam_search(pkg, synth, tiny, tmp_path):
    exe = _build_cpp(pkg, tmp_path)
    arpa = _big_arpa(tiny, tmp_path, 9)
    clip = synth.make_audio(30000, 21)
    fa = str(tmp_path / "a.f32")
    clip.astype(np.float32).tofile(fa)
    out = subprocess.run([exe, tiny.weights_path, tiny.vocab_path, arpa, fa], check=True, capture_output=True, text=True).stdout.splitlines()
    eng = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    lm = pkg.LanguageModel(arpa)
    for line, (W, use_lm) in zip(out[:2], ((6, False), (6, True))):
        eng.set_ctc_beam(W, lm if use_lm else None, tiny.vocab_path, 0.7, 0.3)
        want = eng.transcribe_batch([clip], pkg.Decoder.CTC_BEAM)[0]
        assert line.split() == ["ids"] + [str(t.token_id) for t in want]
    # 30 more transcribe() calls with the LM set: device memory stays flat (each used to copy the LM's tables again)
    assert out[2].startswith("memory_growth ") and int(out[2].split()[1]) < (4 << 20), out[2]
    assert out[3:] == ["boost invalid_argument", "batch_width invalid_argument", "cleared ok"]
    eng.close()
