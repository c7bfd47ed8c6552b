"""Speaker-attributed transcription (DiarizedTranscriber): the word -> speaker step on the host (pk_diarize_transcription,
pk_diarize_words, the C++ diarize_transcription) and its numpy restatement (tests/diarize_oracle.py) against goldens of the
compiled reference (tests/golden/golden_diarized_v1.npz, made by make_golden_diarized.py), and on the GPU the joint call
pk_transcribe_diarize_batch against the two single-engine calls and the reference's DiarizedTranscriber end to end."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import diarize_oracle as DO  # noqa: E402
import sortformer_oracle as SO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_diarized_v1.npz")
SF_GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_sortformer_v1.npz")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libpkref_diarized.so")
CONF_RTOL = 1e-3
F32 = np.float32


@pytest.fixture(scope="module")
def g():
    with np.load(GOLDEN, allow_pickle=False) as f:
        return dict(f)


def crafted(g):
    w_off, s_off = g["c.w_off"], g["c.s_off"]
    for c in range(len(w_off) - 1):
        w, s = slice(w_off[c], w_off[c + 1]), slice(s_off[c], s_off[c + 1])
        yield g["c.ws"][w], g["c.we"][w], g["c.spk"][s], g["c.ss"][s], g["c.se"][s], g["c.want"][w]


def e2e_keys(g):
    return sorted({k.rsplit(".", 1)[0] for k in g if k.startswith("e2e.") and k.count(".") == 3})


def _abi_speakers(pkg, ws, we, spk, ss, se):
    L = pkg.load_library()
    ws, we, ss, se = (np.ascontiguousarray(np.append(a, 0), F32) for a in (ws, we, ss, se))
    spk = np.ascontiguousarray(np.append(spk, 0), np.int32)
    out = np.zeros(len(ws), np.int32)
    f, i = pkg.engine._f32p, pkg.engine._i32p
    assert L.pk_diarize_transcription(f(ws), f(we), len(ws) - 1, i(spk), f(ss), f(se), len(spk) - 1, i(out)) == 0
    return out[:-1]


# ---------------------------------------------------------------- CPU


def test_crafted_cases_equal_reference(pkg, g):
    n = 0
    for ws, we, spk, ss, se, want in crafted(g):
        assert np.array_equal(DO.assign_speakers(ws, we, spk, ss, se), want)
        assert np.array_equal(_abi_speakers(pkg, ws, we, spk, ss, se), want)
        n += 1
    assert n >= 100


def test_crafted_cases_cover_the_edges(g):
    ties = zero_words = minus = 0
    for ws, we, spk, ss, se, want in crafted(g):
        ties += int(DO.exact_tie(ws, we, spk, ss, se).sum())
        zero_words += int((ws == we).sum())
        minus += int((want == -1).sum())
    assert ties >= 2 * (12 + 24 + 24) and zero_words >= 2 and minus >= 4


def test_e2e_speakers_equal_reference(pkg, g):
    keys = e2e_keys(g)
    assert len(keys) == 4                                   # CTC and TDT, 10 s and 30 s
    tie = minus = False
    for k in keys:
        w, segs = g[k + ".w"], g[k + ".segs"]
        spk = segs[:, 0].astype(np.int32)
        want = w[:, 2].astype(np.int32)
        assert np.array_equal(DO.assign_speakers(w[:, 0], w[:, 1], spk, segs[:, 1], segs[:, 2]), want)
        assert np.array_equal(_abi_speakers(pkg, w[:, 0], w[:, 1], spk, segs[:, 1], segs[:, 2]), want)
        tie |= bool(DO.exact_tie(w[:, 0], w[:, 1], spk, segs[:, 1], segs[:, 2]).any())
        minus |= bool((want == -1).any())
    assert tie and minus


def test_segments_in_reference_order(pkg):
    """pk_diarize_words orders segments as the reference's std::sort does, also above 16 segments where equal starts leave
    speaker order (golden_sortformer_v1: the compiled reference's Sortformer::diarize on sortformer-117m)."""
    with np.load(SF_GOLDEN) as gs:
        for i in range(2):
            p, ref = gs[f"s117m.u{i}.probs"], gs[f"s117m.u{i}.segs"]
            segs, _ = pkg.diarize_words(p, [])
            got = np.array([[s.speaker_id, s.start, s.end] for s in segs], F32)
            assert np.array_equal(got, ref)
            assert len(ref) > 16 and any(ref[j, 1] == ref[j + 1, 1] and ref[j, 0] > ref[j + 1, 0] for j in range(len(ref) - 1))
            # at most 16 segments, the order is pk_diar_segments' (and the numpy oracle's)
            short = p[:12]
            a, _ = pkg.diarize_words(short, [])
            if len(a) <= 16:
                assert [(s.speaker_id, s.start) for s in a] == [(s.speaker_id, s.start) for s in pkg.diar_segments(short)]


def test_diarize_words_argument_checks(pkg):
    L = pkg.load_library()
    p = np.zeros((4, 2), F32)
    assert L.pk_diarize_words(None, 4, 2, 0.5, None, None, 0, None, None, None, None, 0) == -1
    assert L.pk_diarize_words(pkg.engine._f32p(p), 4, 0, 0.5, None, None, 0, None, None, None, None, 0) == -1
    assert L.pk_diarize_transcription(None, None, 1, None, None, None, 0, None) != 0
    segs, words = pkg.diarize_words(p, [])
    assert segs == [] and words == []


@pytest.mark.skipif(not os.path.exists(REF_LIB), reason="oracle/_ref/libpkref_diarized.so not built (make_golden_diarized.py)")
def test_fuzz_against_compiled_reference(pkg):
    """Random word and segment lists, many with more than 16 segments and equal starts, against the reference's own
    diarize_transcription."""
    L = C.CDLL(REF_LIB)
    L.pkdz_transcription.argtypes = [C.c_void_p] * 2 + [C.c_int] + [C.c_void_p] * 3 + [C.c_int, C.c_void_p]
    rng = np.random.default_rng(11)
    t = lambda a: a.astype(F32) * F32(0.08)   # noqa: E731
    for case in range(400):
        nw, ns = int(rng.integers(0, 30)), int(rng.integers(0, 60))
        w0 = rng.integers(0, 40, nw)
        ws, we = t(w0), t(w0 + rng.integers(0, 8, nw))
        s0 = rng.integers(0, 12 if case % 2 else 40, ns)            # odd cases: many equal starts
        spk = rng.integers(0, 4, ns).astype(np.int32)
        ss, se = t(s0), t(s0 + rng.integers(0, 10, ns))
        want = np.zeros(max(nw, 1), np.int32)
        a = [np.ascontiguousarray(x) for x in (ws, we, spk, ss, se)]
        L.pkdz_transcription(a[0].ctypes.data, a[1].ctypes.data, nw, a[2].ctypes.data, a[3].ctypes.data, a[4].ctypes.data, ns,
                             want.ctypes.data)
        assert np.array_equal(_abi_speakers(pkg, ws, we, spk, ss, se), want[:nw])
        assert np.array_equal(DO.assign_speakers(ws, we, spk, ss, se), want[:nw])


def _cpp_exe(pkg, tmp_path):
    exe = str(tmp_path / "cpp_diarize_check")
    libdir = os.path.dirname(pkg.lib_path())
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp_diarize_check.cpp"),
                    "-L" + libdir, "-lparakeet_b200", "-Wl,-rpath," + libdir, "-o", exe], check=True)
    return exe


def test_cpp_diarize_transcription_crafted(pkg, g, tmp_path):
    exe = _cpp_exe(pkg, tmp_path)
    fp = str(tmp_path / "cases.bin")
    with open(fp, "wb") as f:
        n = len(g["c.w_off"]) - 1
        for a in (np.array([n], np.int32), g["c.w_off"].astype(np.int32), g["c.s_off"].astype(np.int32), g["c.ws"], g["c.we"],
                  g["c.spk"].astype(np.int32), g["c.ss"], g["c.se"]):
            f.write(np.ascontiguousarray(a).tobytes())
    out = subprocess.run([exe, "crafted", fp], check=True, capture_output=True, text=True).stdout.strip().split("\n")
    cases = list(crafted(g))
    assert len(out) == len(cases)
    for line, c in zip(out, cases):
        assert [int(v) for v in line.split()[1:]] == c[-1].tolist()


# ---------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def models(pkg, synth, tmp_path_factory):
    """The models of the end-to-end golden on disk: tdt-ctc-110m (seed 0) + vocabulary, sortformer-117m with the calibrated
    weights of golden_sortformer_v1.npz, and that file's 10 s and 30 s clips."""
    import __graft_entry__ as ge
    O = ge.load_oracle()
    d = tmp_path_factory.mktemp("diarized")
    ocfg = O.make_110m_config()
    wa, ws, vp = str(d / "asr.safetensors"), str(d / "sf.safetensors"), str(d / "vocab.txt")
    synth.save_safetensors(wa, synth.make_weights(ocfg, seed=0))
    synth.save_vocab(vp, synth.make_vocab(ocfg.vocab - 1, seed=0))
    with np.load(SF_GOLDEN) as gs:
        scfg = pkg.make_sortformer_117m_config()
        synth.save_safetensors(ws, SO.golden_weights(scfg, gs, "s117m", synth))
        lens, aseed = [int(x) for x in gs["s117m.lens"]], int(gs["s117m.audio_seed"])
    clips = [synth.make_audio(n, aseed + i) for i, n in enumerate(lens)]
    return wa, ws, vp, clips


@pytest.fixture(scope="module")
def engines(pkg, models):
    wa, ws, vp, clips = models
    cap = dict(max_batch=8, max_samples=30 * 16000)
    asr = pkg.Engine(pkg.make_110m_config(**cap), wa, 0)
    diar = pkg.Engine(pkg.make_sortformer_117m_config(**cap), ws, 0)
    yield asr, diar
    asr.close()
    diar.close()


def _ragged(clips, synth):
    a, b = clips
    return [a, b[:250000], synth.make_audio(40000, 5), b, a[:90000], synth.make_audio(123457, 6)]


def _separate(asr, diar, pcms, dec):
    return asr.transcribe_batch(pcms, dec), diar.diarize_probs(pcms)


def _assert_same(got, want):
    (gt, gp), (wt, wp) = got, want
    assert len(gt) == len(wt) and len(gp) == len(wp)
    for a, b in zip(gt, wt):
        assert [(t.token_id, t.start_frame, t.end_frame, np.float32(t.confidence).tobytes()) for t in a] == \
               [(t.token_id, t.start_frame, t.end_frame, np.float32(t.confidence).tobytes()) for t in b]
    for a, b in zip(gp, wp):
        assert a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("dec", ["CTC", "TDT"])
def test_joint_equals_separate(pkg, synth, engines, models, dec):
    asr, diar = engines
    pcms = _ragged(models[3], synth)
    d = pkg.Decoder[dec]
    want = _separate(asr, diar, pcms, d)
    for _ in range(3):                                   # eager, capture, replay of both graphs
        _assert_same(asr.transcribe_diarize_batch(diar, pcms, d), want)


@pytest.mark.gpu
def test_buffer_reuse_across_batches(pkg, synth, engines, models):
    """Three batches of different content through pk_prefetch_pcm -> pk_stage_pcm -> the joint run, each prefetch issued
    while the previous batch is still running: every batch equals its separate-call result."""
    import torch
    asr, diar = engines
    clips = models[3]
    batches = [[synth.make_audio(160000, 50 + 10 * k + i) for i in range(6)] + [clips[k % 2]] for k in range(3)]
    d = pkg.Decoder.TDT
    want = [_separate(asr, diar, b, d) for b in batches]
    packed = []
    for b in batches:
        buf, off = pkg.engine._pack(b)
        pin = torch.empty(len(buf), dtype=torch.float32, pin_memory=True).numpy()
        pin[:] = buf
        packed.append((pin, off))
    M = [sum(asr.L.pk_encoder_frames(asr.L.pk_mel_frames(len(p))) for p in b) for b in batches]
    for rnd in range(2):
        asr.prefetch(*packed[0])
        for k in range(3):
            asr.stage(*packed[k])
            asr.run_transcribe_diarize_staged(diar, d)
            if k + 1 < 3:
                asr.prefetch(*packed[k + 1])
            toks = asr.fetch(len(batches[k]))
            probs, lens = np.zeros((M[k], 4), F32), np.zeros(len(batches[k]), np.int32)
            diar.fetch_probs(probs, lens)
            _assert_same((toks, diar._probs(lens, probs)), want[k])


@pytest.mark.gpu
def test_rejections_leave_engines_usable(pkg, synth, engines, models, tmp_path):
    asr, diar = engines
    pcms = [synth.make_audio(32000, 1), synth.make_audio(20000, 2)]
    L = asr.L

    def status(a, b, p, dec):
        buf, off = pkg.engine._pack(p)
        t, _ = a._tokens(len(p))
        probs, lens = np.zeros((4096, 4), F32), np.zeros(max(len(p), 1), np.int32)
        return L.pk_transcribe_diarize_batch(a.h, b.h, pkg.engine._f32p(buf), pkg.engine._i64p(off), len(p), int(dec), C.byref(t),
                                             pkg.engine._f32p(probs), pkg.engine._i32p(lens))

    INVALID, CAPACITY = 1, 5
    assert status(diar, diar, pcms, pkg.Decoder.TDT) == INVALID          # asr is a Sortformer engine
    assert status(asr, asr, pcms, pkg.Decoder.TDT) == INVALID            # diar is not a Sortformer engine
    assert status(diar, asr, pcms, pkg.Decoder.TDT) == INVALID
    assert status(asr, diar, pcms, pkg.Decoder.RNNT) == INVALID          # decoder
    assert status(asr, diar, pcms, 7) == INVALID
    assert status(asr, diar, [pcms[0]] * 9, pkg.Decoder.TDT) == CAPACITY   # n_utt over both capacities
    long = synth.make_audio(30 * 16000 + 1, 3)
    assert status(asr, diar, [long], pkg.Decoder.TDT) == CAPACITY
    # an RNN-T ASR engine
    import __graft_entry__ as ge
    RO = ge.load_rnnt_oracle()
    rcfg = pkg.make_tiny_rnnt_config()
    wr = str(tmp_path / "rnnt.safetensors")
    synth.save_safetensors(wr, synth.make_weights(rcfg, seed=3, blank_bias=-1.0))
    er = pkg.Engine(rcfg, wr, 0)
    try:
        assert status(er, diar, pcms, pkg.Decoder.RNNT) == INVALID
        assert status(er, diar, pcms, pkg.Decoder.TDT) == INVALID
    finally:
        er.close()
    assert RO is not None
    # a smaller Sortformer: the utterance fits asr but not diar
    small = pkg.Engine(pkg.make_sortformer_117m_config(max_batch=1, max_samples=24000), models[1], 0)
    try:
        assert status(asr, small, pcms, pkg.Decoder.TDT) == CAPACITY
        assert "max_samples" in L.pk_last_error(asr.h).decode() or "max_batch" in L.pk_last_error(asr.h).decode()
    finally:
        small.close()
    # both engines still give the separate calls' results
    for dec in (pkg.Decoder.CTC, pkg.Decoder.TDT):
        _assert_same(asr.transcribe_diarize_batch(diar, pcms, dec), _separate(asr, diar, pcms, dec))


def _check_result(pkg, r, g, k):
    text = g[k + ".text"].tobytes().decode("utf-8")
    names = g[k + ".words"].tobytes().decode("utf-8").split("\n")[:-1]
    w, wt, segs = g[k + ".w"], g[k + ".wt"], g[k + ".segs"]
    assert r.text == text
    assert [x.word for x in r.words] == names and [x.word for x in r.word_timestamps] == names
    got = np.array([[x.start, x.end, x.speaker_id] for x in r.words], F32).reshape(-1, 3)
    assert np.array_equal(got, w[:, :3])
    np.testing.assert_allclose(np.array([x.confidence for x in r.words], F32), w[:, 3], rtol=CONF_RTOL)
    got_t = np.array([[x.start, x.end] for x in r.word_timestamps], F32).reshape(-1, 2)
    assert np.array_equal(got_t, wt[:, :2])
    np.testing.assert_allclose(np.array([x.confidence for x in r.word_timestamps], F32), wt[:, 2], rtol=CONF_RTOL)
    got_s = np.array([[x.speaker_id, x.start, x.end] for x in r.segments], F32).reshape(-1, 3)
    assert np.array_equal(got_s, segs)


@pytest.mark.gpu
def test_python_diarized_transcriber_equals_reference(pkg, g, models):
    wa, ws, vp, clips = models
    dt = pkg.DiarizedTranscriber(wa, ws, vp, max_batch=4, max_samples=30 * 16000)
    try:
        for name, dec in (("ctc", pkg.Decoder.CTC), ("tdt", pkg.Decoder.TDT)):
            rs = dt.transcribe_batch(clips, dec)
            for i, r in enumerate(rs):
                _check_result(pkg, r, g, f"e2e.{name}.u{i}")
            _check_result(pkg, dt.to_gpu().transcribe(clips[0], dec), g, f"e2e.{name}.u0")
    finally:
        dt.close()


@pytest.mark.gpu
def test_cpp_diarized_transcriber_equals_reference(pkg, g, models, tmp_path):
    wa, ws, vp, clips = models
    exe = _cpp_exe(pkg, tmp_path)
    pps = []
    for i, c in enumerate(clips):
        pp = str(tmp_path / f"pcm{i}.f32")
        c.astype(F32).tofile(pp)
        pps.append(pp)
    for name in ("ctc", "tdt"):
        out = subprocess.run([exe, "e2e", wa, ws, vp, name, str(30 * 16000)] + pps, check=True, capture_output=True,
                             text=True).stdout.split("\n")
        results, cur = [], None
        for line in out:
            if line.startswith("TEXT"):
                cur = pkg.DiarizedResult(line[5:])
                results.append(cur)
            elif line.startswith("WORD"):
                _, word, a, b, s, c = line.split(" ")
                cur.words.append(pkg.DiarizedWord(word, float.fromhex(a), float.fromhex(b), int(s), float.fromhex(c)))
                cur.word_timestamps.append(pkg.WordTimestamp(word, float.fromhex(a), float.fromhex(b), float.fromhex(c)))
            elif line.startswith("SEG"):
                _, s, a, b = line.split(" ")
                cur.segments.append(pkg.DiarizationSegment(int(s), float.fromhex(a), float.fromhex(b)))
        assert len(results) == len(clips) + 1
        for i, r in enumerate(results):
            _check_result(pkg, r, g, f"e2e.{name}.u{i % len(clips)}")
