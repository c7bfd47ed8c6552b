"""The per-request boosting overloads of the C++ drop-in (include/parakeet/transcribe.hpp): transcribe_batch with one
TranscribeOptions per utterance, StreamingBatch::set_boost and set_boost_phrases.  The argument checking and the packing of
the phrase lists run on the host (tests/cpp_boost_host_check.cpp); the overloads end to end on the device
(tests/cpp_boost_rows_check.cpp), compared with the ctypes binding on the same inputs."""
from __future__ import annotations

import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(pkg, name, tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path / name)
    libdir = os.path.dirname(pkg.lib_path())
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", name + ".cpp"),
                    "-L" + libdir, "-lparakeet_b200", "-Wl,-rpath," + libdir, "-o", exe], check=True)
    return exe


def _phrase(O, pieces, idx):
    return "".join(pieces[i] for i in idx).replace(O.SP_MARK, " ").strip()


def test_cpp_batch_options_are_checked_and_packed_on_the_host(pkg, O, tiny, tmp_path):
    exe = _build(pkg, "cpp_boost_host_check", tmp_path)
    pa, pb = _phrase(O, tiny.pieces, (7, 11, 5)), _phrase(O, tiny.pieces, (3, 9))
    out = subprocess.run([exe, tiny.vocab_path, pa, pb], check=True, capture_output=True, text=True).stdout.splitlines()
    assert out[:7] == ["ok none", "count invalid_argument", "rnnt runtime_error", "rnnt_plain none", "decoder invalid_argument",
                       "timestamps invalid_argument", "empty none"]
    a, b = O.tokenizer_encode(pa, tiny.pieces), O.tokenizer_encode(pb, tiny.pieces)
    assert len(a) >= 2 and len(b) >= 1
    # rows: [a, b] | none | [b] (the phrase without tokens is skipped, as ContextTrie::insert does)
    assert out[7].split()[1:] == [str(v) for v in a + b + b]
    assert out[8].split()[1:] == [str(v) for v in (0, len(a), len(a) + len(b), len(a) + 2 * len(b))]
    assert out[9].split()[1:] == ["0", "2", "2", "3"]
    assert out[10].split()[1:] == ["4", "5", "7.5"]
    assert out[11] == "any 1 0"


@pytest.mark.gpu
def test_cpp_boost_overloads_end_to_end(pkg, O, synth, tiny, tmp_path):
    exe = _build(pkg, "cpp_boost_rows_check", tmp_path)
    pa, pb = _phrase(O, tiny.pieces, (7, 11, 5)), _phrase(O, tiny.pieces, (3, 9))
    clips = [synth.make_audio(32000, 11), synth.make_audio(20000, 12)]
    fa, fb = str(tmp_path / "a.f32"), str(tmp_path / "b.f32")
    clips[0].astype(np.float32).tofile(fa)
    clips[1].astype(np.float32).tofile(fb)
    socfg, scfg = O.make_tiny_stream_config(), pkg.make_tiny_stream_config()
    sw, sp = str(tmp_path / "ts.safetensors"), str(tmp_path / "s.f32")
    synth.save_safetensors(sw, synth.make_weights(socfg, seed=3))
    sched = [2560, 1280, 0, 4000, 2560, 700, 2560, 2560]
    spcm = synth.make_audio(sum(sched), 77)
    spcm.astype(np.float32).tofile(sp)
    out = subprocess.run([exe, tiny.weights_path, tiny.vocab_path, fa, fb, pa, pb, sw, sp, ",".join(str(n) for n in sched)],
                         check=True, capture_output=True, text=True).stdout.strip().split("\n")
    fmt = lambda toks: [f"{t.token_id}:{t.start_frame}:{t.end_frame}" for t in toks]  # noqa: E731
    tk = pkg.engine.Tokenizer(tiny.vocab_path)
    a, b = tk.encode(pa), tk.encode(pb)
    utts = [clips[0], clips[1], clips[0]]
    e = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    try:
        li = 0
        for dec in (pkg.Decoder.CTC, pkg.Decoder.TDT):
            e.set_boost_rows([[a], [], [b, a]], [6.0, 0.0, 9.0])
            want = e.transcribe_batch(utts, dec)
            e.set_boost_rows([], [])
            plain = e.transcribe_batch(utts, dec)
            for i in range(3):
                assert out[li + i].split()[1:] == fmt(want[i]) and out[li + i].startswith("ROW"), (dec, i)
                assert out[li + 3 + i].split()[1:] == fmt(plain[i]) and out[li + 3 + i].startswith("PLAIN"), (dec, i)
            assert fmt(want[1]) == fmt(plain[1])
            li += 6
        assert out[li].startswith("ERR transcribe_batch: one TranscribeOptions per utterance")
        li += 1
    finally:
        e.close()
    # the stream: plain pass, then reset + set_boost_phrases; both equal the binding's stream with the same calls
    es = pkg.Engine(scfg, sw, 0)
    try:
        es.stream_open(1, 5120)
        for tag, boosted in (("SPLAIN", False), ("SBOOST", True)):
            if boosted:
                es.stream_reset(-1)
                es.stream_set_boost(0, [a, b], 25.0)
            pos = 0
            for n in sched:
                got = es.stream_step([spcm[pos:pos + n]])[0]
                pos += n
                assert out[li].startswith(tag) and out[li].split()[1:] == fmt(got), li
                li += 1
    finally:
        es.close()
    assert out[li].startswith("ERR StreamingBatch::set_boost: no such stream")
