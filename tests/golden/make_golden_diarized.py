"""Writes tests/golden/golden_diarized_v1.npz from the compiled reference's speaker-attributed transcription
(src/diarize.cpp) through tests/golden/ref_diarized.cpp.

    python tests/golden/make_golden_diarized.py

Recorded:
  crafted   direct calls of diarize_transcription on word and segment lists built to hit its edges: exact ties between 2, 3
            and 4 speakers in every order of first overlap (whole-word cover and sums of partial overlaps), zero-length
            words, single-frame (zero-length) segments, words outside every segment, several segments of one speaker
            inside one word, and random lists on the 0.08 s grid.  Packed: c.w_off / c.ws / c.we, c.s_off / c.spk / c.ss /
            c.se, c.want (speaker per word).
  e2e       DiarizedTranscriber::transcribe on a 10 s and a 30 s synthetic clip, CTC and TDT: text, words (word, start, end,
            speaker, confidence), segments in the reference's order and word_timestamps.  ASR: the tdt-ctc-110m synthetic
            checkpoint and vocabulary of make_golden.py (seed 0).  Sortformer: sortformer-117m with the calibrated weights of
            golden_sortformer_v1.npz (its seed and output_proj_ bias, chosen there with the MARGIN rule) on that file's own
            clips.  The generator asserts that the set holds a word decided by an exact tie, a word with speaker -1 and an
            utterance of more than 16 segments whose equal starts are not in speaker order.

The reference objects come from oracle/Makefile; ref_diarized.cpp and src/diarize.cpp, src/sortformer.cpp,
src/transformer.cpp are linked against them into oracle/_ref/libpkref_diarized.so.  Needs the reference sources.
"""
from __future__ import annotations

import ctypes as C
import itertools
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import __graft_entry__ as ge  # noqa: E402
import diarize_oracle as DO  # noqa: E402
import sortformer_oracle as SO  # noqa: E402

LIB = os.path.join(ROOT, "oracle", "_ref", "libpkref_diarized.so")
F32 = np.float32


def build_lib():
    mk = os.path.join(tempfile.mkdtemp(), "diarized.mk")
    with open(mk, "w") as f:
        f.write("include Makefile\n"
                "$(OUT)/libpkref_diarized.so: $(AX_OBJS) $(HWY_OBJS) $(PK_OBJS) $(OBJ)/pk/src/diarize.cpp.o $(OBJ)/pk/src/sortformer.cpp.o "
                "$(OBJ)/pk/src/transformer.cpp.o $(OBJ)/ref_diarized.o\n"
                "\t$(CXX) -shared -fopenmp -o $@ $^ -lpthread\n"
                f"$(OBJ)/ref_diarized.o: {os.path.join(HERE, 'ref_diarized.cpp')}\n"
                "\t@mkdir -p $(dir $@)\n"
                "\t$(CXX) $(PK_CXXFLAGS) $(INCS) -c $< -o $@\n")
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", mk, "-j8", "_ref/libpkref_diarized.so"], check=True)
    return load_lib()


def load_lib():
    L = C.CDLL(LIB)
    vp = C.c_void_p
    L.pkdz_last_error.restype = C.c_char_p
    L.pkdz_new.restype = vp
    L.pkdz_new.argtypes = [C.c_char_p] * 3
    L.pkdz_free.argtypes = [vp]
    L.pkdz_transcription.argtypes = [vp, vp, C.c_int, vp, vp, vp, C.c_int, vp]
    L.pkdz_run.argtypes = [vp, vp, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_int] + [vp] * 7 + \
        [C.c_int, vp] + [vp] * 3 + [C.c_int, vp]
    return L


def ref_transcription(L, ws, we, spk, ss, se):
    ws, we, ss, se = (np.ascontiguousarray(a, F32) for a in (ws, we, ss, se))
    spk = np.ascontiguousarray(spk, np.int32)
    out = np.zeros(max(len(ws), 1), np.int32)
    L.pkdz_transcription(ws.ctypes.data, we.ctypes.data, len(ws), spk.ctypes.data, ss.ctypes.data, se.ctypes.data, len(spk),
                         out.ctypes.data)
    return out[:len(ws)]


def crafted_cases(rng):
    """-> list of (words [(start, end)], segments [(speaker, start, end)])."""
    t = lambda f: F32(f) * F32(0.08)   # noqa: E731  (frame_to_seconds)
    cases = []
    for k in (2, 3, 4):
        for perm in itertools.permutations(range(4), k):
            # every speaker covers the whole word: equal overlaps, first overlaps in `perm` order
            cases.append(([(t(10), t(20))], [(s, t(5), t(25)) for s in perm]))
            # the same sums built from parts: the first speaker in two halves, the rest whole
            segs = [(perm[0], t(10), t(15)), (perm[0], t(15), t(20))] + [(s, t(8), t(22)) for s in perm[1:]]
            cases.append(([(t(10), t(20)), (t(12), t(18))], segs))
    cases.append(([(t(7), t(7)), (t(3), t(3))], [(0, t(0), t(10)), (1, t(2), t(9))]))                  # zero-length words
    cases.append(([(t(4), t(9))], [(1, t(6), t(6)), (0, t(5), t(5)), (2, t(7), t(7))]))                # single-frame segments
    cases.append(([(t(4), t(9))], [(1, t(6), t(6)), (0, t(8), t(12))]))
    cases.append(([(t(30), t(40)), (t(0), t(1))], [(0, t(2), t(10)), (1, t(41), t(50))]))              # outside every segment
    cases.append(([(t(10), t(30))], [(2, t(11), t(13)), (2, t(15), t(16)), (2, t(20), t(24)), (1, t(9), t(16))]))   # one speaker, several segments
    cases.append(([(t(10), t(30))], [(2, t(11), t(13)), (1, t(9), t(12)), (2, t(15), t(17))]))        # 2 + 2 frames against 3: speaker 1
    cases.append(([], [(0, t(0), t(3))]))
    cases.append(([(t(1), t(2))], []))
    for _ in range(64):                                                                              # random, on the frame grid
        nw, ns = int(rng.integers(1, 12)), int(rng.integers(0, 40))
        w0 = rng.integers(0, 60, nw)
        words = [(t(a), t(a + int(rng.integers(0, 6)))) for a in w0]
        s0 = rng.integers(0, 60, ns)
        segs = [(int(rng.integers(0, 4)), t(a), t(a + int(rng.integers(0, 8)))) for a in s0]
        cases.append((words, segs))
    return cases


def pack_crafted(L, cases):
    w_off, s_off = [0], [0]
    ws, we, spk, ss, se, want = [], [], [], [], [], []
    for words, segs in cases:
        a = np.array([w[0] for w in words], F32)
        b = np.array([w[1] for w in words], F32)
        sp = np.array([s[0] for s in segs], np.int32)
        s0 = np.array([s[1] for s in segs], F32)
        s1 = np.array([s[2] for s in segs], F32)
        got = ref_transcription(L, a, b, sp, s0, s1)
        assert np.array_equal(got, DO.assign_speakers(a, b, sp, s0, s1)), "the numpy oracle differs from the reference"
        ws += list(a); we += list(b); spk += list(sp); ss += list(s0); se += list(s1); want += list(got)
        w_off.append(len(ws)); s_off.append(len(spk))
    return {"c.w_off": np.array(w_off, np.int32), "c.ws": np.array(ws, F32), "c.we": np.array(we, F32),
            "c.s_off": np.array(s_off, np.int32), "c.spk": np.array(spk, np.int32), "c.ss": np.array(ss, F32),
            "c.se": np.array(se, F32), "c.want": np.array(want, np.int32)}


def run_ref(L, h, pcm, dec):
    pcm = np.ascontiguousarray(pcm, F32)
    cap = 4096
    text, words = C.create_string_buffer(1 << 16), C.create_string_buffer(1 << 18)
    wf = [np.zeros(cap, F32) for _ in range(6)]
    wspk = np.zeros(cap, np.int32)
    sspk, sst, sen = np.zeros(cap, np.int32), np.zeros(cap, F32), np.zeros(cap, F32)
    nw, ns = C.c_int(), C.c_int()
    rc = L.pkdz_run(h, pcm.ctypes.data, len(pcm), dec, text, len(text), words, len(words), wf[0].ctypes.data, wf[1].ctypes.data,
                    wspk.ctypes.data, wf[2].ctypes.data, wf[3].ctypes.data, wf[4].ctypes.data, wf[5].ctypes.data, cap, C.byref(nw),
                    sspk.ctypes.data, sst.ctypes.data, sen.ctypes.data, cap, C.byref(ns))
    if rc != 0:
        raise RuntimeError("pkdz_run: " + L.pkdz_last_error().decode())
    n, m = nw.value, ns.value
    return {"text": np.frombuffer(text.value, np.uint8).copy(), "words": np.frombuffer(words.value, np.uint8).copy(),
            "w": np.stack([wf[0][:n], wf[1][:n], wspk[:n].astype(F32), wf[2][:n]], axis=1),
            "wt": np.stack([wf[3][:n], wf[4][:n], wf[5][:n]], axis=1),
            "segs": np.stack([sspk[:m].astype(F32), sst[:m], sen[:m]], axis=1)}


def unordered_equal_starts(segs):
    """More than 16 segments, and some run of equal starts that is not in speaker order."""
    if len(segs) <= 16:
        return False
    return any(segs[i, 1] == segs[i + 1, 1] and segs[i, 0] > segs[i + 1, 0] for i in range(len(segs) - 1))


def main():
    L = build_lib()
    pkg = ge.load_package()
    from parakeet_cpp_b200 import synth
    O = ge.load_oracle()
    out = pack_crafted(L, crafted_cases(np.random.default_rng(7)))
    print("crafted cases", len(out["c.w_off"]) - 1, "words", len(out["c.want"]), flush=True)
    gs = np.load(os.path.join(HERE, "golden_sortformer_v1.npz"))
    scfg = pkg.make_sortformer_117m_config()
    Wsf = SO.golden_weights(scfg, gs, "s117m", synth)
    lens, aseed = [int(x) for x in gs["s117m.lens"]], int(gs["s117m.audio_seed"])
    out["e2e.lens"] = np.array(lens, np.int64)
    out["e2e.audio_seed"] = np.int64(aseed)
    out["e2e.asr_seed"] = np.int64(0)
    out["e2e.sf_seed"] = gs["s117m.seed"]
    out["e2e.spk_bias"] = gs["s117m.spk_bias"]
    ocfg = O.make_110m_config()
    tie = minus = unordered = False
    with tempfile.TemporaryDirectory() as td:
        wa, wsf, vp = (os.path.join(td, f) for f in ("asr.safetensors", "sf.safetensors", "vocab.txt"))
        synth.save_safetensors(wa, synth.make_weights(ocfg, seed=0))
        synth.save_vocab(vp, synth.make_vocab(ocfg.vocab - 1, seed=0))
        synth.save_safetensors(wsf, Wsf)
        h = L.pkdz_new(wa.encode(), wsf.encode(), vp.encode())
        if not h:
            raise RuntimeError("pkdz_new: " + L.pkdz_last_error().decode())
        for dec, name in ((0, "ctc"), (1, "tdt")):
            for i, n in enumerate(lens):
                r = run_ref(L, h, synth.make_audio(n, aseed + i), dec)
                for k, v in r.items():
                    out[f"e2e.{name}.u{i}.{k}"] = v
                w, segs = r["w"], r["segs"]
                ties = DO.exact_tie(w[:, 0], w[:, 1], segs[:, 0].astype(np.int32), segs[:, 1], segs[:, 2])
                tie |= bool(ties.any())
                minus |= bool((w[:, 2] == -1).any())
                unordered |= unordered_equal_starts(segs)
                assert np.array_equal(DO.assign_speakers(w[:, 0], w[:, 1], segs[:, 0].astype(np.int32), segs[:, 1], segs[:, 2]),
                                      w[:, 2].astype(np.int32)), "the numpy oracle differs from the reference"
                print(name, i, "words", len(w), "segments", len(segs), "ties", int(ties.sum()), "-1", int((w[:, 2] == -1).sum()),
                      flush=True)
        L.pkdz_free(h)
    assert tie and minus and unordered, f"end-to-end set lacks a case: tie {tie}, -1 {minus}, unordered equal starts {unordered}"
    path = os.path.join(HERE, "golden_diarized_v1.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
