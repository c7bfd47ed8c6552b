"""Writes tests/golden/golden_sortformer_v1.npz from the compiled reference's Sortformer (src/sortformer.cpp,
src/transformer.cpp) through the reference CLI's `sortformer` steps (tests/golden/ref_sortformer.cpp).

    python tests/golden/make_golden_sortformer.py

Recorded, per utterance: the transformer output (float16), the sigmoid activities (float32) and the segments of
Sortformer::diarize; features and NEST encoder output (float16) where keep() says so, to keep the file near 1 MB.
  tiny    the test-only tiny Sortformer (head_dim 24, post-norm; parakeet_cpp_b200.make_tiny_sortformer_config) on a ragged
          batch of 16 utterances (tests/test_sortformer.py TINY_LENS);
  s117m   the sortformer-117m preset on a 10 s and a 30 s clip.
Weights: synth.make_sortformer_weights(seed) with output_proj_'s bias calibrated by sortformer_oracle.calibrated_weights on
these clips; the first seed whose smallest |logit| is at least MARGIN is taken.  The seed, the bias, MARGIN and the
smallest |logit| reached are stored.  The numpy oracle runs first (it picks the seed); the reference then loads every
module with strict = true, so the key layout of the synthetic checkpoint is checked against the reference's registration.

The reference objects come from oracle/Makefile (`make -C oracle ref`); ref_sortformer.cpp and src/sortformer.cpp +
src/transformer.cpp are linked against them into oracle/_ref/libpkref_sortformer.so.  Needs the reference sources.
"""
from __future__ import annotations

import ctypes as C
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
import sortformer_oracle as SO  # noqa: E402
from test_sortformer import MARGIN, TINY_LENS  # noqa: E402

pkg = ge.load_package()
from parakeet_cpp_b200 import synth  # noqa: E402

LIB = os.path.join(ROOT, "oracle", "_ref", "libpkref_sortformer.so")
S117_LENS = [160000, 480000]


def keep(tag, i, name):
    """What is stored beyond the transformer output, activities and segments (the file stays near 1 MB): the features of the
    first four tiny utterances and of the 10 s clip, the NEST encoder output of every tiny utterance and of the 10 s clip."""
    if name == "feats":
        return i < 4 if tag == "tiny" else i == 0
    return tag == "tiny" or i == 0


def build_lib():
    mk = os.path.join(tempfile.mkdtemp(), "sortformer.mk")
    with open(mk, "w") as f:
        f.write("include Makefile\n"
                "$(OUT)/libpkref_sortformer.so: $(AX_OBJS) $(HWY_OBJS) $(PK_OBJS) $(OBJ)/pk/src/sortformer.cpp.o "
                "$(OBJ)/pk/src/transformer.cpp.o $(OBJ)/ref_sortformer.o\n"
                "\t$(CXX) -shared -fopenmp -o $@ $^ -lpthread\n"
                f"$(OBJ)/ref_sortformer.o: {os.path.join(HERE, 'ref_sortformer.cpp')}\n"
                "\t@mkdir -p $(dir $@)\n"
                "\t$(CXX) $(PK_CXXFLAGS) $(INCS) -c $< -o $@\n")
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", mk, "-j8", "_ref/libpkref_sortformer.so"], check=True)
    L = C.CDLL(LIB)
    L.pksf_last_error.restype = C.c_char_p
    L.pksf_new.restype = C.c_void_p
    L.pksf_new.argtypes = [C.c_char_p, C.POINTER(C.c_int32)]
    L.pksf_free.argtypes = [C.c_void_p]
    L.pksf_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p, C.c_int, C.c_void_p] + [C.c_void_p] * 3 + \
        [C.c_int, C.c_void_p] + [C.c_void_p] * 3 + [C.c_int, C.c_void_p]
    return L


def run_ref(L, wp, cfg, pcm):
    e = cfg.encoder
    dims = np.array([e.mel_bins, e.sub_channels, e.d_model, e.n_layers, e.n_heads, e.ff, cfg.t_hidden, cfg.t_layers, cfg.t_heads,
                     cfg.t_ff, cfg.max_speakers], np.int32)
    h = L.pksf_new(wp.encode(), dims.ctypes.data_as(C.POINTER(C.c_int32)))
    if not h:
        raise RuntimeError("pksf_new: " + L.pksf_last_error().decode())
    nfr = 1 + len(pcm) // 160
    nt_cap = nfr // 8 + 4
    pcm = np.ascontiguousarray(pcm, np.float32)
    feats = np.zeros((nfr + 4, e.mel_bins), np.float32)
    enc = np.zeros((nt_cap, e.d_model), np.float32)
    trans = np.zeros((nt_cap, cfg.t_hidden), np.float32)
    probs = np.zeros((nt_cap, cfg.max_speakers), np.float32)
    spk, st, en = np.zeros(4096, np.int32), np.zeros(4096, np.float32), np.zeros(4096, np.float32)
    nf, nt, ns = C.c_int(), C.c_int(), C.c_int()
    rc = L.pksf_run(h, pcm.ctypes.data, len(pcm), feats.ctypes.data, len(feats), C.byref(nf), enc.ctypes.data, trans.ctypes.data,
                    probs.ctypes.data, nt_cap, C.byref(nt), spk.ctypes.data, st.ctypes.data, en.ctypes.data, 4096, C.byref(ns))
    L.pksf_free(h)
    if rc != 0:
        raise RuntimeError("pksf_run: " + L.pksf_last_error().decode())
    T = nt.value
    return (feats[:nf.value].copy(), enc[:T].copy(), trans[:T].copy(), probs[:T].copy(),
            np.stack([spk[:ns.value].astype(np.float32), st[:ns.value], en[:ns.value]], axis=1))


def main():
    L = build_lib()
    out = {"margin": np.float32(MARGIN)}
    with tempfile.TemporaryDirectory() as td:
        for tag, cfg, lens, aseed in (("tiny", pkg.make_tiny_sortformer_config(), TINY_LENS, 100),
                                      ("s117m", pkg.make_sortformer_117m_config(), S117_LENS, 300)):
            clips = [synth.make_audio(n, aseed + i) for i, n in enumerate(lens)]
            for seed in range(16):
                W, m = SO.calibrated_weights(cfg, seed, clips, synth)
                print(tag, "seed", seed, "smallest |logit|", m, flush=True)
                if m >= MARGIN:
                    break
            else:
                raise RuntimeError("no seed clears the margin")
            out[tag + ".seed"] = np.int64(seed)
            out[tag + ".spk_bias"] = W["output_proj_.bias"]
            out[tag + ".min_abs_logit"] = np.float32(m)
            out[tag + ".lens"] = np.array(lens, np.int64)
            out[tag + ".audio_seed"] = np.int64(aseed)
            wp = os.path.join(td, tag + ".safetensors")
            synth.save_safetensors(wp, W)
            for i, c in enumerate(clips):
                f, e, t, p, segs = run_ref(L, wp, cfg, c)
                k = f"{tag}.u{i}."
                if keep(tag, i, "feats"):
                    out[k + "feats"] = f.astype(np.float16)
                if keep(tag, i, "enc"):
                    out[k + "enc"] = e.astype(np.float16)
                out[k + "trans"] = t.astype(np.float16)
                out[k + "probs"] = p
                out[k + "segs"] = segs
                print(tag, i, "frames", len(f), "T'", len(p), "segments", len(segs), flush=True)
    path = os.path.join(ROOT, "tests", "golden", "golden_sortformer_v1.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
