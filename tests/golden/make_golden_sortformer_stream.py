"""Writes tests/golden/golden_sortformer_stream_v1.npz from the compiled reference's streaming Sortformer
(Sortformer::diarize_chunk, AOSCCache; src/sortformer.cpp) through tests/golden/ref_sortformer_stream.cpp.

    python tests/golden/make_golden_sortformer_stream.py

Recorded per step and stream: the number of encoder rows C (0 where diarize_chunk returns {}), the frame base, the
activities (float32), the segments diarize_chunk returns (chunk-local times) and the AOSC arrival order after the call;
the NEST encoder rows (float16) where keep_enc() says so, to keep the file near 1 MB.
  tiny    the test-only tiny Sortformer on TINY_SCHED (tests/test_sortformer_stream.py): several streams with ragged
          chunk sizes, among them chunks that yield no encoder frame and chunks that leave 1-7 mel frames queued;
  s117m   sortformer-117m on one 30 s clip, at 2560 and at 16000 samples per chunk (sets c2560 and c16000).
Weights: synth.make_sortformer_weights(seed) with output_proj_'s bias calibrated on the STREAMING logits of these
schedules (sortformer_stream_oracle.calibrated_weights); the first seed whose smallest |logit| is at least MARGIN is
taken.  The numpy oracle runs first (it picks the seed); the reference then loads every module with strict = true.

The reference objects come from oracle/Makefile (`make -C oracle ref`); the harness and src/sortformer.cpp +
src/transformer.cpp are linked against them into oracle/_ref/libpkref_sortformer_stream.so.  Needs the reference sources.
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
import sortformer_stream_oracle as SSO  # noqa: E402
from test_sortformer_stream import MARGIN, S117_CHUNKS, S117_LEN, TINY_SCHED, tiny_clips  # noqa: E402

pkg = ge.load_package()
from parakeet_cpp_b200 import synth  # noqa: E402

LIB = os.path.join(ROOT, "oracle", "_ref", "libpkref_sortformer_stream.so")
S117_ENC_STEPS = 6          # encoder rows stored for the first steps of each sortformer-117m set


def keep_enc(tag, k):
    return tag == "tiny" or k < S117_ENC_STEPS


def build_lib():
    mk = os.path.join(tempfile.mkdtemp(), "sortformer_stream.mk")
    with open(mk, "w") as f:
        f.write("include Makefile\n"
                "$(OUT)/libpkref_sortformer_stream.so: $(AX_OBJS) $(HWY_OBJS) $(PK_OBJS) $(OBJ)/pk/src/sortformer.cpp.o "
                "$(OBJ)/pk/src/transformer.cpp.o $(OBJ)/ref_sortformer_stream.o\n"
                "\t$(CXX) -shared -fopenmp -o $@ $^ -lpthread\n"
                f"$(OBJ)/ref_sortformer_stream.o: {os.path.join(HERE, 'ref_sortformer_stream.cpp')}\n"
                "\t@mkdir -p $(dir $@)\n"
                "\t$(CXX) $(PK_CXXFLAGS) $(INCS) -c $< -o $@\n")
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", mk, "-j8", "_ref/libpkref_sortformer_stream.so"], check=True)
    L = C.CDLL(LIB)
    L.pkss_last_error.restype = C.c_char_p
    L.pkss_new.restype = C.c_void_p
    L.pkss_new.argtypes = [C.c_char_p, C.POINTER(C.c_int32)]
    L.pkss_free.argtypes = [C.c_void_p]
    L.pkss_stream_new.restype = C.c_void_p
    L.pkss_stream_new.argtypes = [C.c_void_p]
    L.pkss_stream_free.argtypes = [C.c_void_p]
    L.pkss_chunk.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p] + \
        [C.c_void_p] * 3 + [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def run_ref(L, wp, cfg, clips, sched):
    """-> steps[k][s] = dict(C, probs, enc, segs, order) of the compiled reference."""
    e = cfg.encoder
    dims = np.array([e.mel_bins, e.sub_channels, e.d_model, e.n_layers, e.n_heads, e.ff, cfg.t_hidden, cfg.t_layers, cfg.t_heads,
                     cfg.t_ff, cfg.max_speakers, 70], np.int32)
    h = L.pkss_new(wp.encode(), dims.ctypes.data_as(C.POINTER(C.c_int32)))
    if not h:
        raise RuntimeError("pkss_new: " + L.pkss_last_error().decode())
    streams = [L.pkss_stream_new(h) for _ in clips]
    pos = [0] * len(clips)
    steps = []
    try:
        for k in range(len(sched[0])):
            row = []
            for s, c in enumerate(clips):
                n = sched[s][k]
                pcm = np.ascontiguousarray(c[pos[s]:pos[s] + n], np.float32)
                pos[s] += n
                if n == 0:                      # no input for this stream this step: diarize_chunk is not called
                    row.append(dict(C=0, probs=np.zeros((0, cfg.max_speakers), np.float32), enc=np.zeros((0, e.d_model), np.float32),
                                    segs=np.zeros((0, 3), np.float32), order=None))
                    continue
                cap = n // 1280 + 4
                enc = np.zeros((cap, e.d_model), np.float32)
                probs = np.zeros((cap, cfg.max_speakers), np.float32)
                spk, st, en = np.zeros(256, np.int32), np.zeros(256, np.float32), np.zeros(256, np.float32)
                order = np.zeros(64, np.int32)
                nt, ns, no = C.c_int(), C.c_int(), C.c_int()
                rc = L.pkss_chunk(h, streams[s], pcm.ctypes.data, n, enc.ctypes.data, probs.ctypes.data, cap, C.byref(nt), spk.ctypes.data,
                                  st.ctypes.data, en.ctypes.data, 256, C.byref(ns), order.ctypes.data, C.byref(no))
                if rc != 0:
                    raise RuntimeError("pkss_chunk: " + L.pkss_last_error().decode())
                row.append(dict(C=nt.value, probs=probs[:nt.value].copy(), enc=enc[:nt.value].copy(),
                                segs=np.stack([spk[:ns.value].astype(np.float32), st[:ns.value], en[:ns.value]], axis=1),
                                order=order[:no.value].copy()))
            steps.append(row)
    finally:
        for st_ in streams:
            L.pkss_stream_free(st_)
        L.pkss_free(h)
    # an empty chunk leaves the order as it was
    for s in range(len(clips)):
        last = np.zeros(0, np.int32)
        for row in steps:
            if row[s]["order"] is None:
                row[s]["order"] = last
            last = row[s]["order"]
    return steps


def main():
    L = build_lib()
    out = {"margin": np.float32(MARGIN)}
    tiny_cfg, s117_cfg = pkg.make_tiny_sortformer_config(), pkg.make_sortformer_117m_config()
    clip117 = synth.make_audio(S117_LEN, 500)
    sets = [("tiny", tiny_cfg, [(tiny_clips(synth), TINY_SCHED)])]
    sets.append(("s117m", s117_cfg, [([clip117], [SSO.split(S117_LEN, ch)]) for ch in S117_CHUNKS]))
    with tempfile.TemporaryDirectory() as td:
        for tag, cfg, runs in sets:
            for seed in range(16):
                W, m = SSO.calibrated_weights(cfg, seed, runs, synth)
                print(tag, "seed", seed, "smallest |logit|", m, flush=True)
                if m >= MARGIN:
                    break
            else:
                raise RuntimeError("no seed clears the margin")
            out[tag + ".seed"] = np.int64(seed)
            out[tag + ".spk_bias"] = W["output_proj_.bias"]
            out[tag + ".min_abs_logit"] = np.float32(m)
            wp = os.path.join(td, tag + ".safetensors")
            synth.save_safetensors(wp, W)
            for clips, sched in runs:
                sub = tag if tag == "tiny" else f"{tag}.c{sched[0][0]}"
                steps = run_ref(L, wp, cfg, clips, sched)
                for k, row in enumerate(steps):
                    for s, r in enumerate(row):
                        key = f"{sub}.k{k}.s{s}."
                        out[key + "C"] = np.int32(r["C"])
                        out[key + "probs"] = r["probs"]
                        out[key + "segs"] = r["segs"]
                        out[key + "order"] = r["order"].astype(np.int32)
                        if keep_enc(tag, k) and r["C"]:
                            out[key + "enc"] = r["enc"].astype(np.float16)
                print(sub, "steps", len(steps), "rows", sum(r["C"] for row in steps for r in row), flush=True)
    path = os.path.join(ROOT, "tests", "golden", "golden_sortformer_stream_v1.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
