"""Writes tests/golden/golden_nemotron_v1.npz from the compiled reference's Nemotron streaming model (ParakeetNemotron,
src/nemotron.cpp), chunk by chunk through the steps of NemotronTranscriber::transcribe_chunk with blank = vocab - 1.

    python tests/golden/make_golden_nemotron.py

Recorded:
  tnemo    the tiny Nemotron shape (head_dim 128, two LSTM layers; tests/nemotron_oracle.py) on the ragged
           STREAM_SCHEDULE of make_golden.py;
  nemo600  the nemotron-600m preset with seed-0 synthetic weights on 14 x 2560 samples at latency 0: per chunk the new
           mel frames, the encoder rows, tokens, frames and confidences, and the text at the end.
The 600m stream is run again at latencies 1, 6 and 13: the reference's outputs must be byte-identical to latency 0 (its
bounded-context mask is inert on the CPU), and only their digests are stored.  The numpy oracle runs FIRST on every model:
the reference would hang on a livelocking decode.

The reference objects come from oracle/Makefile (`make -C oracle ref`); ref_nemotron.cpp (next to this file) and
src/nemotron.cpp are linked against them into oracle/_ref/libpkref_nemotron.so.  Needs the reference sources (REF, default
as in oracle/Makefile).  A few minutes on 8 cores.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import __graft_entry__ as ge  # noqa: E402
import oracle as O  # noqa: E402
import nemotron_oracle as NO  # noqa: E402

ge.load_package()
from parakeet_cpp_b200 import synth  # noqa: E402

LIB = os.path.join(ROOT, "oracle", "_ref", "libpkref_nemotron.so")
STREAM_SCHEDULE = [2560, 2560, 2560, 1000, 4000, 2560, 2560, 2560, 2560, 5000, 2560, 2560, 2560, 2560, 2560, 2560, 2560]
LATENCIES = (1, 6, 13)


def build_lib():
    mk = os.path.join(tempfile.mkdtemp(), "nemotron.mk")
    with open(mk, "w") as f:
        f.write("include Makefile\n"
                "$(OUT)/libpkref_nemotron.so: $(AX_OBJS) $(HWY_OBJS) $(PK_OBJS) $(OBJ)/pk/src/nemotron.cpp.o $(OBJ)/ref_nemotron.o\n"
                "\t$(CXX) -shared -fopenmp -o $@ $^ -lpthread\n"
                f"$(OBJ)/ref_nemotron.o: {os.path.join(HERE, 'ref_nemotron.cpp')}\n"
                "\t@mkdir -p $(dir $@)\n"
                "\t$(CXX) $(PK_CXXFLAGS) $(INCS) -c $< -o $@\n")
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", mk, "-j8", "_ref/libpkref_nemotron.so"], check=True)
    L = C.CDLL(LIB)
    vp = C.c_void_p
    L.pknemo_last_error.restype = C.c_char_p
    L.pknemo_new.restype = vp
    L.pknemo_new.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_int32)]
    L.pknemo_free.argtypes = [vp]
    L.pknemo_chunk.argtypes = [vp, vp, C.c_int, vp, C.c_int, vp, vp, C.c_int, vp, vp, vp, C.c_int, vp]
    return L


class RefNemotron:
    """One stream through the reference (ref_nemotron.cpp)."""

    def __init__(self, L, weights_path, cfg):
        self.L, self.cfg = L, cfg
        dims = np.array([cfg.mel_bins, cfg.sub_channels, cfg.d_model, cfg.n_layers, cfg.n_heads, cfg.ff, cfg.vocab,
                         cfg.pred_hidden, cfg.lstm_layers, cfg.joint_hidden, cfg.att_context_left], np.int32)
        self.h = L.pknemo_new(weights_path.encode(), cfg.att_context_right, dims.ctypes.data_as(C.POINTER(C.c_int32)))
        if not self.h:
            raise RuntimeError("pknemo_new: " + L.pknemo_last_error().decode())

    def close(self):
        if self.h:
            self.L.pknemo_free(self.h)
            self.h = None

    def chunk(self, pcm):
        """-> (feats (n, mel) | None, enc (C, d) | None, [(id, start, end, conf), ...])"""
        pcm = np.ascontiguousarray(pcm, np.float32)
        cap_f, cap_e, cap_t = 4 + len(pcm) // 160, 4 + len(pcm) // 1280, 4096
        feats = np.zeros((cap_f, self.cfg.mel_bins), np.float32)
        enc = np.zeros((cap_e, self.cfg.d_model), np.float32)
        tok = np.zeros((cap_t, 3), np.int32)
        conf = np.zeros(cap_t, np.float32)
        nf, ne, nt = C.c_int(), C.c_int(), C.c_int()
        rc = self.L.pknemo_chunk(self.h, pcm.ctypes.data, len(pcm), feats.ctypes.data, cap_f, C.byref(nf), enc.ctypes.data, cap_e,
                                 C.byref(ne), tok.ctypes.data, conf.ctypes.data, cap_t, C.byref(nt))
        if rc != 0:
            raise RuntimeError("pknemo_chunk: " + self.L.pknemo_last_error().decode())
        toks = [(int(tok[i, 0]), int(tok[i, 1]), int(tok[i, 2]), float(conf[i])) for i in range(nt.value)]
        return (feats[:nf.value].copy() if nf.value else None, enc[:ne.value].copy() if ne.value else None, toks)


def toks_arr(toks):
    return np.array([[t[0], t[1], t[2]] for t in toks], np.int32).reshape(-1, 3), np.array([t[3] for t in toks], np.float32)


def stream_digest(chunks):
    """sha256 over every chunk's feats, encoder rows, tokens and confidences, in order."""
    h = hashlib.sha256()
    for f, e, toks in chunks:
        for a in (f, e):
            h.update(b"-" if a is None else np.ascontiguousarray(a, np.float32).tobytes())
        t, c = toks_arr(toks)
        h.update(t.tobytes())
        h.update(c.tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def main():
    L = build_lib()
    out = {}
    with tempfile.TemporaryDirectory() as td:
        for tag, ocfg, wseed, aseed, sched in (("tnemo", NO.make_tiny_nemotron_config(), 5, 78, STREAM_SCHEDULE),
                                               ("nemo600", NO.make_nemotron_600m_config(0), 0, 1400, [2560] * 14)):
            W = synth.make_weights(ocfg, seed=wseed)
            pcm = synth.make_audio(sum(sched), aseed)
            pre, cache, st = O.StreamingPreprocessor(ocfg.mel_bins), O.StreamEncoderCache(ocfg.n_layers), O.StreamDecodeState(ocfg)
            pos = 0
            for n in sched:                                   # raises RuntimeError on a livelock
                f = pre.process_chunk(pcm[pos:pos + n]); pos += n
                e = O.stream_encoder_chunk(W, f, cache, ocfg) if f is not None else None
                if e is not None:
                    O.stream_decode_chunk(W, e, st, ocfg, max_steps=5000)
            wp = os.path.join(td, tag + ".safetensors")
            synth.save_safetensors(wp, W)
            del W

            def run(cfg):
                rs = RefNemotron(L, wp, cfg)
                p, res = 0, []
                for n in sched:
                    res.append(rs.chunk(pcm[p:p + n])); p += n
                rs.close()
                return res

            res = run(ocfg)
            out[tag + ".schedule"] = np.array(sched, np.int64)
            out[tag + ".seeds"] = np.array([wseed, aseed], np.int64)
            ids = []
            for ci, (f, e, toks) in enumerate(res):
                k = f"{tag}.k{ci}."
                out[k + "feats"] = f if f is not None else np.zeros((0, ocfg.mel_bins), np.float32)
                out[k + "enc"] = e if e is not None else np.zeros((0, ocfg.d_model), np.float32)
                out[k + "tok"], out[k + "conf"] = toks_arr(toks)
                ids += [t[0] for t in toks]
            pieces = synth.make_vocab(ocfg.vocab - 1, seed=wseed)
            out[tag + ".text"] = np.frombuffer(O.detokenize(ids, pieces).encode(), np.uint8)
            out[tag + ".digest"] = stream_digest(res)
            print(tag, "chunks", len(sched), "tokens", len(ids), flush=True)
            if tag == "nemo600":
                for lat in LATENCIES:
                    d = stream_digest(run(NO.make_nemotron_600m_config(lat)))
                    assert np.array_equal(d, out[tag + ".digest"]), f"reference output at latency {lat} differs from latency 0"
                    out[f"{tag}.digest_latency{lat}"] = d
                    print(tag, "latency", lat, "identical to latency 0", flush=True)
    path = os.path.join(ROOT, "tests", "golden", "golden_nemotron_v1.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
