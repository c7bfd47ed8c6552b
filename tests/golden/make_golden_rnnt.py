"""Writes the RNN-T golden fixtures from the compiled reference (ParakeetRNNT, src/rnnt.cpp).

    python tests/golden/make_golden_rnnt.py tiny | 600m | 600m_long

tiny      -> golden_rnnt_v1.npz       tiny RNN-T: 4 clips, plus a "chatty" weight set (low blank bias) whose decodes
                                      hit the forced advance after max_symbols emissions on one frame
600m      -> golden_rnnt_600m_v1.npz  rnnt-600m preset (config.hpp:118-135): one 4 s clip
600m_long -> golden_rnnt_600m_long_v1.npz  rnnt-600m: one 30 s clip (every 4th encoder row; ~10 minutes on 8 cores)

The reference objects come from oracle/Makefile (`make -C oracle ref`); ref_rnnt.cpp (next to this file) is linked
against them into oracle/_ref/libpkref_rnnt.so.  Needs the reference sources (REF, default as in oracle/Makefile).
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
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import __graft_entry__ as ge  # noqa: E402
import oracle as O  # noqa: E402

pkg = ge.load_package()
from parakeet_cpp_b200 import synth  # noqa: E402

LIB = os.path.join(ROOT, "oracle", "_ref", "libpkref_rnnt.so")

TINY_SEED, TINY_BLANK_BIAS, CHATTY_SEED, CHATTY_BLANK_BIAS = 5, 7.0, 6, -1.0
TINY_CLIPS = [(16000, 301), (40000, 302), (27200, 303), (64000, 304)]
# rnnt-600m: blank bias 7 gives ~0.25 tokens per encoder frame, the rate of real speech (the default of 5 makes the
# synthetic 600m checkpoint emit ~7 tokens per frame, almost every frame ending in a forced advance)
M600_SEED, M600_BLANK_BIAS = 0, 7.0
M600_CLIP = (64000, 2000)
M600_LONG_CLIP = (480000, 2100)


def build_lib():
    mk = os.path.join(tempfile.mkdtemp(), "rnnt.mk")
    with open(mk, "w") as f:
        f.write("include Makefile\n"
                "$(OUT)/libpkref_rnnt.so: $(AX_OBJS) $(HWY_OBJS) $(PK_OBJS) $(OBJ)/ref_rnnt.o\n"
                "\t$(CXX) -shared -fopenmp -o $@ $^ -lpthread\n"
                f"$(OBJ)/ref_rnnt.o: {os.path.join(HERE, 'ref_rnnt.cpp')}\n"
                "\t@mkdir -p $(dir $@)\n"
                "\t$(CXX) $(PK_CXXFLAGS) $(INCS) -c $< -o $@\n")
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", mk, "-j8", "_ref/libpkref_rnnt.so"], check=True)
    L = C.CDLL(LIB)
    vp, i32p, f32p = C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_float)
    L.pkrnnt_last_error.restype = C.c_char_p
    L.pkrnnt_load.restype = vp
    L.pkrnnt_load.argtypes = [C.c_char_p, C.c_char_p, C.c_int, i32p]
    L.pkrnnt_free.argtypes = [vp]
    L.pkrnnt_encode_pcm.argtypes = [vp, f32p, C.c_int64, f32p, f32p]
    L.pkrnnt_greedy.argtypes = [vp, f32p, C.c_int, C.c_int, C.c_int, C.c_int, i32p, i32p, i32p, f32p]
    L.pkrnnt_detok.argtypes = [vp, i32p, C.c_int, C.c_char_p, C.c_int]
    L.pkrnnt_group_words.argtypes = [vp, i32p, i32p, i32p, f32p, C.c_int, C.c_char_p, C.c_int, f32p, f32p, f32p]
    return L


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class Ref:
    def __init__(self, L, cfg, weights_path, vocab_path, preset):
        self.L, self.cfg = L, cfg
        dims = np.array([cfg.mel_bins, cfg.sub_channels, cfg.d_model, cfg.n_layers, cfg.n_heads, cfg.ff, cfg.vocab,
                         cfg.pred_hidden, cfg.lstm_layers, cfg.joint_hidden], np.int32)
        self.h = L.pkrnnt_load(weights_path.encode(), vocab_path.encode(), preset, _p(dims, C.c_int32))
        if not self.h:
            raise RuntimeError(L.pkrnnt_last_error().decode())

    def encode(self, pcm):
        nf = 1 + len(pcm) // 160
        mel = np.zeros((nf, self.cfg.mel_bins), np.float32)
        enc = np.zeros((O.encoder_len(nf), self.cfg.d_model), np.float32)
        T = self.L.pkrnnt_encode_pcm(self.h, _p(pcm, C.c_float), len(pcm), _p(mel, C.c_float), _p(enc, C.c_float))
        assert T == enc.shape[0], self.L.pkrnnt_last_error()
        return mel, enc

    def greedy(self, enc, max_symbols=10):
        T = enc.shape[0]
        cap = max_symbols * T + 8
        ids, st, en = (np.zeros(cap, np.int32) for _ in range(3))
        cf = np.zeros(cap, np.float32)
        n = self.L.pkrnnt_greedy(self.h, _p(enc, C.c_float), T, enc.shape[1], max_symbols, cap, _p(ids, C.c_int32),
                                 _p(st, C.c_int32), _p(en, C.c_int32), _p(cf, C.c_float))
        assert n >= 0, self.L.pkrnnt_last_error()
        return np.stack([ids[:n], st[:n], en[:n]], axis=1), cf[:n]

    def detok(self, ids):
        ids = np.ascontiguousarray(ids, np.int32)
        buf = C.create_string_buffer(64 + 16 * max(len(ids), 1))
        self.L.pkrnnt_detok(self.h, _p(ids, C.c_int32), len(ids), buf, len(buf))
        return buf.value.decode()

    def words(self, tok, conf):
        n = len(tok)
        ids, st, en = (np.ascontiguousarray(tok[:, i], np.int32) for i in range(3))
        cf = np.ascontiguousarray(conf, np.float32)
        buf = C.create_string_buffer(64 + 64 * max(n, 1))
        ws, we, wc = (np.zeros(max(n, 1), np.float32) for _ in range(3))
        k = self.L.pkrnnt_group_words(self.h, _p(ids, C.c_int32), _p(st, C.c_int32), _p(en, C.c_int32), _p(cf, C.c_float), n, buf,
                                      len(buf), _p(ws, C.c_float), _p(we, C.c_float), _p(wc, C.c_float))
        return buf.value.decode().split("\n")[:k], np.stack([ws[:k], we[:k], wc[:k]], axis=1).astype(np.float32)

    def close(self):
        self.L.pkrnnt_free(self.h)


def run(L, out, tag, cfg, seed, clips, td, preset, blank_bias=None, enc_stride=1, full=True):
    W = synth.make_weights(cfg, seed=seed, blank_bias=blank_bias)
    wp = os.path.join(td, tag + ".safetensors")
    synth.save_safetensors(wp, W)
    del W
    pieces = synth.make_vocab(cfg.vocab - 1, seed=seed)
    vp = os.path.join(td, tag + ".vocab.txt")
    synth.save_vocab(vp, pieces)
    m = Ref(L, cfg, wp, vp, preset)
    for ci, (n, aseed) in enumerate(clips):
        k = f"{tag}.c{ci}."
        pcm = synth.make_audio(n, aseed)
        mel, enc = m.encode(pcm)
        tok, conf = m.greedy(enc)
        out[k + "n_samples"] = np.array([n, aseed], np.int64)
        out[k + "mel_stats"] = np.array([mel.mean(), mel.std(), np.abs(mel).max(), mel[::7, ::3].sum()], np.float64)
        out[k + "T"] = np.array(enc.shape[0], np.int32)
        out[k + "enc"] = enc[::enc_stride]
        out[k + "tok"], out[k + "conf"] = tok, conf
        # frames on which the decode emitted max_symbols tokens (the reference's forced advance)
        per_frame = np.bincount(tok[:, 1], minlength=enc.shape[0]) if len(tok) else np.zeros(enc.shape[0], np.int64)
        out[k + "forced_frames"] = np.array(int((per_frame >= 10).sum()), np.int32)
        if full:
            out[k + "text"] = np.frombuffer(m.detok(tok[:, 0]).encode(), np.uint8)
            words, times = m.words(tok, conf)
            out[k + "words"] = np.frombuffer("\n".join(words).encode(), np.uint8)
            out[k + "word_times"] = times.reshape(-1, 3)
        print(tag, ci, "T", enc.shape[0], "tokens", len(tok), "forced frames", int(out[k + "forced_frames"]), flush=True)
    m.close()


def main(which):
    L = build_lib()
    out = {}
    with tempfile.TemporaryDirectory() as td:
        if which == "tiny":
            cfg = pkg.make_tiny_rnnt_config()
            run(L, out, "tiny", cfg, TINY_SEED, TINY_CLIPS, td, 0, blank_bias=TINY_BLANK_BIAS)
            run(L, out, "chatty", cfg, CHATTY_SEED, TINY_CLIPS, td, 0, blank_bias=CHATTY_BLANK_BIAS)
            name = "golden_rnnt_v1.npz"
        elif which == "600m":
            run(L, out, "m600", pkg.make_rnnt_600m_config(), M600_SEED, [M600_CLIP], td, 2, blank_bias=M600_BLANK_BIAS)
            name = "golden_rnnt_600m_v1.npz"
        elif which == "600m_long":
            run(L, out, "m600l", pkg.make_rnnt_600m_config(), M600_SEED, [M600_LONG_CLIP], td, 2,
                blank_bias=M600_BLANK_BIAS, enc_stride=4, full=False)
            name = "golden_rnnt_600m_long_v1.npz"
        else:
            raise SystemExit(__doc__)
    path = os.path.join(HERE, name)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "tiny")
