"""RNN-T model family (ParakeetRNNT, reference src/rnnt.cpp): the rnnt-600m preset and the batched RNN-T greedy decode
in the persistent decode kernel (csrc/tdt.cu, n_dur == 0), against fixtures written by the compiled reference
(tests/golden/make_golden_rnnt.py) and the numpy restatement in tests/rnnt_oracle.py."""
import ctypes as C
import dataclasses
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, HERE)
import rnnt_oracle as RO  # noqa: E402

# weight sets of golden_rnnt_v1.npz: (tag, seed, blank bias); "chatty" hits the forced advance on many frames
SETS = [("tiny", 5, 7.0), ("chatty", 6, -1.0)]
MATH = {"bf16x3": 0, "fp32": 2}
BENCH_LINE = os.path.join(GOLD, "bench", "h100_rnnt600m_16x30s.json")


def _load(name):
    with np.load(os.path.join(GOLD, name), allow_pickle=False) as f:
        return {k: f[k] for k in f.files}


@pytest.fixture(scope="module")
def g():
    return _load("golden_rnnt_v1.npz")


def _clips(g, tag):
    return sorted({k.split(".")[1] for k in g if k.startswith(tag + ".")})


class RnntModel:
    def __init__(self, tmpdir, pkg, synth, tag, seed, blank_bias):
        self.cfg, self.ocfg = pkg.make_tiny_rnnt_config(), RO.make_tiny_rnnt_config()
        self.W = synth.make_weights(self.cfg, seed=seed, blank_bias=blank_bias)
        self.weights_path = os.path.join(tmpdir, f"{tag}.safetensors")
        synth.save_safetensors(self.weights_path, self.W)
        self.pieces = synth.make_vocab(self.cfg.vocab - 1, seed=seed)
        self.vocab_path = os.path.join(tmpdir, f"{tag}.vocab.txt")
        synth.save_vocab(self.vocab_path, self.pieces)


@pytest.fixture(scope="module")
def models(tmp_path_factory, pkg, synth):
    td = str(tmp_path_factory.mktemp("rnnt"))
    return {tag: RnntModel(td, pkg, synth, tag, seed, bb) for tag, seed, bb in SETS}


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", [s[0] for s in SETS])
def test_oracle_reproduces_reference_rnnt_decodes(g, models, tag):
    """rnnt_greedy_decode restated in numpy gives the reference's tokens, frames and confidences on the reference's
    encoder output; the chatty set really contains frames with max_symbols = 10 emissions (the forced advance)."""
    m = models[tag]
    forced = 0
    for c in _clips(g, tag):
        k = f"{tag}.{c}."
        got = RO.rnnt_greedy_decode(m.W, g[k + "enc"], m.ocfg, with_timestamps=True)
        want = g[k + "tok"]
        assert [t[:3] for t in got] == [tuple(int(v) for v in r) for r in want], k
        np.testing.assert_allclose([t[3] for t in got], g[k + "conf"], rtol=1e-4)
        per_frame = np.bincount(want[:, 1], minlength=int(g[k + "T"])) if len(want) else np.zeros(1)
        assert int((per_frame == 10).sum()) == int(g[k + "forced_frames"])
        assert per_frame.max() <= 10
        forced += int(g[k + "forced_frames"])
    if tag == "chatty":
        assert forced >= 10


def test_rnnt_preset_matches_reference_config(pkg):
    L = pkg.load_library()
    c = pkg.engine._PkConfig()
    L.pk_config_rnnt_600m(C.byref(c))           # config.hpp:119-135
    assert (c.mel_bins, c.sub_channels, c.d_model, c.n_layers, c.ff, c.n_heads, c.conv_kernel) == (80, 256, 1024, 24, 4096, 8, 9)
    assert (c.vocab, c.pred_hidden, c.joint_hidden, c.lstm_layers) == (1025, 640, 640, 2)
    assert (c.n_durations, c.has_ctc, c.joint_prefix_tdt, c.max_symbols) == (0, 0, 0, 10)
    assert (c.max_batch, c.max_samples) == (16, 480000)
    py = pkg.make_rnnt_600m_config().to_c()
    assert bytes(py)[:C.sizeof(c) - 4] == bytes(c)[:C.sizeof(c) - 4]    # all but `math`
    o = RO.make_rnnt_600m_config()
    assert (o.mel_bins, o.d_model, o.n_layers, o.vocab, o.lstm_layers, o.durations) == (80, 1024, 24, 1025, 2, ())


def test_synth_rnnt_checkpoint_has_the_parakeet_rnnt_key_set(pkg, synth):
    """ParakeetRNNT (rnnt.cpp:48-52) registers encoder_, prediction_ and joint_ {enc_proj_, pred_proj_, out_proj_}: the
    TDT model's keys without the label / duration heads, plus out_proj_."""
    r = {n: s for n, s, _ in synth.tensor_specs(pkg.make_rnnt_600m_config())}
    t = {n: s for n, s, _ in synth.tensor_specs(pkg.make_rnnt_600m_config(durations=(0, 1, 2, 3, 4)))}
    heads = {"joint_.label_proj_.weight", "joint_.label_proj_.bias", "joint_.duration_proj_.weight", "joint_.duration_proj_.bias"}
    assert heads <= set(t)
    assert set(r) == (set(t) - heads) | {"joint_.out_proj_.weight", "joint_.out_proj_.bias"}
    assert r["joint_.out_proj_.weight"] == (1025, 640) and r["joint_.out_proj_.bias"] == (1025,)
    assert not any(n.startswith("ctc_decoder_") or n.startswith("tdt_joint_") for n in r)
    W = synth.make_weights(pkg.make_tiny_rnnt_config(), seed=1)
    assert W["joint_.out_proj_.bias"][-1] == np.float32(2.5)       # blank bias on the last row


def test_cpp_shim_rnnt_transcriber_compiles(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(HERE, "cpp_rnnt_check.cpp")], check=True)


def test_rnnt_bench_line_has_the_measurement_keys():
    with open(BENCH_LINE) as f:
        r = json.loads(f.readline())
    for k in ("config", "rtfx_device", "rtfx_e2e", "ms_per_step", "steps", "warmup", "n_clips", "clip_s", "gpu_launches",
              "per_class_ms", "encoder_gflop_per_clip", "gpu_name", "power_limit_w", "sm_clock_mhz"):
        assert k in r, k
    assert r["config"] == "rnnt-600m-16x30s" and r["n_clips"] == 16 and r["steps"] >= 20 and r["warmup"] >= 3
    assert r["rtfx_device"] > 0 and r["ms_per_step"] > 0
    assert r["clip0_tokens_match_reference"] is True          # clip 0 is the 30 s clip of golden_rnnt_600m_long_v1.npz


# ------------------------------------------------------------------ GPU
def _tt(toks):
    return [(t.token_id, t.start_frame, t.end_frame) for t in toks]


@pytest.fixture(scope="module", params=list(MATH))
def engines(request, pkg, models):
    es = {tag: pkg.Engine(dataclasses.replace(m.cfg, math=MATH[request.param]), m.weights_path, 0) for tag, m in models.items()}
    yield es
    for e in es.values():
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("tag", [s[0] for s in SETS])
def test_tiny_rnnt_matches_reference(pkg, synth, g, models, engines, tag):
    e = engines[tag]
    clips = _clips(g, tag)
    encs = [g[f"{tag}.{c}.enc"] for c in clips]
    # decode-only on the reference's encoder output: tokens and frames exact, confidences 1e-4
    got = e.decode(encs, pkg.Decoder.RNNT)
    for c, toks in zip(clips, got):
        k = f"{tag}.{c}."
        assert _tt(toks) == [tuple(int(v) for v in r) for r in g[k + "tok"]], k
        np.testing.assert_allclose([t.confidence for t in toks], g[k + "conf"], rtol=1e-4)
    assert e.truncated_count() == 0
    # the whole path from PCM
    pcms = [synth.make_audio(*(int(v) for v in g[f"{tag}.{c}.n_samples"])) for c in clips]
    got = e.transcribe_batch(pcms, pkg.Decoder.RNNT)
    for c, toks in zip(clips, got):
        assert _tt(toks) == [tuple(int(v) for v in r) for r in g[f"{tag}.{c}.tok"]], c
    assert e.truncated_count() == 0


@pytest.mark.gpu
def test_rnnt_lock_step_batches_equal_single_runs(pkg, g, models):
    """A ragged batch and a batch of 70 utterances (two 64-utterance chunks of the decode kernel) give what
    single-utterance decodes give."""
    m = models["chatty"]
    encs = [g[f"chatty.{c}.enc"] for c in _clips(g, "chatty")] + [g[f"tiny.{c}.enc"] for c in _clips(g, "tiny")]
    e = pkg.Engine(dataclasses.replace(m.cfg, max_batch=72), m.weights_path, 0)
    try:
        single = [_tt(e.decode([x], pkg.Decoder.RNNT)[0]) for x in encs]
        assert [_tt(t) for t in e.decode(encs, pkg.Decoder.RNNT)] == single
        big = [encs[i % len(encs)][: max(1, len(encs[i % len(encs)]) - i // len(encs))] for i in range(70)]
        got = e.decode(big, pkg.Decoder.RNNT)
        assert [_tt(t) for t in got] == [_tt(e.decode([x], pkg.Decoder.RNNT)[0]) for x in big]
        assert e.truncated_count() == 0
    finally:
        e.close()


@pytest.mark.gpu
def test_rnnt_invalid_combinations_are_refused(pkg, g, models, engines, tiny):
    e = engines["tiny"]
    enc = [g["tiny.c0.enc"]]
    with pytest.raises(RuntimeError, match="PK_DECODER_TDT on an RNN-T model"):
        e.decode(enc, pkg.Decoder.TDT)
    with pytest.raises(RuntimeError, match="no CTC head"):
        e.decode(enc, pkg.Decoder.CTC)
    with pytest.raises(RuntimeError, match="pk_set_boost"):
        e.set_boost([[3, 4]])
    with pytest.raises(RuntimeError, match="pk_stream_open"):
        e.stream_open(1, 2560)
    assert len(e.decode(enc, pkg.Decoder.RNNT)) == 1        # the engine is still usable
    # PK_DECODER_RNNT on a TDT model
    et = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    try:
        with pytest.raises(RuntimeError, match="PK_DECODER_RNNT on a TDT model"):
            et.decode([np.zeros((5, tiny.cfg.d_model), np.float32)], pkg.Decoder.RNNT)
    finally:
        et.close()
    # the model contract of n_durations = 0
    m = models["tiny"]
    for bad in (dict(joint_prefix="tdt_joint_."), dict(has_ctc=True), dict(max_symbols=0), dict(max_symbols=65)):
        with pytest.raises(RuntimeError, match="pk_engine_create"):
            pkg.Engine(dataclasses.replace(m.cfg, **bad), m.weights_path, 0)


@pytest.mark.gpu
def test_rnnt_job_with_world1_allgather_equals_direct_decodes(pkg, synth, g, models):
    m = models["tiny"]
    e = pkg.Engine(m.cfg, m.weights_path, 0)
    try:
        pcms = [synth.make_audio(*(int(v) for v in g[f"{t}.{c}.n_samples"])) for t in ("tiny", "chatty") for c in _clips(g, t)]
        direct = [[x.token_id for x in toks] for toks in e.transcribe_batch(pcms[:8], pkg.Decoder.RNNT)]
        from parakeet_cpp_b200.engine import _pack
        buf, off = _pack(pcms)
        e.job_stage(buf, off)
        e.comm_init_rank(e.nccl_unique_id(), 0, 1)
        e.job_begin(10, 1)
        for first, n in ((0, 5), (5, 3)):
            e.job_select(first, n)
            e.run_staged(pkg.Decoder.RNNT)
            e.job_append()
        e.allgather_tokens()
        rows = e.job_fetch(10, gathered=True)
        assert rows.shape[1] == 1 + 10 * e.Tmax + 8
        for i in range(8):
            assert rows[i, 1:1 + rows[i, 0]].tolist() == direct[i]
        assert rows[8, 0] == 0 and rows[9, 0] == 0
    finally:
        e.close()


@pytest.mark.gpu
def test_rnnt_transcriber_text_and_words_python_and_cpp(pkg, synth, g, models, tmp_path):
    import struct
    m = models["tiny"]
    t = pkg.Transcriber(m.weights_path, m.vocab_path, m.cfg)
    k = "tiny.c3."
    pcm = synth.make_audio(*(int(v) for v in g[k + "n_samples"]))
    r = t.transcribe(pcm, timestamps=True)
    assert r.text == g[k + "text"].tobytes().decode()
    assert [w.word for w in r.word_timestamps] == g[k + "words"].tobytes().decode().split("\n")
    np.testing.assert_allclose([[w.start, w.end] for w in r.word_timestamps], g[k + "word_times"][:, :2], rtol=0, atol=1e-6)
    np.testing.assert_allclose([w.confidence for w in r.word_timestamps], g[k + "word_times"][:, 2], rtol=1e-4)
    t.engine.close()
    # C++ RNNTTranscriber
    exe = str(tmp_path / "cpp_rnnt_check")
    libdir = os.path.dirname(pkg.lib_path())
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), os.path.join(HERE, "cpp_rnnt_check.cpp"),
                    "-L" + libdir, "-lparakeet_b200", "-Wl,-rpath," + libdir, "-o", exe], check=True)
    i16 = np.round(pcm * 32768.0).astype(np.int16)
    wav = str(tmp_path / "a.wav")
    with open(wav, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + 2 * len(i16)) + b"WAVEfmt " +
                struct.pack("<IHHIIHH", 16, 1, 1, 16000, 32000, 2, 16) + b"data" + struct.pack("<I", 2 * len(i16)))
        f.write(i16.tobytes())
    out = subprocess.run([exe, m.weights_path, m.vocab_path, wav], capture_output=True, text=True, env=dict(os.environ))
    assert out.returncode == 0, out.stderr
    lines = dict(ln.split(" ", 1) if " " in ln else (ln, "") for ln in out.stdout.splitlines())
    assert lines["TOK"].split() == [f"{a}:{b}:{c}" for a, b, c in g[k + "tok"]]
    assert lines["TEXT"] == g[k + "text"].tobytes().decode()
    assert lines["WORDS"].split() == g[k + "words"].tobytes().decode().split("\n")
    assert "BOOST_THROWS" in lines


# ------------------------------------------------------------------ rnnt-600m preset
M600_BLANK_BIAS = 7.0     # the rnnt-600m fixtures' checkpoint: ~0.25 tokens per encoder frame (make_golden_rnnt.py)


@pytest.fixture(scope="module")
def m600(tmp_path_factory, pkg, synth):
    """Two synthetic rnnt-600m checkpoints that differ only in the blank bias: "ref" (the reference fixtures') and
    "chatty" (the default bias of 5: ~7 tokens per frame, most frames end in the forced advance)."""
    W = synth.make_weights(pkg.make_rnnt_600m_config(), seed=0, blank_bias=M600_BLANK_BIAS)
    d = tmp_path_factory.mktemp("rnnt600")
    paths = {"ref": str(d / "rnnt600.safetensors"), "chatty": str(d / "rnnt600_chatty.safetensors")}
    synth.save_safetensors(paths["ref"], W)
    W["joint_.out_proj_.bias"][-1] = np.float32(5.0)
    synth.save_safetensors(paths["chatty"], W)
    del W
    return paths


@pytest.mark.gpu
def test_rnnt_600m_matches_reference(pkg, synth, m600):
    g6 = _load("golden_rnnt_600m_v1.npz")
    k = "m600.c0."
    pcm = synth.make_audio(*(int(v) for v in g6[k + "n_samples"]))
    e = pkg.Engine(pkg.make_rnnt_600m_config(max_batch=2, max_samples=80000), m600["ref"], 0)
    try:
        feats = e.mel([pcm])
        enc = e.encode(feats)[0]
        ref = g6[k + "enc"]
        assert enc.shape == ref.shape
        assert np.abs(enc - ref).max() / np.abs(ref).max() < 1e-3
        toks = e.transcribe_batch([pcm], pkg.Decoder.RNNT)[0]
        assert _tt(toks) == [tuple(int(v) for v in r) for r in g6[k + "tok"]]
        assert len(toks) > 0
    finally:
        e.close()


def _ragged_30s(synth, first):
    """16 clips of 30 s down to 15 s (the preset's full capacity), `first` in row 0."""
    return [first] + [synth.make_audio(480000 - 16000 * i, 2200 + i) for i in range(1, 16)]


@pytest.mark.gpu
def test_rnnt_600m_30s_clip_in_full_batch_matches_reference(pkg, synth, m600):
    """The 30 s clip the compiled reference decoded (make_golden_rnnt.py 600m_long, T' = 376) as row 0 of a ragged
    batch of 16: encoder rows within 1e-3 and tokens / frames equal to the reference's."""
    gl = _load("golden_rnnt_600m_long_v1.npz")
    k = "m600l.c0."
    e = pkg.Engine(pkg.make_rnnt_600m_config(), m600["ref"], 0)
    try:
        pcms = _ragged_30s(synth, synth.make_audio(*(int(v) for v in gl[k + "n_samples"])))
        got = e.transcribe_batch(pcms, pkg.Decoder.RNNT)
        assert len(gl[k + "tok"]) > 0
        assert _tt(got[0]) == [tuple(int(v) for v in r) for r in gl[k + "tok"]]
        np.testing.assert_allclose([t.confidence for t in got[0]], gl[k + "conf"], rtol=1e-3)
        enc = e.encode(e.mel(pcms[:1]))[0]
        assert enc.shape[0] == int(gl[k + "T"]) == 376
        ref = gl[k + "enc"]
        assert np.abs(enc[::4] - ref).max() / np.abs(ref).max() < 1e-3
        assert e.truncated_count() == 0
    finally:
        e.close()


@pytest.mark.gpu
def test_rnnt_600m_full_capacity_batch_equals_single_decodes(pkg, synth, m600):
    """The largest shape the preset accepts (16 utterances, T' up to 376, 2 LSTM layers, 1025-row head) with a checkpoint
    that emits several tokens on most frames: every row of the lock-step batch equals its single-utterance decode, the
    forced advance bounds every frame, and no hypothesis reaches the token capacity (10 T'max + 8 = 3768)."""
    e = pkg.Engine(pkg.make_rnnt_600m_config(), m600["chatty"], 0)
    try:
        pcms = _ragged_30s(synth, synth.make_audio(480000, 2100))
        got = e.transcribe_batch(pcms, pkg.Decoder.RNNT)
        assert e.truncated_count() == 0
        assert e.cap == 10 * 376 + 8
        for i, pcm in enumerate(pcms):
            assert _tt(e.transcribe_batch([pcm], pkg.Decoder.RNNT)[0]) == _tt(got[i]), i
        for toks in got:
            per_frame = np.bincount([t.start_frame for t in toks])
            assert per_frame.max() <= 10 and all(t.start_frame == t.end_frame for t in toks)
        assert max(len(t) for t in got) > 3 * 376          # the hypotheses really are long
        assert sum(int((np.bincount([t.start_frame for t in toks]) == 10).sum()) for toks in got) > 0
    finally:
        e.close()
