"""Nemotron streaming (reference include/parakeet/nemotron.hpp, src/nemotron.cpp): the nemotron-600m preset, its latency
modes and lock-step streaming of 600M-class models on the device.

Fixtures: tests/golden/golden_nemotron_v1.npz (tests/golden/make_golden_nemotron.py) -- the compiled reference running
NemotronTranscriber::transcribe_chunk's steps with blank = vocab - 1 on
  * tnemo:   the tiny Nemotron shape (head_dim 128, two LSTM layers) on the ragged STREAM_SCHEDULE;
  * nemo600: the nemotron-600m preset, seed-0 synthetic weights, 14 x 2560 samples at latency 0.  The generator asserts
             that latencies 1, 6 and 13 give byte-identical outputs and stores their digests.
CPU: the numpy restatement against the fixtures, the preset.  GPU: per-chunk parity, latency modes, lock step, the 600m
geometry at 8 and 64 streams, the C++ drop-in.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import subprocess

import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import nemotron_oracle as NO  # noqa: E402
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_nemotron_v1.npz")
ENC_TOL = 1e-3                      # relative, as the eou streaming tests
MATH = {"bf16x3": 0, "fp32": 2}
LATENCIES = (0, 1, 6, 13)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(float(np.abs(b).max()), 1e-30))


def _tt(toks):
    return [[t.token_id, t.start_frame, t.end_frame] for t in toks]


@pytest.fixture(scope="module")
def g():
    with np.load(GOLDEN, allow_pickle=False) as f:
        return {k: f[k] for k in f.files}


def _cfgs(pkg, O, tag, latency=0):
    if tag == "tnemo":
        return NO.make_tiny_nemotron_config(), pkg.make_tiny_nemotron_config()
    return NO.make_nemotron_600m_config(latency), pkg.make_nemotron_600m_config(latency)


def _stream(g, tag):
    wseed, aseed = (int(v) for v in g[tag + ".seeds"])
    return wseed, aseed, [int(v) for v in g[tag + ".schedule"]]


# ------------------------------------------------------------------------------------------------------------- CPU
def test_nemotron_preset_values(pkg, O):
    """make_nemotron_600m_config (nemotron.hpp:33-54) pinned as literals; mel_bins stays at EncoderConfig's 80."""
    for c in (pkg.make_nemotron_600m_config(), NO.make_nemotron_600m_config()):
        assert (c.mel_bins, c.sub_channels, c.d_model, c.n_layers, c.n_heads, c.ff, c.conv_k) == (80, 256, 1024, 24, 8, 4096, 9)
        assert (c.vocab, c.pred_hidden, c.lstm_layers, c.joint_hidden, tuple(c.durations)) == (8193, 640, 2, 640, (0, 1, 2, 3, 4))
        assert (c.att_context_left, c.att_context_right, c.has_ctc, c.joint_prefix) == (70, 0, False, "joint_.")
        assert c.d_model // c.n_heads == 128
    for lat in LATENCIES:
        assert pkg.make_nemotron_600m_config(lat).att_context_right == lat
        assert NO.make_nemotron_600m_config(lat).att_context_right == lat
    p = pkg.make_nemotron_600m_config()
    assert (p.max_symbols, p.max_batch, p.max_samples) == (10, 64, 102400)
    t = pkg.make_tiny_nemotron_config()
    assert t.d_model // t.n_heads == 128 and t.lstm_layers == 2
    ot = NO.make_tiny_nemotron_config()
    for f in ("mel_bins", "sub_channels", "d_model", "n_layers", "n_heads", "ff", "conv_k", "vocab", "pred_hidden", "lstm_layers",
              "joint_hidden", "durations", "has_ctc", "joint_prefix", "att_context_left", "att_context_right"):
        assert getattr(t, f) == getattr(ot, f), f


def test_pk_config_nemotron_600m_equals_python_preset(pkg):
    L = pkg.load_library()
    c = pkg.engine._PkConfig()
    L.pk_config_nemotron_600m(C.byref(c))
    want = pkg.make_nemotron_600m_config().to_c()
    for name, _ in pkg.engine._PkConfig._fields_:
        a, b = getattr(c, name), getattr(want, name)
        if name == "durations":
            a, b = list(a), list(b)
        assert a == b, name
    # capacity: the K/V ring (70 rows) plus one chunk's frames fit the encoder-frame capacity
    assert pkg.engine.load_library().pk_encoder_frames(1 + c.max_samples // 160) >= 70 + 4


@pytest.mark.parametrize("tag", ["tnemo", "nemo600"])
def test_oracle_streaming_matches_reference_golden(O, synth, g, tag):
    """The numpy streaming restatement (StreamingPreprocessor, stream_encoder_chunk, stream_decode_chunk) at the Nemotron
    shapes -- head_dim 128, two carried LSTM layers, 8193 labels for nemo600 -- against the compiled reference."""
    ocfg = NO.make_tiny_nemotron_config() if tag == "tnemo" else NO.make_nemotron_600m_config(0)
    wseed, aseed, sched = _stream(g, tag)
    W = synth.make_weights(ocfg, seed=wseed)
    pcm = synth.make_audio(sum(sched), aseed)
    pre, cache, st = O.StreamingPreprocessor(ocfg.mel_bins), O.StreamEncoderCache(ocfg.n_layers), O.StreamDecodeState(ocfg)
    pos, ids = 0, []
    for ci, n in enumerate(sched):
        f = pre.process_chunk(pcm[pos:pos + n])
        pos += n
        e = O.stream_encoder_chunk(W, f, cache, ocfg) if f is not None else None
        t = O.stream_decode_chunk(W, e, st, ocfg, max_steps=5000) if e is not None else []
        k = f"{tag}.k{ci}."
        gf, ge_, gt, gc = g[k + "feats"], g[k + "enc"], g[k + "tok"], g[k + "conf"]
        assert (0 if f is None else f.shape[0]) == gf.shape[0], ci
        if gf.shape[0]:
            assert _rel(f, gf) < 1e-4, ci
        assert (0 if e is None else e.shape[0]) == ge_.shape[0], ci
        if ge_.shape[0]:
            assert _rel(e, ge_) < 1e-4, ci
        assert [list(x[:3]) for x in t] == gt.tolist(), ci
        assert np.allclose([x[3] for x in t], gc, rtol=1e-3), ci
        ids += [x[0] for x in t]
    assert len(ids) >= 10
    assert O.detokenize(ids, synth.make_vocab(ocfg.vocab - 1, seed=wseed)) == bytes(g[tag + ".text"]).decode()


def test_golden_records_latency_invariance(g):
    """The generator ran the reference at latencies 1, 6 and 13 and found byte-identical outputs (DESIGN.md section 5)."""
    for lat in LATENCIES[1:]:
        assert np.array_equal(g[f"nemo600.digest_latency{lat}"], g["nemo600.digest"])


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module", params=["bf16x3", "fp32"])
def math_mode(request):
    return request.param


@pytest.fixture(scope="module")
def weights(tmp_path_factory, pkg, O, synth, g):
    """tag -> safetensors path of the fixture's synthetic checkpoint (written once per module)."""
    d = tmp_path_factory.mktemp("nemotron")
    paths = {}

    def get(tag):
        if tag not in paths:
            ocfg = NO.make_tiny_nemotron_config() if tag == "tnemo" else NO.make_nemotron_600m_config(0)
            wseed = int(g[tag + ".seeds"][0])
            p = str(d / f"{tag}.safetensors")
            synth.save_safetensors(p, synth.make_weights(ocfg, seed=wseed))
            paths[tag] = p
        return paths[tag]
    return get


def _engine(pkg, O, weights, g, tag, S, math="bf16x3", latency=0, max_chunk=None):
    _, cfg = _cfgs(pkg, O, tag, latency)
    cfg = dataclasses.replace(cfg, math=MATH[math], max_batch=max(S, 8))
    e = pkg.Engine(cfg, weights(tag), 0)
    e.stream_open(S, max_chunk or max(_stream(g, tag)[2]))
    return e


def _check_chunks(g, tag, e, pcm, sched, mel_tol=2e-3):
    pos, n_tok, encs = 0, 0, []
    for ci, n in enumerate(sched):
        toks, mel, enc = e.stream_step([pcm[pos:pos + n]], taps=True)
        pos += n
        k = f"{tag}.k{ci}."
        gf, ge_, gt, gc = g[k + "feats"], g[k + "enc"], g[k + "tok"], g[k + "conf"]
        assert mel[0].shape == gf.shape, ci
        if gf.shape[0]:
            assert np.abs(mel[0] - gf).max() < mel_tol * max(1.0, float(np.abs(gf).max())), ci
        assert enc[0].shape == ge_.shape, ci
        if ge_.shape[0]:
            assert _rel(enc[0], ge_) < ENC_TOL, ci
        assert _tt(toks[0]) == gt.tolist(), ci
        assert np.allclose([t.confidence for t in toks[0]], gc, rtol=1e-3, atol=1e-6), ci
        n_tok += len(toks[0])
        encs.append(enc[0])
    return n_tok, encs


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["tnemo", "nemo600"])
def test_nemotron_chunks_match_reference_golden(pkg, O, synth, g, weights, math_mode, tag):
    """One stream, chunk by chunk, against the compiled reference: new log-mel frames, the chunk's encoder rows (K/V ring
    of head_dim 128, conv cache), tokens with absolute frames and confidences (two carried LSTM layers); then reset() and
    a replay give identical tokens."""
    _, aseed, sched = _stream(g, tag)
    pcm = synth.make_audio(sum(sched), aseed)
    e = _engine(pkg, O, weights, g, tag, 1, math_mode)
    n_tok, _ = _check_chunks(g, tag, e, pcm, sched)
    assert n_tok >= 10
    e.stream_reset(0)
    pos, again = 0, []
    for n in sched:
        again.append(_tt(e.stream_step([pcm[pos:pos + n]])[0]))
        pos += n
    assert again == [g[f"{tag}.k{ci}.tok"].tolist() for ci in range(len(sched))]
    e.close()


@pytest.mark.gpu
def test_nemotron_latency_modes_give_identical_output(pkg, O, synth, g, weights):
    """Engines opened at latency 0, 1, 6 and 13 (att_context_right) give byte-identical tokens and encoder taps, each equal
    to the reference's latency-0 stream (which the generator found identical at every latency)."""
    tag = "nemo600"
    _, aseed, sched = _stream(g, tag)
    pcm = synth.make_audio(sum(sched), aseed)
    runs = []
    for lat in LATENCIES:
        e = _engine(pkg, O, weights, g, tag, 1, latency=lat)
        pos, toks, encs = 0, [], []
        for n in sched:
            t, _, enc = e.stream_step([pcm[pos:pos + n]], taps=True)
            pos += n
            toks.append([(x.token_id, x.start_frame, x.end_frame, x.confidence) for x in t[0]])
            encs.append(enc[0])
        e.close()
        runs.append((toks, encs))
        assert [[list(x[:3]) for x in tk] for tk in toks] == [g[f"{tag}.k{ci}.tok"].tolist() for ci in range(len(sched))], lat
    for lat, (toks, encs) in zip(LATENCIES[1:], runs[1:]):
        assert toks == runs[0][0], lat
        assert all(np.array_equal(a, b) for a, b in zip(encs, runs[0][1])), lat


@pytest.mark.gpu
def test_nemotron_many_streams_lockstep(pkg, O, synth, g, weights, math_mode):
    """S = 6 tiny Nemotron streams in lock step: copies of the golden stream started at different steps, an always-silent
    stream and one reset half way.  Every copy reproduces the reference's tokens of its own timeline."""
    tag, S = "tnemo", 6
    _, aseed, sched = _stream(g, tag)
    pcm = synth.make_audio(sum(sched), aseed)
    e = _engine(pkg, O, weights, g, tag, S, math_mode)
    want = [g[f"{tag}.k{ci}.tok"].tolist() for ci in range(len(sched))]
    starts = [0, 1, 3, 4, None, 0]
    cuts = np.concatenate([[0], np.cumsum(sched)])
    empty = np.zeros(0, np.float32)
    got = [[] for _ in range(S)]
    local = [0] * S
    for step in range(len(sched) + 5):
        if step == 8:
            e.stream_reset(5)
            local[5], got[5] = 0, []
        chunks = []
        for s in range(S):
            active = starts[s] is not None and step >= starts[s] and local[s] < len(sched)
            chunks.append(pcm[cuts[local[s]]:cuts[local[s] + 1]] if active else empty)
        toks = e.stream_step(chunks)
        for s in range(S):
            if len(chunks[s]):
                got[s].append(_tt(toks[s]))
                local[s] += 1
            else:
                assert toks[s] == []
    for s in (0, 1, 2, 3):
        assert got[s] == want, s
    assert got[5] == want[:len(got[5])] and len(got[5]) >= 10
    e.close()


def _decode_geometry(pkg, S, seed=0):
    """The TDT decode launch the engine makes for S Nemotron streams (P = J = 640, V = 8193 + 5 durations, two LSTM layers,
    carried state), run through pk_kernel_tdt_decode on random weights: -> the geometry it chose (TdtLaunchCtl)."""
    L, E = pkg.load_library(), pkg.engine
    rng = np.random.default_rng(seed)
    P = J = 640
    V, D, Lh, rows = 8193, 5, 2, 2 * S
    keep = []

    def ptr(a, t=C.c_float):
        a = np.ascontiguousarray(a, np.float32 if t is C.c_float else np.int32)
        keep.append(a)
        return a.ctypes.data_as(C.POINTER(t))

    hi = E.TdtHookIn()
    hi.P, hi.J, hi.V, hi.n_dur, hi.L, hi.max_sym = P, J, V, D, Lh, 10
    for i in range(D):
        hi.durations[i] = i
    hi.n_utt, hi.rows = S, rows
    hi.row_off = ptr(np.arange(S + 1) * 2, C.c_int32)
    hi.EP, hi.G0 = ptr(rng.standard_normal((rows, J)) * 0.1), ptr(rng.standard_normal((V, 4 * P)) * 0.1)
    for l in range(Lh):
        hi.W_hh[l] = ptr(rng.standard_normal((4 * P, P)) * 0.04)
        if l:
            hi.W_ih[l], hi.b_ih[l] = ptr(rng.standard_normal((4 * P, P)) * 0.04), ptr(np.zeros(4 * P))
    hi.W_p, hi.W_out, hi.b_out = ptr(rng.standard_normal((J, P)) * 0.04), ptr(rng.standard_normal((V + D, J)) * 0.04), ptr(np.zeros(V + D))
    cap = 2 * rows + 8
    hi.cap, hi.max_steps, hi.carry = cap, 2 * rows + cap + 2, 1
    hi.h0, hi.c0 = ptr(np.zeros((Lh, S, P))), ptr(np.zeros((Lh, S, P)))
    hi.tok0, hi.frame_base = ptr(np.full(S, V - 1), C.c_int32), ptr(np.zeros(S), C.c_int32)
    o = dict(tok=np.zeros((S, 1 + cap), np.int32), t_start=np.zeros((S, cap), np.int32), t_end=np.zeros((S, cap), np.int32),
             t_conf=np.zeros((S, cap), np.float32), overflow=np.zeros(S, np.int32), h_hi=np.zeros((Lh, 2, S, P), np.float32),
             h_lo=np.zeros((Lh, 2, S, P), np.float32), z_hi=np.zeros((S, J), np.float32), z_lo=np.zeros((S, J), np.float32),
             lab_val=np.zeros(S, np.float32), dur_val=np.zeros(S, np.float32), lab_idx=np.zeros(S, np.int32),
             dur_idx=np.zeros(S, np.int32), lse=np.zeros(S, np.float64), c_state=np.zeros((Lh, S, P), np.float32),
             tok_state=np.zeros(S, np.int32))
    ho = E.TdtHookOut()
    for k, a in o.items():
        t = {np.dtype(np.int32): C.c_int32, np.dtype(np.float32): C.c_float, np.dtype(np.float64): C.c_double}[a.dtype]
        setattr(ho, k, a.ctypes.data_as(C.POINTER(t)))
    gb = C.c_int64(-1)
    st = L.pk_kernel_tdt_decode(0, C.byref(hi), C.byref(ho), C.byref(gb))
    assert st == 0 and gb.value == 0, (st, gb.value)
    return {k: getattr(ho, k) for k in ("grid", "cl", "upc", "opc", "out_in_smem", "wih_in_smem", "staged_ih", "wstage_rows")}


@pytest.mark.gpu
@pytest.mark.parametrize("S", [8, 64])
def test_nemotron_600m_streams_match_solo_runs(pkg, O, synth, g, weights, S):
    """nemotron-600m with S streams in lock step (Bpad 32 / 64 in the decode): stream s gets its own audio and starts at
    step s % 5; each row equals the same audio run alone on a one-stream engine, and stream 0 (the fixture's audio) equals
    the reference.  The decode geometry of this stream count is reported."""
    tag = "nemo600"
    _, aseed, sched = _stream(g, tag)
    K, CH = len(sched), sched[0]
    audio = [synth.make_audio(K * CH, aseed + s) for s in range(S)]
    solo_e = _engine(pkg, O, weights, g, tag, 1)
    solo = []
    for s in range(S):
        solo_e.stream_reset(-1)
        solo.append([_tt(solo_e.stream_step([audio[s][k * CH:(k + 1) * CH]])[0]) for k in range(K)])
    solo_e.close()
    assert solo[0] == [g[f"{tag}.k{ci}.tok"].tolist() for ci in range(K)]
    e = _engine(pkg, O, weights, g, tag, S)
    starts = [s % 5 for s in range(S)]
    got = [[] for _ in range(S)]
    empty = np.zeros(0, np.float32)
    for step in range(K + 4):
        chunks = []
        for s in range(S):
            k = step - starts[s]
            chunks.append(audio[s][k * CH:(k + 1) * CH] if 0 <= k < K else empty)
        toks = e.stream_step(chunks)
        for s in range(S):
            if len(chunks[s]):
                got[s].append(_tt(toks[s]))
    e.close()
    for s in range(S):
        assert got[s] == solo[s], s
    assert sum(len(t) for row in got for t in row) >= S * 5
    geom = _decode_geometry(pkg, S)
    print(f"nemotron-600m decode geometry at {S} streams (Bpad {(S + 31) // 32 * 32}): {geom}")
    assert geom["grid"] > 0


@pytest.mark.gpu
def test_cpp_nemotron_transcriber(pkg, O, synth, g, tmp_path):
    """parakeet::NemotronTranscriber and StreamingBatch(NemotronConfig) of the C++ drop-in on the tiny Nemotron shape: each
    transcribe_chunk overload, the partial callback, get_text, timestamps, reset, and a batch of three streams."""
    tag = "tnemo"
    exe = str(tmp_path / "cpp_nemotron_check")
    libdir = os.path.dirname(pkg.lib_path())
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp_nemotron_check.cpp"),
                    "-L" + libdir, "-lparakeet_b200", "-Wl,-rpath," + libdir, "-o", exe], check=True)
    ocfg = NO.make_tiny_nemotron_config()
    wseed, aseed, sched = _stream(g, tag)
    wp, vp, pp = str(tmp_path / "tn.safetensors"), str(tmp_path / "tn.vocab.txt"), str(tmp_path / "pcm.f32")
    synth.save_safetensors(wp, synth.make_weights(ocfg, seed=wseed))
    pieces = synth.make_vocab(ocfg.vocab - 1, seed=wseed)
    synth.save_vocab(vp, pieces)
    synth.make_audio(sum(sched), aseed).astype(np.float32).tofile(pp)
    out = subprocess.run([exe, wp, vp, pp, ",".join(str(n) for n in sched)], check=True, capture_output=True, text=True).stdout.strip().split("\n")
    want = [g[f"{tag}.k{ci}.tok"].tolist() for ci in range(len(sched))]
    all_ids = [w[0] for ci in range(len(sched)) for w in want[ci]]
    text = bytes(g[tag + ".text"]).decode()
    assert text == O.detokenize(all_ids, pieces)
    n_with = sum(1 for w in want if w)
    lines = iter(out)
    for mode in ("F32", "VEC"):
        for ci in range(len(sched)):
            line = next(lines).split()
            assert line[0] == "CHUNK_" + mode and line[1:] == [f"{a}:{b}:{c}" for a, b, c in want[ci]], (mode, ci)
        assert next(lines) == "TEXT " + text, mode
        assert next(lines) == f"CALLBACKS {n_with}", mode
        assert next(lines) == "AFTER_RESET 0", mode
    # int16 PCM (the reference's /32768 conversion) gives the tokens of the same samples passed as floats
    i16 = next(lines).split()
    assert i16[0] == "I16" and i16[1] == "1" and int(i16[2]) > 0, i16
    for s in range(3):                  # the batch: stream 0 the fixture, stream 1 the same one step late, stream 2 silent
        line = next(lines).split()
        assert line[0] == f"BATCH{s}"
        expect = [] if s == 2 else [f"{a}:{b}:{c}" for w in want for a, b, c in w]
        assert line[1:] == expect, s
    assert next(lines) == "BATCH_TEXT0 " + text
