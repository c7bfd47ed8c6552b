"""Streaming Sortformer diarization (Sortformer::diarize_chunk with AOSCCache): the numpy restatement
(tests/sortformer_stream_oracle.py) pinned to goldens of the compiled reference (tests/golden/golden_sortformer_stream_v1.npz,
made by make_golden_sortformer_stream.py), the AOSC known answers, and on the GPU the lock-step streams of a Sortformer
engine against both.

The weights are calibrated on streaming logits (sortformer_stream_oracle.calibrated_weights) and seeds whose smallest
|logit| is below MARGIN are rejected, so device rounding cannot flip a threshold decision: segments and arrival orders
must be exactly equal."""
from __future__ import annotations

import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sortformer_stream_oracle as SSO  # noqa: E402

MARGIN = 1e-3
MEL_TOL = 2e-3
ENC_TOL = 1e-3             # relative to max |enc|
PROBS_TOL = 1e-3
PROBS_REF_TOL = 1e-4       # oracle vs the compiled reference
GOLD_TOL = 2e-3            # relative: float16 storage of the encoder rows
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_sortformer_stream_v1.npz")
# per stream, the chunk lengths of each step: chunks with no encoder frame (400, 250, 160, 2 samples), empty chunks (no input
# that step), and chunks that leave 1..7 mel frames queued
TINY_SCHED = [[2560] * 6,
              [400, 0, 1000, 5000, 160, 3000],
              [8000, 250, 2, 0, 12000, 1700]]
TINY_MAX_CHUNK = 12000
TINY_MAX_SAMPLES = 160000  # the tiny preset's 64 000 samples hold fewer encoder frames than the 70-frame left context
S117_LEN = 480000
S117_CHUNKS = (2560, 16000)


def tiny_clips(synth):
    return [synth.make_audio(sum(s), 700 + i) for i, s in enumerate(TINY_SCHED)]


def _segs(segs):
    return [(int(s), np.float32(a), np.float32(b)) for s, a, b in segs]


# ---------------------------------------------------------------- CPU


def _aosc_known_answers(make):
    """The reference's AOSC known answers (tests/test_all.cpp:299-341 of the reference)."""
    f = np.float32
    c = make(4)
    assert c.speaker_order() == []
    c.update(np.array([[0.1, 0.9, 0.2, 0.8]], f))              # 1 and 3 arrive in index order within the frame
    assert c.speaker_order() == [1, 3]
    c.update(np.array([[0.6, 0.1, 0.1, 0.1], [0.1, 0.9, 0.1, 0.9]], f))
    assert c.speaker_order() == [1, 3, 0]                       # a speaker is never forgotten or repeated
    c.update(np.array([[0.5, 0.5, 0.5, 0.5]], f))               # 0.5 is not "> 0.5"
    assert c.speaker_order() == [1, 3, 0]
    c.update(np.array([[0.1, 0.1, 0.51, 0.1]], f))
    assert c.speaker_order() == [1, 3, 0, 2]
    c.reset()
    assert c.speaker_order() == []
    c.update(np.array([[0.1, 0.1, 0.9, 0.1]], f))
    assert c.speaker_order() == [2]
    c2 = make(2)                                                # wider probs than max_speakers: the extra columns are ignored
    c2.update(np.array([[0.1, 0.1, 0.9, 0.9], [0.1, 0.9, 0.9, 0.9]], f))
    assert c2.speaker_order() == [1]


def test_aosc_known_answers_python(pkg):
    _aosc_known_answers(pkg.AOSCCache)


def test_aosc_oracle_agrees(pkg):
    rng = np.random.default_rng(1)
    for _ in range(20):
        p = rng.random((int(rng.integers(1, 9)), 4)).astype(np.float32)
        a, b = pkg.AOSCCache(4), SSO.AOSCCache(4)
        a.update(p)
        b.update(p)
        assert a.speaker_order() == b.order


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


def _golden_weights(synth, g, tag, cfg):
    W = synth.make_sortformer_weights(cfg, seed=int(g[tag + ".seed"]))
    W["output_proj_.bias"] = g[tag + ".spk_bias"].astype(np.float32)
    return W


def _golden_runs(pkg, synth, tag):
    if tag == "tiny":
        return pkg.make_tiny_sortformer_config(), [("tiny", tiny_clips(synth), TINY_SCHED)]
    clip = synth.make_audio(S117_LEN, 500)
    return pkg.make_sortformer_117m_config(), [(f"s117m.c{ch}", [clip], [SSO.split(S117_LEN, ch)]) for ch in S117_CHUNKS]


def test_golden_margin_and_activity(g):
    assert float(g["margin"]) == np.float32(MARGIN)
    for tag in ("tiny", "s117m"):
        assert float(g[tag + ".min_abs_logit"]) >= MARGIN
        act = np.concatenate([g[k] for k in g if k.startswith(tag) and k.endswith(".probs") and len(g[k])]) > 0.5
        assert act.any(axis=0).all() and (~act).any(axis=0).all(), tag


def test_golden_schedule_shape(g):
    """The tiny schedule has {} returns for non-empty chunks, and every stream's order grows by arrival only."""
    empties = [(k, s) for k in range(6) for s in range(3) if TINY_SCHED[s][k] > 0 and int(g[f"tiny.k{k}.s{s}.C"]) == 0]
    assert len(empties) >= 4
    for s in range(3):
        prev = []
        for k in range(6):
            o = list(g[f"tiny.k{k}.s{s}.order"])
            assert o[:len(prev)] == prev
            prev = o


@pytest.mark.parametrize("tag", ["tiny", "s117m"])
def test_oracle_equals_reference_goldens(pkg, synth, g, tag):
    cfg, runs = _golden_runs(pkg, synth, tag)
    W = _golden_weights(synth, g, tag, cfg)
    for sub, clips, sched in runs:
        steps = SSO.run_schedule(W, cfg, clips, sched)
        base = [0] * len(clips)
        for k, row in enumerate(steps):
            for s, r in enumerate(row):
                key = f"{sub}.k{k}.s{s}."
                assert r["probs"].shape[0] == int(g[key + "C"]), key
                assert r["base"] == base[s]
                base[s] += r["probs"].shape[0]
                if len(r["probs"]):
                    assert np.abs(r["probs"] - g[key + "probs"]).max() < PROBS_REF_TOL, key
                assert _segs(r["segs"]) == _segs(g[key + "segs"]), key
                assert r["order"] == list(g[key + "order"]), key
                if key + "enc" in g:
                    assert np.abs(r["enc"] - g[key + "enc"]).max() <= GOLD_TOL * np.abs(r["enc"]).max(), key


# ---------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def tiny_model(pkg, synth, g, tmp_path_factory):
    cfg = pkg.make_tiny_sortformer_config()
    W = _golden_weights(synth, g, "tiny", cfg)
    path = str(tmp_path_factory.mktemp("sortformer_stream") / "tiny.safetensors")
    synth.save_safetensors(path, W)
    clips = tiny_clips(synth)
    return W, path, clips, SSO.run_schedule(W, cfg, clips, TINY_SCHED)


def _open(pkg, path, math, n_streams=3, max_batch=8, max_chunk=TINY_MAX_CHUNK):
    eng = pkg.Engine(pkg.make_tiny_sortformer_config(math=math, max_batch=max_batch, max_samples=TINY_MAX_SAMPLES), path, 0)
    eng.diar_stream_open(n_streams, max_chunk)
    return eng


def _chunks(clips, sched, k):
    return [c[sum(sch[:k]):sum(sch[:k + 1])] for c, sch in zip(clips, sched)]


def _check_step(pkg, got, base, ref_row, g, k, enc=None, speakers=None):
    for s, r in enumerate(ref_row):
        key = f"tiny.k{k}.s{s}."
        assert got[s].shape == r["probs"].shape, key
        assert base[s] == r["base"], key
        if len(r["probs"]):
            assert np.abs(got[s] - r["probs"]).max() < PROBS_TOL, key
            assert np.abs(got[s] - g[key + "probs"]).max() < PROBS_TOL, key
        segs = [(x.speaker_id, x.start, x.end) for x in pkg.diar_segments(got[s])]
        assert _segs(segs) == _segs(r["segs"]) == _segs(g[key + "segs"]), key
        if enc is not None and len(r["enc"]):
            assert np.abs(enc[s] - r["enc"]).max() <= ENC_TOL * np.abs(r["enc"]).max(), key
        if speakers is not None:
            assert speakers[s] == r["order"] == list(g[key + "order"]), key


@pytest.mark.gpu
@pytest.mark.parametrize("math", [0, 2])
def test_tiny_schedule_matches_oracle_and_reference(pkg, g, tiny_model, math):
    W, path, clips, ref = tiny_model
    eng = _open(pkg, path, math)
    try:
        for k in range(len(TINY_SCHED[0])):
            got, base, enc = eng.diar_stream_step(_chunks(clips, TINY_SCHED, k), taps=True)
            _check_step(pkg, got, base, ref[k], g, k, enc=enc, speakers=[eng.diar_stream_speakers(s) for s in range(3)])
        # a second run of the schedule replays the step graphs: bit-identical
        eng.diar_stream_reset(-1)
        first = [eng.diar_stream_step(_chunks(clips, TINY_SCHED, k))[0] for k in range(6)]
        eng.diar_stream_reset(-1)
        again = [eng.diar_stream_step(_chunks(clips, TINY_SCHED, k))[0] for k in range(6)]
        eng.diar_stream_reset(-1)
        third = [eng.diar_stream_step(_chunks(clips, TINY_SCHED, k))[0] for k in range(6)]
        for a, b, c in zip(first, again, third):
            assert all(np.array_equal(x, y) and np.array_equal(x, z) for x, y, z in zip(a, b, c))
        for k in range(6):
            _check_step(pkg, first[k], [r["base"] for r in ref[k]], ref[k], g, k)
    finally:
        eng.close()


# TINY_SCHED with every non-empty chunk >= 400 samples (pk_mel's shortest utterance); 400-sample chunks still yield no frame
FEAT_SCHED = [[2560] * 6,
              [400, 0, 1000, 5000, 480, 3000],
              [8000, 400, 0, 0, 12000, 1700]]


@pytest.mark.gpu
def test_pcm_and_feature_entry_points_agree(pkg, synth):
    """pk_diar_stream_step_feats fed the features pk_mel makes for each chunk equals the PCM step bit for bit."""
    cfg = pkg.make_tiny_sortformer_config()
    W = synth.make_sortformer_weights(cfg, seed=0)
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "w.safetensors")
        synth.save_safetensors(path, W)
        clips = [synth.make_audio(sum(s), 900 + i) for i, s in enumerate(FEAT_SCHED)]
        a, b = _open(pkg, path, 0), _open(pkg, path, 0)
        try:
            rows = 0
            for k in range(6):
                ch = _chunks(clips, FEAT_SCHED, k)
                pa, ba = a.diar_stream_step(ch)
                feats = [b.mel([c])[0] if len(c) else np.zeros((0, cfg.mel_bins), np.float32) for c in ch]
                pb, bb = b.diar_stream_step(feats, feats=True)
                assert np.array_equal(ba, bb)
                for s in range(3):
                    assert np.array_equal(pa[s], pb[s]), (k, s)
                    rows += len(pa[s])
                    assert a.diar_stream_speakers(s) == b.diar_stream_speakers(s)
            assert rows > 0
        finally:
            a.close()
            b.close()


@pytest.mark.gpu
def test_streams_equal_solo_runs_reset_and_offline_between(pkg, tiny_model):
    """8 streams (the schedule's three, each given to several slots at different offsets) equal their solo runs; a reset of
    one stream mid-schedule replays its first chunks exactly and leaves the others untouched; an offline pk_diarize_batch
    between steps gives the bytes of a fresh engine and does not disturb the streams."""
    W, path, clips, ref = tiny_model
    sched = [TINY_SCHED[i % 3] for i in range(8)]
    cl = [clips[i % 3] for i in range(8)]
    eng, solo = _open(pkg, path, 0, n_streams=8), _open(pkg, path, 0, n_streams=1)
    fresh = pkg.Engine(pkg.make_tiny_sortformer_config(math=0, max_batch=8, max_samples=TINY_MAX_SAMPLES), path, 0)
    try:
        offline_want = fresh.diarize_probs(clips[:2])
        many = []
        for k in range(6):
            many.append(eng.diar_stream_step(_chunks(cl, sched, k))[0])
            if k == 2:
                off = eng.diarize_probs(clips[:2])
                assert all(np.array_equal(x, y) for x, y in zip(off, offline_want))
        orders = [eng.diar_stream_speakers(s) for s in range(8)]
        for s in range(8):
            solo.diar_stream_reset(-1)
            for k in range(6):
                p = solo.diar_stream_step([_chunks(cl, sched, k)[s]])[0][0]
                assert p.shape == many[k][s].shape
                if len(p):
                    assert np.abs(p - many[k][s]).max() < PROBS_TOL
                    assert _segs([(x.speaker_id, x.start, x.end) for x in pkg.diar_segments(p)]) == \
                        _segs([(x.speaker_id, x.start, x.end) for x in pkg.diar_segments(many[k][s])])
            assert solo.diar_stream_speakers(0) == orders[s]
        # reset stream 5 after step 3: it restarts from the schedule's beginning while the others continue
        eng.diar_stream_reset(-1)
        for k in range(3):
            eng.diar_stream_step(_chunks(cl, sched, k))
        eng.diar_stream_reset(5)
        assert eng.diar_stream_speakers(5) == []
        for k in range(3, 6):
            ch = _chunks(cl, sched, k)
            ch[5] = _chunks(cl, sched, k - 3)[5]
            got = eng.diar_stream_step(ch)[0]
            for s in range(8):
                want = many[k - 3][s] if s == 5 else many[k][s]
                assert got[s].shape == want.shape
                if s == 5 or len(want) == 0:
                    assert got[s].shape == want.shape
                if len(want):
                    assert np.abs(got[s] - want).max() < PROBS_TOL
    finally:
        eng.close()
        solo.close()
        fresh.close()


@pytest.mark.gpu
def test_refusals_and_capacity(pkg, synth, tiny_model):
    W, path, clips, ref = tiny_model
    eng = _open(pkg, path, 0)
    try:
        with pytest.raises(RuntimeError, match=r"\(5\)"):                  # PK_ERR_CAPACITY: chunk over max_chunk_samples
            eng.diar_stream_step([np.zeros(TINY_MAX_CHUNK + 1, np.float32), np.zeros(0, np.float32), np.zeros(0, np.float32)])
        with pytest.raises(RuntimeError, match=r"\(1\)"):                  # a 1-sample chunk: the reference does not return
            eng.diar_stream_step([np.zeros(1, np.float32), np.zeros(0, np.float32), np.zeros(0, np.float32)])
        p, base = eng.diar_stream_step([np.zeros(2, np.float32), np.zeros(0, np.float32), np.zeros(0, np.float32)])
        assert [len(x) for x in p] == [0, 0, 0]
        off = np.zeros(4, np.int64)                                         # the ASR stream calls on a Sortformer engine
        assert eng.L.pk_stream_step(eng.h, None, off.ctypes.data_as(__import__("ctypes").POINTER(__import__("ctypes").c_int64)),
                                    None, None, None, None, None) == 1
        assert eng.L.pk_stream_reset(eng.h, -1) == 1
        with pytest.raises(RuntimeError, match=r"\(1\)"):
            eng.L_open = eng._check(eng.L.pk_stream_open(eng.h, 1, 2560, 70, 0), "pk_stream_open")
        assert eng.L.pk_stream_count(eng.h) == 0 and eng.L.pk_diar_stream_count(eng.h) == 3
        with pytest.raises(RuntimeError, match=r"\(1\)"):                  # already open
            eng.diar_stream_open(2, 2560)
    finally:
        eng.close()
    with pytest.raises(RuntimeError, match=r"\(5\)"):                      # left context + chunk frames over the capacity
        e2 = pkg.Engine(pkg.make_tiny_sortformer_config(math=2), path, 0)
        try:
            e2.diar_stream_open(2, 2560)
        finally:
            e2.close()
    with pytest.raises(RuntimeError, match=r"\(5\)"):                      # more streams than max_batch
        e3 = pkg.Engine(pkg.make_tiny_sortformer_config(math=2, max_batch=2, max_samples=TINY_MAX_SAMPLES), path, 0)
        try:
            e3.diar_stream_open(3, 2560)
        finally:
            e3.close()


@pytest.mark.gpu
def test_asr_engine_refuses_diar_streams(pkg, synth, tmp_path):
    cfg = pkg.make_tiny_stream_config()
    O = __import__("__graft_entry__").load_oracle()
    W = synth.make_weights(O.make_tiny_stream_config(), seed=1)
    p = str(tmp_path / "asr.safetensors")
    synth.save_safetensors(p, W)
    eng = pkg.Engine(cfg, p, 0)
    try:
        with pytest.raises(RuntimeError, match=r"\(1\)"):
            eng.diar_stream_open(1, 2560)
        assert eng.L.pk_diar_stream_step(eng.h, None, None, None, None, None, None) == 1
        assert eng.L.pk_diar_stream_speakers(eng.h, 0, None, 0) == -1
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("math", [0, 2])
def test_117m_matches_reference(pkg, synth, g, tmp_path, math):
    """sortformer-117m on the golden 30 s clip at 2560 and 16000 samples per chunk."""
    cfg0, runs = _golden_runs(pkg, synth, "s117m")
    W = _golden_weights(synth, g, "s117m", cfg0)
    path = str(tmp_path / "sf117m.safetensors")
    synth.save_safetensors(path, W)
    eng = pkg.Engine(pkg.make_sortformer_117m_config(max_batch=2, max_samples=160000, math=math), path, 0)
    try:
        for sub, clips, sched in runs:
            eng.diar_stream_open(1, sched[0][0])
            pos, base_want = 0, 0
            for k, n in enumerate(sched[0]):
                key = f"{sub}.k{k}.s0."
                if k < 6:
                    p, base, enc = eng.diar_stream_step([clips[0][pos:pos + n]], taps=True)
                else:
                    p, base = eng.diar_stream_step([clips[0][pos:pos + n]])
                pos += n
                assert p[0].shape[0] == int(g[key + "C"]) and base[0] == base_want, key
                base_want += p[0].shape[0]
                if len(p[0]):
                    assert np.abs(p[0] - g[key + "probs"]).max() < PROBS_TOL, key
                if key + "enc" in g:
                    e_ref = g[key + "enc"].astype(np.float32)
                    assert np.abs(enc[0] - e_ref).max() <= (ENC_TOL + GOLD_TOL) * np.abs(e_ref).max(), key
                segs = [(x.speaker_id, x.start, x.end) for x in pkg.diar_segments(p[0])]
                assert _segs(segs) == _segs(g[key + "segs"]), key
                assert eng.diar_stream_speakers(0) == list(g[key + "order"]), key
            eng.L.pk_diar_stream_count(eng.h)
            # the streams of this chunk size are done: close by recreating the engine for the next
            eng.close()
            eng = pkg.Engine(pkg.make_sortformer_117m_config(max_batch=2, max_samples=160000, math=math), path, 0)
    finally:
        eng.close()


@pytest.mark.gpu
def test_cpp_sortformer_stream(pkg, tiny_model, tmp_path):
    """parakeet::Sortformer::diarize_chunk and parakeet::DiarizationStreamingBatch of the C++ drop-in equal the Python
    engine's results on the tiny schedule."""
    W, path, clips, ref = tiny_model
    exe = str(tmp_path / "cpp_sortformer_stream_check")
    libdir = os.path.dirname(pkg.lib_path())
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp_sortformer_stream_check.cpp"), "-L" + libdir, "-lparakeet_b200",
                    "-Wl,-rpath," + libdir, "-o", exe], check=True)
    cfg = pkg.make_tiny_sortformer_config()
    files = []
    for s in range(3):
        for k in range(6):
            ch = _chunks(clips, TINY_SCHED, k)[s]
            fp = str(tmp_path / f"s{s}k{k}.f32")
            SSO.chunk_features(ch, cfg).astype(np.float32).tofile(fp)
            pp = str(tmp_path / f"s{s}k{k}.pcm")
            ch.astype(np.float32).tofile(pp)
            files += [fp, pp]
    out = subprocess.run([exe, path, str(TINY_MAX_SAMPLES), str(TINY_MAX_CHUNK)] + files, check=True, capture_output=True,
                         text=True).stdout.strip().split("\n")
    eng = _open(pkg, path, 0)
    try:
        lines = iter(out)
        for k in range(6):
            got, base = eng.diar_stream_step(_chunks(clips, TINY_SCHED, k))
            for s in range(3):
                segs = " ".join(f"{x.speaker_id}:{np.float32(x.start)}:{np.float32(x.end)}" for x in pkg.diar_segments(got[s]))
                order = " ".join(str(v) for v in eng.diar_stream_speakers(s))
                for kind in ("CHUNK", "BATCH"):
                    line = next(lines).split("|")
                    assert line[0].split() == [kind, str(k), str(s)]
                    parse = lambda t: [f"{a}:{np.float32(b)}:{np.float32(c)}" for a, b, c in (x.split(":") for x in t.split())]  # noqa: E731
                    assert parse(line[1]) == parse(segs), (kind, k, s)
                    assert line[2].split() == order.split(), (kind, k, s)
        assert next(lines) == "AOSC ok"
    finally:
        eng.close()
