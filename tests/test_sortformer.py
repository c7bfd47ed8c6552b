"""Sortformer offline diarization (sortformer-117m): the preset, the host segmenter, the numpy restatement
(tests/sortformer_oracle.py) pinned to goldens of the compiled reference (tests/golden/golden_sortformer_v1.npz, made by
make_golden_sortformer.py), and on the GPU the whole path (features, NEST encoder, probs, segments) against both.

The synthetic weights come from sortformer_oracle.calibrated_weights: output_proj_'s bias puts each speaker's threshold in a
gap of its logits, so every speaker is active and inactive somewhere, and seeds whose smallest |logit| is below MARGIN are
rejected: device rounding (about 1e-5 on a logit) cannot flip a threshold decision there, so segments must be exactly
equal.  The golden file records the seed, the bias, MARGIN and the smallest |logit| reached."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sortformer_oracle as SO  # noqa: E402

MARGIN = 1e-3              # smallest |logit| a seed must keep (device error on a logit is ~1e-5)
MEL_TOL = 2e-3             # abs, log-mel (as test_gpu_parity.py)
ENC_TOL = 1e-3             # relative to max |enc|
PROBS_TOL = 1e-3           # abs on sigmoid activities (bf16x3 / fp32 GEMMs, fp32 attention and head)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_sortformer_v1.npz")
GOLD_TOL = 2e-3            # relative to max |x|: float16 storage of features / encoder / transformer outputs
PROBS_REF_TOL = 1e-4       # abs: oracle vs the compiled reference (fp32 re-association)
TINY_LENS = [48000, 20000, 400, 33000, 16000, 401, 64000, 5000, 12000, 40000, 7000, 28000, 56000, 960, 23000, 31000]


# ---------------------------------------------------------------- CPU


def test_preset_literals(pkg):
    c = pkg.make_sortformer_117m_config()
    e = c.encoder
    assert (e.mel_bins, e.sub_channels, e.d_model, e.n_layers, e.n_heads, e.ff, e.conv_k) == (128, 256, 512, 17, 8, 2048, 9)
    assert (c.t_hidden, c.t_layers, c.t_heads, c.t_ff, c.max_speakers, c.activity_threshold) == (192, 18, 8, 768, 4, 0.5)
    assert c.t_hidden // c.t_heads == 24
    t = pkg.make_tiny_sortformer_config()
    assert t.t_hidden // t.t_heads == 24


def test_c_preset_equals_python(pkg):
    from parakeet_cpp_b200.engine import _PkSortformerConfig
    L = pkg.load_library()
    got = _PkSortformerConfig()
    L.pk_config_sortformer_117m(C.byref(got))
    want = pkg.make_sortformer_117m_config().to_c()
    assert bytes(got) == bytes(want)
    assert (got.enc.max_batch, got.enc.max_samples) == (16, 90 * 16000)


def _segs(pkg, p, thr=0.5):
    return [(g.speaker_id, g.start, g.end) for g in pkg.diar_segments(np.asarray(p, np.float32), thr)]


def test_segments_known_answers(pkg):
    f = np.float32
    assert _segs(pkg, np.zeros((5, 4))) == []
    # active to the last frame; p == 0.5 is not active; single-frame segments
    p = np.array([[0.2, 0.5, 0.9], [0.6, 0.5, 0.1], [0.2, 0.51, 0.9], [0.7, 0.1, 0.9]], f)
    assert _segs(pkg, p) == [(2, 0.0, 0.0), (0, f(1) * f(0.08), f(1) * f(0.08)), (1, f(2) * f(0.08), f(2) * f(0.08)),
                             (2, f(2) * f(0.08), f(3) * f(0.08)), (0, f(3) * f(0.08), f(3) * f(0.08))]
    # equal starts keep speaker order
    p = np.full((3, 4), 0.9, f)
    assert [s for s, _, _ in _segs(pkg, p)] == [0, 1, 2, 3]
    assert pkg.load_library().pk_diar_segments(None, 3, 4, 0.5, None, None, None, 0) == -1


def test_segments_equal_oracle_on_random_probs(pkg):
    rng = np.random.default_rng(4)
    for T, S in ((1, 1), (7, 4), (200, 4), (64, 3)):
        p = (rng.random((T, S)) < 0.5).astype(np.float32) * 0.8 + 0.1
        got = _segs(pkg, p)
        want = SO.probs_to_segments(p)
        assert [(s, np.float32(a), np.float32(b)) for s, a, b in got] == [(s, np.float32(a), np.float32(b)) for s, a, b in want]


# ---------------------------------------------------------------- goldens of the compiled reference


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


def _golden_model(pkg, synth, g, tag):
    cfg = pkg.make_tiny_sortformer_config() if tag == "tiny" else pkg.make_sortformer_117m_config()
    lens = [int(n) for n in g[tag + ".lens"]]
    clips = [synth.make_audio(n, int(g[tag + ".audio_seed"]) + i) for i, n in enumerate(lens)]
    return cfg, SO.golden_weights(cfg, g, tag, synth), clips


def assert_same_segments(got, ref):
    """DESIGN.md section 5 (iv): the reference orders segments with std::sort by start, which for more than 16 segments
    (introsort) does not keep equal starts in speaker order.  Up to 16 segments the order must be identical; beyond, the
    segments must be the same and both sorted by start."""
    got = [(int(s), np.float32(a), np.float32(b)) for s, a, b in got]
    ref = [(int(s), np.float32(a), np.float32(b)) for s, a, b in ref]
    if len(ref) <= 16:
        assert got == ref
    else:
        assert sorted(got) == sorted(ref)
        assert [x[1] for x in got] == [x[1] for x in ref]


def _golden_segs(g, k):
    return [(int(s), float(a), float(b)) for s, a, b in g[k + "segs"]]


def test_golden_activity_changes_over_time(g):
    """Each speaker is active and inactive somewhere, and more than one is active at once, in the reference's activities."""
    for tag in ("tiny", "s117m"):
        act = np.concatenate([g[f"{tag}.u{i}.probs"] for i in range(len(g[tag + ".lens"]))]) > 0.5
        assert act.any(axis=0).all() and (~act).any(axis=0).all(), tag
        assert (act.sum(axis=1) > 1).any(), tag


def test_golden_margin_recorded(g):
    assert float(g["margin"]) == np.float32(MARGIN)
    for tag in ("tiny", "s117m"):
        m = float(g[tag + ".min_abs_logit"])
        print(f"{tag}: seed {int(g[tag + '.seed'])}, smallest |logit| {m:.3g} (margin {MARGIN})")
        assert m >= MARGIN


@pytest.mark.parametrize("tag", ["tiny", "s117m"])
def test_oracle_equals_reference_goldens(pkg, synth, g, tag):
    cfg, W, clips = _golden_model(pkg, synth, g, tag)
    lg_min = np.inf
    for i, c in enumerate(clips):
        k = f"{tag}.u{i}."
        f = SO.features(c, cfg)
        if k + "feats" in g:
            assert f.shape == g[k + "feats"].shape
            assert np.abs(f - g[k + "feats"]).max() <= GOLD_TOL * np.abs(f).max()
        p, taps = SO.forward(W, f, cfg, taps=True)
        for name in ("enc", "trans"):
            if k + name not in g:
                continue
            assert taps[name].shape == g[k + name].shape
            assert np.abs(taps[name] - g[k + name]).max() <= GOLD_TOL * np.abs(taps[name]).max(), name
        assert np.abs(p - g[k + "probs"]).max() < PROBS_REF_TOL
        assert_same_segments(SO.probs_to_segments(p), _golden_segs(g, k))
        lg_min = min(lg_min, float(np.abs(taps["logits"]).min()))
    assert lg_min == pytest.approx(float(g[tag + ".min_abs_logit"]), rel=1e-3)


def test_segments_reproduce_reference_goldens(pkg, g):
    n = 0
    for k in g:
        if k.endswith(".probs"):
            base = k[:-len("probs")]
            assert_same_segments(_segs(pkg, g[k]), _golden_segs(g, base))
            n += 1
    assert n == len(g["tiny.lens"]) + len(g["s117m.lens"])


# ---------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def tiny_model(pkg, synth, g, tmp_path_factory):
    cfg, W, clips = _golden_model(pkg, synth, g, "tiny")
    path = str(tmp_path_factory.mktemp("sortformer") / "tiny.safetensors")
    synth.save_safetensors(path, W)
    return cfg, W, path, clips


@pytest.mark.gpu
@pytest.mark.parametrize("math", [0, 2])
def test_tiny_ragged_batch_matches_oracle(pkg, g, tiny_model, math):
    cfg0, W, path, clips = tiny_model
    cfg = pkg.make_tiny_sortformer_config(math=math)
    eng = pkg.Engine(cfg, path, 0)
    try:
        feats = eng.mel(clips)
        encs = eng.encode(feats)
        probs = eng.diarize_probs(clips)
        fwd = eng.sortformer_forward(feats)
        segs = eng.diarize_batch(clips)
        for i, c in enumerate(clips):
            f_ref = SO.features(c, cfg)
            assert np.abs(feats[i] - f_ref).max() < MEL_TOL
            p_ref, taps = SO.forward(W, f_ref, cfg, taps=True)
            e_ref = taps["enc"]
            assert np.abs(encs[i] - e_ref).max() <= ENC_TOL * np.abs(e_ref).max()
            assert probs[i].shape == p_ref.shape
            assert np.abs(probs[i] - p_ref).max() < PROBS_TOL
            assert np.abs(fwd[i] - p_ref).max() < PROBS_TOL
            got = [(x.speaker_id, x.start, x.end) for x in segs[i]]
            assert got == SO.probs_to_segments(p_ref)
            assert_same_segments(got, _golden_segs(g, f"tiny.u{i}."))
        # the whole batch equals each utterance's solo run bit for bit
        for i, c in enumerate(clips):
            solo = eng.diarize_probs([c])[0]
            assert np.array_equal(solo, probs[i])
        # a second call replays the CUDA graph of this batch shape: same result
        again = eng.diarize_probs(clips)
        assert all(np.array_equal(a, b) for a, b in zip(again, probs))
    finally:
        eng.close()


@pytest.mark.gpu
def test_decode_entry_points_refuse(pkg, tiny_model):
    cfg, W, path, clips = tiny_model
    eng = pkg.Engine(cfg, path, 0)
    try:
        for call in (lambda: eng.transcribe_batch(clips[:1], pkg.Decoder.TDT), lambda: eng.run_staged(pkg.Decoder.CTC),
                     lambda: eng.set_boost([[1, 2]]), lambda: eng.decode([np.zeros((4, cfg.d_model), np.float32)], pkg.Decoder.CTC)):
            with pytest.raises(RuntimeError, match=r"\(1\)"):
                call()
    finally:
        eng.close()


@pytest.mark.gpu
def test_loader_keys(pkg, synth, tiny_model, tmp_path):
    cfg, W, path, clips = tiny_model
    W2 = {k: v for k, v in W.items() if not k.startswith("hidden_to_spks_")}
    p2 = str(tmp_path / "no_h2s.safetensors")
    synth.save_safetensors(p2, W2)
    pkg.Engine(cfg, p2, 0).close()
    for missing in ("transformer_.layers_.1.norm2_.bias", "nest_encoder_.layers_.0.attn_.pos_bias_u_", "output_proj_.weight"):
        p3 = str(tmp_path / "missing.safetensors")
        synth.save_safetensors(p3, {k: v for k, v in W.items() if k != missing})
        with pytest.raises(RuntimeError, match=r"\(4\)"):
            pkg.Engine(cfg, p3, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("math", [0, 2])
def test_117m_matches_reference(pkg, synth, g, tmp_path, math):
    """sortformer-117m on the golden 10 s and 30 s clips, in one batch."""
    cfg0, W, clips = _golden_model(pkg, synth, g, "s117m")
    cfg = pkg.make_sortformer_117m_config(max_batch=2, max_samples=max(len(c) for c in clips), math=math)
    path = str(tmp_path / "sf117m.safetensors")
    synth.save_safetensors(path, W)
    eng = pkg.Engine(cfg, path, 0)
    try:
        feats = eng.mel(clips)
        encs = eng.encode(feats)
        probs = eng.diarize_probs(clips)
        segs = eng.diarize_batch(clips)
        for i, c in enumerate(clips):
            k = f"s117m.u{i}."
            f_ref = SO.features(c, cfg)
            assert np.abs(feats[i] - f_ref).max() < MEL_TOL
            p_ref, taps = SO.forward(W, feats[i], cfg, taps=True)
            assert np.abs(encs[i] - taps["enc"]).max() <= ENC_TOL * np.abs(taps["enc"]).max()
            if k + "enc" in g:
                assert np.abs(encs[i] - g[k + "enc"]).max() <= (ENC_TOL + GOLD_TOL) * np.abs(taps["enc"]).max()
            assert np.abs(probs[i] - p_ref).max() < PROBS_TOL
            assert np.abs(probs[i] - g[k + "probs"]).max() < PROBS_TOL
            assert_same_segments([(x.speaker_id, x.start, x.end) for x in segs[i]], _golden_segs(g, k))
    finally:
        eng.close()


@pytest.mark.gpu
def test_cpp_sortformer(pkg, synth, tiny_model, tmp_path):
    """parakeet::Sortformer of the C++ drop-in (include/parakeet/sortformer.hpp): forward, diarize and diarize_batch on the
    tiny shape equal the Python engine's results."""
    cfg, W, path, clips = tiny_model
    exe = str(tmp_path / "cpp_sortformer_check")
    libdir = os.path.dirname(pkg.lib_path())
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp_sortformer_check.cpp"),
                    "-L" + libdir, "-lparakeet_b200", "-Wl,-rpath," + libdir, "-o", exe], check=True)
    use = clips[:3]
    fp = str(tmp_path / "feats.f32")
    feats = SO.features(use[0], cfg)
    feats.astype(np.float32).tofile(fp)
    pps = []
    for i, c in enumerate(use):
        pp = str(tmp_path / f"pcm{i}.f32")
        c.astype(np.float32).tofile(pp)
        pps.append(pp)
    out = subprocess.run([exe, path, fp] + pps, check=True, capture_output=True, text=True).stdout.strip().split("\n")
    eng = pkg.Engine(pkg.make_tiny_sortformer_config(max_batch=8, max_samples=64000), path, 0)
    try:
        want_p = eng.sortformer_forward([feats])[0]
        want_batch = eng.diarize_batch(use)
    finally:
        eng.close()
    fmt = lambda segs: [f"{x.speaker_id}:{np.float32(x.start)}:{np.float32(x.end)}" for x in segs]  # noqa: E731
    got_p = np.array([float(v) for v in out[0].split()[1:]], np.float32).reshape(want_p.shape)
    assert np.array_equal(got_p, want_p)
    parse = lambda line: [f"{a}:{np.float32(b)}:{np.float32(c)}" for a, b, c in (t.split(":") for t in line.split()[1:])]  # noqa: E731
    assert out[1].split()[0] == "DIARIZE" and parse(out[1]) == fmt(pkg.diar_segments(want_p))
    for i in range(len(use)):
        assert out[2 + i].split()[0] == "BATCH" and parse(out[2 + i]) == fmt(want_batch[i])
    assert out[2 + len(use)] == "PRE_LN refused"
