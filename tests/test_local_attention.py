"""Limited-context (banded) relative-position attention for long offline utterances (DESIGN.md section 16).

Kernels against float64 through pk_kernel_attention_local (guarded outputs, the band's exact 2W + 1-row table between NaN
rows, NaN sentinel rows outside every utterance), the bound rejecting a band off by one and a dropped u bias, byte identity
of a band that covers the utterance with full attention (kernels and whole engine), the tiny checkpoint end to end against
the banded oracle, a 60-minute utterance on the 110m shape, the mel front end at one hour, configuration and refusals.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np
import pytest

from local_attention_oracle import brute_attention_local, encoder_forward_local, ref_attention_local
from test_kernels_fp64 import MATH_F32, MATH_X1, MATH_X3, attn_inputs, check_planes, f32p, i32p, nan, ratio, ref_attention

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENC_TOL = 1e-3                       # the encoder tolerance of the parity tests (max-abs error / max-abs reference)
BANDS = [(1, 1), (3, 0), (0, 5), (70, 0), (64, 64), (128, 128), (256, 256), (256, 17)]
KERNELS = [(0, MATH_F32), (1, MATH_X3), (1, MATH_X1)]


def run_local(pkg, kernel, math_mode, row_off, rows, d, H, tmax, left, right, qkv, pp, u, v):
    L = pkg.load_library()
    ro = np.ascontiguousarray(row_off, np.int32)
    f32 = math_mode == MATH_F32
    of = nan((rows, d)) if f32 else None
    oh = None if f32 else nan((rows, d))
    ol = nan((rows, d)) if math_mode == MATH_X3 else None
    gb = C.c_int64(-1)
    st = L.pk_kernel_attention_local(0, kernel, math_mode, len(ro) - 1, i32p(ro), rows, d, H, tmax, left, right, f32p(qkv), f32p(pp),
                                     f32p(u), f32p(v), f32p(of), f32p(oh), f32p(ol), C.byref(gb))
    assert st == 0, f"pk_kernel_attention_local -> {st}"
    assert gb.value == 0, "a guard byte changed"
    return of, oh, ol


def check_local(out, row_off, rows, ref, bd, checked):
    of, oh, ol = out
    inside = np.zeros(rows, bool)
    for b in range(len(row_off) - 1):
        inside[row_off[b]:row_off[b + 1]] = True
    main = of if of is not None else oh
    assert np.all(np.isfinite(main[inside])), "a ctx element was not written (or read a NaN row)"
    assert np.all(np.isnan(main[~inside])), "a row outside the batch was written"
    if ol is not None:
        assert np.all(np.isfinite(ol[inside])) and np.all(np.isnan(ol[~inside]))
    sel = inside & checked
    if of is not None:
        return ratio(of[sel], ref[sel], bd[sel])
    return check_planes(oh[sel], None if ol is None else ol[sel], ref[sel], bd[sel])


def lengths_for(left, right):
    edge = sorted({max(1, x) for w in (left, right, left + right) for x in (w - 1, w, w + 1)})
    return [1, 63, 64, 65, 1000] + edge


# ------------------------------------------------------------------------------------------------- CPU: the oracle itself
@pytest.mark.parametrize("band", [(1, 1), (3, 0), (0, 5), (7, 2), (40, 40)])
def test_banded_reference_is_masked_full_attention(band):
    rng = np.random.default_rng(3)
    d, H, T = 32, 2, 23
    tmax = max(band) + 1
    qkv, pp, u, v = attn_inputs(rng, T, d, tmax)
    got, _, checked = ref_attention_local(qkv, pp, u, v, np.array([0, T]), 1, d, H, tmax, *band, kernel=1, block=8)
    assert checked.all()
    want = brute_attention_local(qkv, pp, u, v, T, d, H, tmax, *band)
    assert np.abs(got - want).max() < 1e-12


def test_band_covering_the_utterance_is_full_attention(O, tiny):
    """Kernel level: ref_attention_local with band >= T is test_kernels_fp64.ref_attention; encoder level: the banded
    conformer_attention with band >= T is oracle.conformer_attention bit for bit."""
    from local_attention_oracle import conformer_attention_local
    rng = np.random.default_rng(4)
    d, H, T = 64, 2, 77
    qkv, pp, u, v = attn_inputs(rng, T, d, T)
    off = np.array([0, T])
    got, gb, _ = ref_attention_local(qkv, pp, u, v, off, 1, d, H, T, T, T, kernel=1)
    want, wb = ref_attention(qkv, pp, u, v, off, 1, d, H, T, MATH_X3, 1)
    assert np.abs(got - want).max() < 1e-12
    x = rng.standard_normal((50, tiny.ocfg.d_model)).astype(np.float32)
    pos = O.sinusoidal_position_embedding(50, tiny.ocfg.d_model)
    p = "encoder_.layers_.0.attn_."
    assert np.array_equal(conformer_attention_local(tiny.W, p, x, pos, tiny.ocfg, 50, 50), O.conformer_attention(tiny.W, p, x, pos, tiny.ocfg))


def test_chunked_subsampling_is_the_oracle_subsampling(O, synth, tiny):
    from local_attention_oracle import conv_subsampling_chunked
    f = O.preprocess_audio(synth.make_audio(16000 * 40, 5))
    want = O.conv_subsampling(tiny.W, f, tiny.ocfg)
    got = conv_subsampling_chunked(tiny.W, f, tiny.ocfg, rows=100)
    assert got.shape == want.shape and np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


# ------------------------------------------------------------------------------------------------- CPU: configuration
def test_presets_leave_the_band_zero_and_to_c_carries_it(pkg):
    L = pkg.load_library()
    c = pkg.engine._PkConfig()
    for preset in (L.pk_config_110m, L.pk_config_tdt_600m, L.pk_config_rnnt_600m, L.pk_config_nemotron_600m):
        c.local_att_left = c.local_att_right = 99
        preset(C.byref(c))
        assert (c.local_att_left, c.local_att_right) == (0, 0)
    s = pkg.engine._PkSortformerConfig()
    L.pk_config_sortformer_117m(C.byref(s))
    assert (s.enc.local_att_left, s.enc.local_att_right) == (0, 0)
    assert pkg.make_110m_config().local_attention == (0, 0)
    cc = pkg.make_110m_config(local_attention=(256, 17)).to_c()
    assert (cc.local_att_left, cc.local_att_right) == (256, 17)
    cc = pkg.make_tdt_600m_config(local_attention=(5, 0), att_context_left=3).to_c()
    assert (cc.local_att_left, cc.local_att_right) == (5, 0)


def test_cpp_fill_carries_the_band(tmp_path):
    src = tmp_path / "fill.cpp"
    src.write_text("""
#include "parakeet/transcribe.hpp"
#include <cstdio>
int main() {
    auto cfg = parakeet::make_110m_config();
    if (cfg.encoder.local_att_left != 0 || cfg.encoder.local_att_right != 0) return 1;
    cfg.encoder.local_att_left = 256; cfg.encoder.local_att_right = 17;
    pk_config c{};
    parakeet::detail::fill(c, cfg.encoder, cfg.prediction, cfg.joint, cfg.durations);
    std::printf("%d %d\\n", c.local_att_left, c.local_att_right);
    return 0;
}
""")
    exe = tmp_path / "fill"
    subprocess.run(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split() == ["256", "17"]


# ------------------------------------------------------------------------------------------------- GPU: kernels
@gpu
@pytest.mark.parametrize("kernel,math_mode", KERNELS, ids=["fp32", "mma-x3", "mma-x1"])
@pytest.mark.parametrize("cfg", [(128, 2), (512, 8), (1024, 8)], ids=lambda c: f"d{c[0]}h{c[1]}")
def test_local_attention_against_fp64(pkg, kernel, math_mode, cfg):
    """Every band on a ragged batch of the lengths around 64 and the band's edges, inside NaN sentinel rows, with the engine's
    table (tmax = max(left, right) + 1); then a 5,000-row utterance."""
    d, H = cfg
    worst = 0.0
    for bi, (left, right) in enumerate(BANDS):
        rng = np.random.default_rng(1000 * bi + d + kernel + math_mode)
        lens = list(rng.permutation(lengths_for(left, right)))
        off = np.concatenate([[3], 3 + np.cumsum(lens)]).astype(np.int32)
        rows = int(off[-1]) + 5
        tmax = max(left, right) + 1
        qkv, pp, u, v = attn_inputs(rng, rows, d, tmax, sentinel_rows=[0, 1, 2, *range(rows - 5, rows)])
        ref, bd, ck = ref_attention_local(qkv, pp, u, v, off, len(lens), d, H, tmax, left, right, kernel)
        r = check_local(run_local(pkg, kernel, math_mode, off, rows, d, H, tmax, left, right, qkv, pp, u, v), off, rows, ref, bd, ck)
        print(f"band {left},{right} kernel {kernel} math {math_mode} d {d}: error / bound {r:.3g}")
        worst = max(worst, r)
    rng = np.random.default_rng(77 + d)
    T, (left, right) = 5000, (256, 17)
    off = np.array([0, T], np.int32)
    qkv, pp, u, v = attn_inputs(rng, T, d, max(left, right) + 1)
    blocks = {0, 256, 2560, 4864}
    ref, bd, ck = ref_attention_local(qkv, pp, u, v, off, 1, d, H, max(left, right) + 1, left, right, kernel, blocks=blocks)
    r = check_local(run_local(pkg, kernel, math_mode, off, T, d, H, max(left, right) + 1, left, right, qkv, pp, u, v), off, T, ref, bd, ck)
    print(f"T 5000 band 256,17 kernel {kernel} math {math_mode} d {d}: error / bound {r:.3g}")
    assert max(worst, r) <= 1.0


@gpu
def test_local_attention_one_hour_utterance(pkg):
    """45,001 encoder frames (one hour of audio), band (256, 256), the mma kernel in the parity mode, d 512."""
    d, H, T, band = 512, 8, 45001, (256, 256)
    rng = np.random.default_rng(45001)
    off = np.array([2, 2 + T], np.int32)
    rows = T + 4
    tmax = max(band) + 1
    qkv, pp, u, v = attn_inputs(rng, rows, d, tmax, sentinel_rows=[0, 1, rows - 2, rows - 1])
    blocks = {0, 256, 22528, 44800}
    ref, bd, ck = ref_attention_local(qkv, pp, u, v, off, 1, d, H, tmax, *band, 1, blocks=blocks)
    r = check_local(run_local(pkg, 1, MATH_X3, off, rows, d, H, tmax, *band, qkv, pp, u, v), off, rows, ref, bd, ck)
    print(f"T 45001 band 256,256 mma-x3: error / bound {r:.3g}")
    assert r <= 1.0


@gpu
@pytest.mark.parametrize("kernel,math_mode", [(0, MATH_F32), (1, MATH_X3)], ids=["fp32", "mma-x3"])
def test_local_attention_bound_rejects_mutations(pkg, kernel, math_mode):
    d, H, band = 512, 8, (16, 16)
    lens = [65, 300, 40]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    M, tmax = int(off[-1]), max(band) + 1
    rng = np.random.default_rng(12)
    qkv, pp, u, v = attn_inputs(rng, M, d, tmax)
    out = run_local(pkg, kernel, math_mode, off, M, d, H, tmax, *band, qkv, pp, u, v)
    ref, bd, ck = ref_attention_local(qkv, pp, u, v, off, len(lens), d, H, tmax, *band, kernel)
    assert check_local(out, off, M, ref, bd, ck) <= 1.0
    for name, kw in (("left edge + 1", dict(widen=(1, 0))), ("left edge - 1", dict(widen=(-1, 0))), ("right edge + 1", dict(widen=(0, 1))),
                     ("right edge - 1", dict(widen=(0, -1))), ("pos_bias_u dropped", dict(drop_u=True))):
        mref, _, _ = ref_attention_local(qkv, pp, u, v, off, len(lens), d, H, tmax, *band, kernel, **kw)
        r = check_local(out, off, M, mref, bd, ck)
        print(f"mutation {name}: error / bound {r:.3g}")
        assert r > 1.0, name


@gpu
@pytest.mark.parametrize("kernel,math_mode", KERNELS, ids=["fp32", "mma-x3", "mma-x1"])
def test_band_covering_the_batch_is_byte_identical_to_full_kernels(pkg, kernel, math_mode):
    """The same tiles in the same order: a band >= the longest utterance gives the full kernel's bytes (the table rows of a
    relative position are the same values in both tables)."""
    d, H = 512, 8
    lens = [376, 1, 64, 129, 200]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    M, T = int(off[-1]), max(lens)
    rng = np.random.default_rng(5)
    qkv, _, u, v = attn_inputs(rng, M, d, T)
    W = T + 3
    pp_band = rng.uniform(-1, 1, (2 * W + 1, d)).astype(np.float32)        # relative positions -W..W
    pp_full = np.ascontiguousarray(pp_band[W - (T - 1):W + T])              # -(T-1)..T-1
    L = pkg.load_library()
    ro = np.ascontiguousarray(off)
    f32 = math_mode == MATH_F32
    full = [nan((M, d)) if f32 else None, None if f32 else nan((M, d)), nan((M, d)) if math_mode == MATH_X3 else None]
    assert L.pk_kernel_attention(0, kernel, math_mode, len(lens), i32p(ro), M, d, H, T, f32p(qkv), f32p(pp_full), f32p(u), f32p(v),
                                 *(f32p(a) for a in full), C.byref(C.c_int64(-1))) == 0
    band = run_local(pkg, kernel, math_mode, off, M, d, H, W + 1, W, W, qkv, pp_band, u, v)
    for a, b in zip(full, band):
        assert (a is None) == (b is None)
        if a is not None:
            assert a.tobytes() == b.tobytes()


# ------------------------------------------------------------------------------------------------- GPU: engine
def _tok_bytes(toks):
    return [np.array([(t.token_id, t.start_frame, t.end_frame) for t in r], np.int64).tobytes() +
            np.array([t.confidence for t in r], np.float32).tobytes() for r in toks]


@gpu
def test_band_covering_the_batch_is_byte_identical_to_full_engine(pkg, O, synth, tiny):
    cfg = dataclasses.replace(tiny.cfg, max_batch=4, max_samples=200000)
    Tmax = pkg.load_library().pk_encoder_frames(pkg.load_library().pk_mel_frames(cfg.max_samples))
    pcms = [synth.make_audio(n, 900 + i) for i, n in enumerate([176000, 30000, 400, 64000])]
    feats = [O.preprocess_audio(p) for p in pcms]
    res = {}
    # a band past T'max keeps the full table (2 T'max - 1 rows), whatever its width: up to INT32_MAX on both sides
    for name, band in (("full", (0, 0)), ("band", (Tmax, Tmax)), ("wide", (Tmax + 40, Tmax)), ("1e5", (100000, 100000)),
                       ("int32 max", (2 ** 31 - 1, 2 ** 31 - 1))):
        e = pkg.Engine(dataclasses.replace(cfg, local_attention=band), tiny.weights_path, 0)
        try:
            res[name] = ([x.tobytes() for x in e.encode(feats)], _tok_bytes(e.transcribe_batch(pcms, 0)), _tok_bytes(e.transcribe_batch(pcms, 1)))
        finally:
            e.close()
    for name in res:
        assert res[name] == res["full"], name


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@gpu
def test_tiny_ragged_batch_against_banded_oracle(pkg, O, synth, tiny):
    """Band (16, 16), a ragged batch of 60 min, 7 min, 10 s and 3 s: the encoder within the parity tolerance of the banded
    oracle (blockwise, so it runs at 45,001 frames).  CTC: the device's frame labels equal the oracle's on every frame whose top-two log-prob margin is wider than twice
    the device's log-prob error (and the tokens are identical when every frame is); TDT: the device decode of the banded
    oracle's encoder output gives the oracle's tokens and frames, and the whole path stays finite and in range."""
    band = (16, 16)
    cfg = dataclasses.replace(tiny.cfg, max_batch=4, max_samples=3600 * 16000, local_attention=band)
    pcms = [synth.make_audio(n, 1100 + i) for i, n in enumerate([3600 * 16000, 420 * 16000, 10 * 16000, 3 * 16000])]
    compare_against_banded_oracle(pkg, O, tiny, cfg, pcms, band)


def compare_against_banded_oracle(pkg, O, model, cfg, pcms, band):
    feats = [O.preprocess_audio(p, model.ocfg.mel_bins) for p in pcms]
    wants = [encoder_forward_local(model.W, f, model.ocfg, *band) for f in feats]
    blank = model.ocfg.vocab - 1
    e = pkg.Engine(cfg, model.weights_path, 0)
    try:
        encs = e.encode(feats)
        ctc, tdt = e.transcribe_batch(pcms, 0), e.transcribe_batch(pcms, 1)
        lps = [e.ctc_logprobs(g) for g in encs]
        tdt_of_oracle = e.decode(wants, 1)
        cap = e.cap
    finally:
        e.close()
    full_differs, tdt_compared = False, 0
    for f, got, want, c, t, lp_dev, tw in zip(feats, encs, wants, ctc, tdt, lps, tdt_of_oracle):
        assert _rel(got, want) < ENC_TOL
        if want.shape[0] < 2000:        # the dense full-attention oracle, where it fits in memory
            full_differs |= want.shape[0] > 40 and _rel(want, O.encoder_forward(model.W, f, model.ocfg)) > 10 * ENC_TOL
        lp = O.ctc_log_probs(model.W, want)
        err = float(np.abs(lp_dev - lp).max())
        top2 = np.sort(lp, axis=1)[:, -2:]
        clear = (top2[:, 1] - top2[:, 0]) > 2 * err + 1e-6
        assert np.array_equal(lp_dev.argmax(axis=1)[clear], lp.argmax(axis=1)[clear])
        if clear.all():
            assert [x.token_id for x in c] == O.ctc_greedy_decode(lp, blank=blank)
        print(f"T {want.shape[0]}: encoder rel {_rel(got, want):.3g}, log-prob error {err:.3g}, near-tie frames {int((~clear).sum())}")
        try:
            wt = O.tdt_greedy_decode(model.W, want, model.ocfg, with_timestamps=True, max_steps=4 * want.shape[0] + 1000)
        except RuntimeError:      # the reference algorithm livelocks on this input (tdt.cpp:66-104): the row is cut at capacity
            assert len(tw) == cap
        else:
            assert [(x.token_id, x.start_frame, x.end_frame) for x in tw] == [w[:3] for w in wt]
            tdt_compared += 1
        assert all(0 <= x.start_frame <= x.end_frame < want.shape[0] and np.isfinite(x.confidence) for x in t)
    assert tdt_compared >= 1
    assert full_differs, "the band changed nothing: the test would not see a kernel that ignores it"


@gpu
def test_110m_five_minutes_against_banded_oracle(pkg, O, synth, m110):
    """The 110m shape (d 512, 17 layers) on a 5-minute utterance with band (256, 256), compared with the banded oracle as the
    tiny batch is."""
    n = 300 * 16000
    cfg = dataclasses.replace(m110.cfg, max_batch=2, max_samples=n, local_attention=(256, 256))
    compare_against_banded_oracle(pkg, O, m110, cfg, [synth.make_audio(n, 300), synth.make_audio(37 * 16000, 301)], (256, 256))


def one_hour_run(pkg, synth, cfg, weights_path):
    """60 minutes, band (256, 256), max_batch 1: CTC (where the model has a head) and TDT; finite encoder output, token rows
    within the engine's capacity, monotone timestamps inside the utterance, device memory flat over three runs."""
    import torch
    n = 3600 * 16000
    cfg = dataclasses.replace(cfg, max_batch=1, max_samples=n, local_attention=(256, 256))
    pcm = synth.make_audio(n, 3600)
    e = pkg.Engine(cfg, weights_path, 0)
    try:
        T = e.L.pk_encoder_frames(e.L.pk_mel_frames(n))
        used = []
        for _ in range(3):
            for dec in ((0, 1) if cfg.has_ctc else (1,)):
                toks = e.transcribe_batch([pcm], dec)[0]
                assert 0 < len(toks) <= e.cap
                st = [t.start_frame for t in toks]
                assert st == sorted(st) and all(0 <= t.start_frame <= t.end_frame < T for t in toks)
                assert all(np.isfinite(t.confidence) for t in toks)
            free, total = torch.cuda.mem_get_info()
            used.append(total - free)
        # cudaMemGetInfo counts the whole card, which other processes share: a leak of this engine would grow by its per-run
        # allocations every run; allow 16 MiB of unrelated movement
        assert used[2] - used[1] <= 16 << 20 and used[1] - used[0] <= 16 << 20, used
        enc = e.encode(e.mel([pcm]))[0]
        assert enc.shape == (T, cfg.d_model) and np.all(np.isfinite(enc))
    finally:
        e.close()


@gpu
def test_110m_one_hour_utterance(pkg, synth, m110):
    one_hour_run(pkg, synth, m110.cfg, m110.weights_path)


@gpu
def test_600m_one_hour_utterance(pkg, O, synth, tmp_path):
    cfg = pkg.make_tdt_600m_config()
    wp = str(tmp_path / "tdt600m.safetensors")
    synth.save_safetensors(wp, synth.make_weights(O.make_tdt_600m_config(), seed=0))
    one_hour_run(pkg, synth, cfg, wp)


@gpu
def test_mel_normalisation_at_one_hour(pkg):
    """The per-utterance mel statistics of a 60-minute utterance (360,001 frames), as the engine's front end runs them,
    against test_frontend_fp64.ref_normalize: float64 normalisation of the kernel's own log-mel with its per-element bound."""
    from test_frontend_fp64 import ref_normalize, run_mel
    n = 3600 * 16000
    rng = np.random.default_rng(36)
    t = np.arange(n) / 16000.0
    pcm = (0.3 * np.sin(2 * np.pi * 440.0 * t) * (0.6 + 0.4 * np.sin(2 * np.pi * t / 900.0)) + rng.normal(0, 0.02, n)).astype(np.float32)
    worst = 0.0
    for n_mels in (80, 128):
        (lm,), (ft,) = run_mel(pkg, [pcm], n_mels, True)
        y, bd = ref_normalize(lm, n_mels)
        worst = max(worst, ratio(ft, y, bd))
    print(f"mel normalisation at one hour: error / bound {worst:.3g}")
    assert worst <= 1.0


@gpu
def test_band_refusals(pkg, tiny):
    with pytest.raises(RuntimeError, match=r"\(1\)"):
        pkg.Engine(dataclasses.replace(tiny.cfg, local_attention=(-1, 4)), tiny.weights_path, 0)
    with pytest.raises(RuntimeError, match=r"\(5\)"):
        pkg.Engine(dataclasses.replace(tiny.cfg, max_batch=1, max_samples=172_800_001, local_attention=(16, 16)), tiny.weights_path, 0)
    # a batch of more than 3 h of encoder frames in all (two utterances of 70,000 frames)
    e = pkg.Engine(dataclasses.replace(tiny.cfg, max_batch=2, max_samples=70000 * 1280, local_attention=(16, 16)), tiny.weights_path, 0)
    try:
        encs = [np.zeros((70000, tiny.cfg.d_model), np.float32)] * 2
        with pytest.raises(RuntimeError, match=r"\(5\).*3 h"):
            e.decode(encs, 1)
        assert len(e.decode(encs[:1], 1)) == 1
    finally:
        e.close()
    e = pkg.Engine(dataclasses.replace(tiny.cfg, local_attention=(16, 16)), tiny.weights_path, 0)
    try:
        assert e.L.pk_stream_open(e.h, 1, 16000, 12, 0) == 1
    finally:
        e.close()
    c = pkg.engine.make_tiny_sortformer_config().to_c()
    c.enc.local_att_left = 8
    h = C.c_void_p()
    assert e.L.pk_sortformer_create(C.byref(c), b"no.safetensors", 0, C.byref(h)) == 1 and "full attention" in e.L.pk_last_error(None).decode()
