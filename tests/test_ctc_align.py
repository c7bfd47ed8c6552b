"""CTC forced alignment (PK_DECODER_CTC_ALIGN, DESIGN.md section 15).

CPU: the float64 oracle (tests/ctc_align_oracle.py) against brute-force enumeration, torch's CTC loss and torchaudio's
forced_align.  GPU: the kernel through pk_kernel_ctc_align against the oracle, the engine end to end (aligning the greedy
transcript gives back the greedy row), batching and graph replay, the rejections, the other decodes left untouched, device
memory, and the C++ Transcriber::align.  Every comparison of paths first requires each decision of the oracle to clear
1e-9 (and what the log-prob error could move), so a near tie fails loudly instead of flipping."""
from __future__ import annotations

import ctypes as C
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_align_oracle as A  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
PK_ERR_INVALID, PK_ERR_CAPACITY = 1, 5
NEG = -math.inf


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


# ------------------------------------------------------------------ CPU: the oracle
@pytest.mark.parametrize("T", [0, 1, 2, 3, 4, 5, 6])
def test_oracle_equals_brute_force(T):
    n_feasible = n_infeasible = n_repeat = 0
    for V in (2, 3, 4):
        rng = np.random.default_rng(10 * T + V)
        for k in range(8):
            lp = A.make_logprobs(rng, T, V, peak=float(rng.uniform(0, 3)))
            y = A.targets_with_repeats(rng, int(rng.integers(0, 5)), V, p_repeat=0.5)
            res = A.align(lp, y)
            best, paths, tot = A.brute_force(lp, y)
            if not A.feasible(T, y):
                n_infeasible += 1
                assert best == NEG and res["score"] == NEG and res["loglik"] == NEG and res["tokens"] == []
                assert res["path"] == [-1] * T
                continue
            n_feasible += 1
            n_repeat += any(y[i] == y[i + 1] for i in range(len(y) - 1))
            assert math.isclose(res["score"], best, rel_tol=1e-12, abs_tol=1e-12)
            assert res["labels"] in paths
            if len(paths) == 1:
                assert A.min_margin(res) > 0.0
            assert math.isclose(res["loglik"], tot, rel_tol=1e-12, abs_tol=1e-12)
            assert [t[0] for t in res["tokens"]] == y
    assert n_feasible > 0
    if T >= 3:
        assert n_infeasible > 0 and n_repeat > 0


def test_oracle_loglik_matches_torch_ctc_loss():
    import torch
    rng = np.random.default_rng(5)
    n = 0
    for T in (1, 7, 40, 126):
        for V in (5, 33):
            for L in (0, 1, T // 3, T // 2):
                y = A.targets_with_repeats(rng, L, V)
                if not A.feasible(T, y) or (L == 0 and T == 0):
                    continue
                lp = A.make_logprobs(rng, T, V)
                want = -torch.nn.functional.ctc_loss(torch.from_numpy(lp.astype(np.float64))[:, None, :], torch.tensor(y, dtype=torch.long),
                                                     torch.tensor([T]), torch.tensor([L]), blank=V - 1, reduction="none").item()
                assert math.isclose(A.align(lp, y)["loglik"], want, rel_tol=1e-9), (T, V, L)
                n += 1
    assert n >= 20


def test_oracle_path_matches_torchaudio_forced_align():
    import torch
    import torchaudio.functional as F
    rng = np.random.default_rng(11)
    n = 0
    while n < 40:
        T, V = int(rng.integers(1, 80)), int(rng.choice([5, 33]))
        y = A.targets_with_repeats(rng, int(rng.integers(1, max(2, T // 2))), V)
        if not A.feasible(T, y):
            continue
        lp = A.make_logprobs(rng, T, V, peak=float(rng.uniform(0, 3)))
        res = A.align(lp, y)
        if not A.margins_clear(res):                        # a near tie: either answer is right
            continue
        labels, _ = F.forced_align(torch.from_numpy(lp.astype(np.float64))[None], torch.tensor([y], dtype=torch.int32), blank=V - 1)
        assert labels[0].tolist() == res["labels"]
        n += 1


# ------------------------------------------------------------------ GPU: the kernel against the oracle
def hook(pkg, lps, targets, cap=None):
    """pk_kernel_ctc_align on [T][V] log-prob matrices -> (tokens per row, score, loglik, path)."""
    L = pkg.load_library()
    V = lps[0].shape[1]
    n = len(lps)
    off = np.zeros(n + 1, np.int32)
    off[1:] = np.cumsum([x.shape[0] for x in lps])
    toff = np.zeros(n + 1, np.int32)
    toff[1:] = np.cumsum([len(y) for y in targets])
    rows = int(off[-1])
    lp = np.ascontiguousarray(np.concatenate(lps) if rows else np.zeros((1, V), np.float32), np.float32)
    tg = np.array([c for y in targets for c in y] or [0], np.int32)
    cap = cap or max(1, max(len(y) for y in targets) + 8)
    tok = np.zeros((n, 1 + cap), np.int32)
    st, en, cf = np.zeros((n, cap), np.int32), np.zeros((n, cap), np.int32), np.zeros((n, cap), np.float32)
    sc, ll, path = np.zeros(n), np.zeros(n), np.zeros(max(rows, 1), np.int32)
    gb = C.c_int64(-1)
    i32, f32, f64 = C.c_int32, C.c_float, C.c_double
    s = L.pk_kernel_ctc_align(0, n, _p(off, i32), rows, V, _p(lp, f32), _p(tg, i32), _p(toff, i32), cap, _p(tok, i32), _p(st, i32),
                              _p(en, i32), _p(cf, f32), _p(sc, f64), _p(ll, f64), _p(path, i32), C.byref(gb))
    assert s == 0, f"pk_kernel_ctc_align -> {s}"
    assert gb.value == 0, "a guard band was written"
    out = []
    for b in range(n):
        k = int(tok[b, 0])
        out.append([(int(tok[b, 1 + i]), int(st[b, i]), int(en[b, i]), float(cf[b, i])) for i in range(k)])
    return out, sc, ll, path[:rows]


def _check_hook(got, sc, ll, path, lps, targets):
    r0 = 0
    for b, (lp, y) in enumerate(zip(lps, targets)):
        ref = A.align(lp, y)
        T = lp.shape[0]
        assert [t[:3] for t in got[b]] == [t[:3] for t in ref["tokens"]], b
        assert path[r0:r0 + T].tolist() == ref["path"], b
        assert sc[b] == ref["score"], (b, sc[b], ref["score"])                    # bit-identical
        if ref["loglik"] == NEG:
            assert ll[b] == NEG
        else:
            assert math.isclose(ll[b], ref["loglik"], rel_tol=1e-12, abs_tol=1e-12), (b, ll[b], ref["loglik"])
        # confidence = expf(lp[start][token]): within the 2 ulp of the device expf
        assert np.allclose([t[3] for t in got[b]], [np.exp(np.float64(lp[t[1], t[0]])) for t in got[b]], rtol=3e-7, atol=0)
        r0 += T


def _geometry(V, seed):
    """Rows of T 0..400, each with a random L up to the feasible limit, the limit itself, one past it, L = 0, repeats."""
    rng = np.random.default_rng(seed)
    while True:
        lps, targets = [], []
        for T in (0, 1, 2, 3, 17, 126, 126, 126, 250, 400, 400, 64):
            lps.append(A.make_logprobs(rng, T, V, sigma=float(rng.uniform(0.5, 2.0)), peak=float(rng.uniform(1.0, 5.0))))
            gen = A.targets_with_repeats(rng, T + 4, V, p_repeat=0.4)
            lim = A.max_feasible_len(T, gen)
            k = len(lps) % 4
            L = [lim, int(rng.integers(0, lim + 1)), min(lim + 1, len(gen)), 0][k]
            targets.append(gen[:L])
        targets[-1] = [5 % (V - 1)] * 20                   # a run of repeats: 39 frames needed
        if all(A.margins_clear(A.align(lp, y)) for lp, y in zip(lps, targets)):
            return lps, targets
        seed += 1000                                       # a decision within 1e-9: reseed, never loosen the bound
        rng = np.random.default_rng(seed)


@gpu
@pytest.mark.parametrize("V", [33, 1025, 8193])
def test_kernel_hook_matches_the_oracle(pkg, V):
    lps, targets = _geometry(V, V)
    got, sc, ll, path = hook(pkg, lps, targets)
    _check_hook(got, sc, ll, path, lps, targets)
    n_inf = sum(not A.feasible(lp.shape[0], y) for lp, y in zip(lps, targets))
    assert n_inf >= 2 and any(len(y) == 0 and lp.shape[0] > 0 for lp, y in zip(lps, targets))
    assert got[0] == [] and sc[0] == 0.0                    # T = 0, L = 0: the empty path


@gpu
def test_kernel_hook_longest_row(pkg):
    rng = np.random.default_rng(2048)
    y = A.targets_with_repeats(rng, 2048, 33, p_repeat=0.05)
    T = 2048 + sum(y[i] == y[i + 1] for i in range(2047)) + 150
    for seed in range(20):
        lp = A.make_logprobs(np.random.default_rng(seed), T, 33, peak=3.0)
        if A.margins_clear(A.align(lp, y)):
            break
    else:
        pytest.fail("no seed whose decisions all clear 1e-9")
    got, sc, ll, path = hook(pkg, [lp], [y], cap=2100)
    _check_hook(got, sc, ll, path, [lp], [y])
    assert [t[0] for t in got[0]] == y


# ------------------------------------------------------------------ GPU: the engine
def _pcms(synth):
    return [synth.make_audio(n, s) for s, n in ((61, 40000), (62, 9000), (63, 26000), (64, 17000))]


def _ids(rows):
    return [[t.token_id for t in r] for r in rows]


@gpu
@pytest.mark.parametrize("kind", ["tiny", "110m"])
def test_aligning_the_greedy_transcript_gives_back_the_greedy_row(pkg, synth, tiny, m110, kind):
    mdl = tiny if kind == "tiny" else m110
    eng = pkg.Engine(mdl.cfg, mdl.weights_path, 0)
    pcms = _pcms(synth)
    greedy = eng.transcribe_batch(pcms, pkg.Decoder.CTC)
    assert sum(len(r) for r in greedy) > 10
    eng.set_align_targets(_ids(greedy))
    for _ in range(3):                                      # eager, capture, replay
        got = eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)
        for g, w in zip(got, greedy):
            assert [(t.token_id, t.start_frame, t.end_frame) for t in g] == [(t.token_id, t.start_frame, t.end_frame) for t in w]
            assert np.allclose([t.confidence for t in g], [t.confidence for t in w], rtol=1e-6, atol=0)
        assert all(sc > NEG and ll >= sc for sc, ll in eng.align_scores(len(pcms)))
    eng.close()


@gpu
@pytest.mark.parametrize("kind", ["tiny", "110m"])
def test_decode_matches_the_oracle_on_the_device_log_probs(pkg, synth, tiny, m110, kind):
    mdl = tiny if kind == "tiny" else m110
    eng = pkg.Engine(mdl.cfg, mdl.weights_path, 0)
    pcms = _pcms(synth)
    encs = eng.encode(eng.mel(pcms))
    greedy = _ids(eng.decode(encs, pkg.Decoder.CTC))
    rng = np.random.default_rng(1)
    targets = [g[::2] + [int(rng.integers(0, mdl.cfg.vocab - 1))] for g in greedy]   # not the greedy answer: real choices
    for enc, y in zip(encs, targets):                       # one row at a time: the log-probs of pk_ctc_logprobs bit for bit
        lp = eng.ctc_logprobs(enc)
        ref = A.align(lp, y)
        assert A.margins_clear(ref), "a decision of the oracle is within 1e-9"
        eng.set_align_targets([y])
        got = eng.decode([enc], pkg.Decoder.CTC_ALIGN)[0]
        assert [(t.token_id, t.start_frame, t.end_frame) for t in got] == [t[:3] for t in ref["tokens"]]
        sc, ll = eng.align_scores(1)[0]
        assert sc == ref["score"]
        assert math.isclose(ll, ref["loglik"], rel_tol=1e-12)
    # the whole path gives the rows of pk_decode
    eng.set_align_targets(targets)
    assert eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN) == eng.decode(encs, pkg.Decoder.CTC_ALIGN)
    eng.close()


@gpu
def test_rows_are_independent_and_replays_follow_the_targets(pkg, synth, tiny):
    eng = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    pcms = _pcms(synth)
    encs = eng.encode(eng.mel(pcms))
    greedy = _ids(eng.transcribe_batch(pcms, pkg.Decoder.CTC))
    T = [e.shape[0] for e in encs]
    sets = [[greedy[0], [], greedy[2][1:], [3] * T[3]],                   # an empty row; an infeasible row
            [greedy[0][:-1], greedy[1], [7] * (T[1] + 1), greedy[3][::-1]]]
    want = []
    for ts in sets:
        rows = []
        for enc, y in zip(encs, ts):
            ref = A.align(eng.ctc_logprobs(enc), y)
            assert A.margins_clear(ref, 1e-4), "a decision within what the batch's log-prob rounding could move"
            rows.append((ref, y))
        want.append(rows)
    for k in range(6):                                      # alternating target sets over one captured graph
        ts = sets[k % 2]
        eng.set_align_targets(ts)
        got = eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)
        scores = eng.align_scores(len(pcms))
        for b, (g, (ref, y)) in enumerate(zip(got, want[k % 2])):
            assert [(t.token_id, t.start_frame, t.end_frame) for t in g] == [t[:3] for t in ref["tokens"]], (k, b)
            if ref["score"] == NEG:
                assert scores[b] == (NEG, NEG) and g == []
            else:
                assert math.isclose(scores[b][0], ref["score"], rel_tol=1e-4)
    # a row aligns the same alone as in the batch
    eng.set_align_targets(sets[0])
    batch = eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)
    for b in range(len(pcms)):
        eng.set_align_targets([sets[0][b]])
        alone = eng.transcribe_batch([pcms[b]], pkg.Decoder.CTC_ALIGN)[0]
        assert [(t.token_id, t.start_frame, t.end_frame) for t in alone] == [(t.token_id, t.start_frame, t.end_frame) for t in batch[b]]
    eng.close()


@gpu
def test_rejections(pkg, synth, tiny, tmp_path):
    L = pkg.load_library()
    eng = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    pcms = [synth.make_audio(20000, 5), synth.make_audio(30000, 6)]
    i32 = C.c_int32

    def set_raw(rows):
        flat = np.array([c for r in rows for c in r] or [0], np.int32)
        off = np.zeros(len(rows) + 1, np.int32)
        off[1:] = np.cumsum([len(r) for r in rows])
        return L.pk_set_align_targets(eng.h, _p(flat, i32), _p(off, i32), len(rows))

    with pytest.raises(RuntimeError, match="pk_set_align_targets first"):
        eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)
    assert set_raw([[1, 2], [tiny.cfg.vocab - 1]]) == PK_ERR_INVALID                 # the blank
    assert "row 1" in L.pk_last_error(eng.h).decode()
    assert set_raw([[-1]]) == PK_ERR_INVALID
    assert set_raw([[1] * 2049]) == PK_ERR_CAPACITY
    assert set_raw([[1]] * (tiny.cfg.max_batch + 1)) == PK_ERR_CAPACITY
    eng.set_align_targets([[1, 2]])
    with pytest.raises(RuntimeError, match="rows"):
        eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)                          # one row of targets, two utterances
    eng.transcribe_batch(pcms, pkg.Decoder.CTC)
    sc = np.zeros(2)
    assert L.pk_fetch_align_scores(eng.h, _p(sc, C.c_double), None) == PK_ERR_INVALID   # the last run was not an alignment
    eng.set_align_targets([[1, 2], [3]])
    assert len(eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)) == 2
    eng.set_align_targets([])
    with pytest.raises(RuntimeError, match="pk_set_align_targets first"):
        eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)
    # speaker-attributed transcription takes CTC or TDT only
    scfg = pkg.make_tiny_sortformer_config(max_batch=4, max_samples=64000)
    sp = str(tmp_path / "sf.safetensors")
    synth.save_safetensors(sp, synth.make_sortformer_weights(scfg, seed=1))
    diar = pkg.Engine(scfg, sp, 0)
    eng.set_align_targets([[1, 2], [3]])
    tok = eng._tokens(2)[0]
    buf, off = pkg.engine._pack(pcms)
    probs, tl = np.zeros((4096, 4), np.float32), np.zeros(2, np.int32)
    assert L.pk_transcribe_diarize_batch(eng.h, diar.h, pkg.engine._f32p(buf), pkg.engine._i64p(off), 2, int(pkg.Decoder.CTC_ALIGN),
                                         C.byref(tok), pkg.engine._f32p(probs), pkg.engine._i32p(tl)) == PK_ERR_INVALID
    eng.stage(buf, off)
    assert L.pk_run_transcribe_diarize_staged(eng.h, diar.h, int(pkg.Decoder.CTC_ALIGN)) == PK_ERR_INVALID
    assert L.pk_set_align_targets(diar.h, None, None, 0) == PK_ERR_INVALID          # a Sortformer engine
    diar.close()
    eng.close()
    rcfg = pkg.make_tiny_rnnt_config()
    wp = str(tmp_path / "r.safetensors")
    synth.save_safetensors(wp, synth.make_weights(rcfg, seed=3, blank_bias=-1.0))
    er = pkg.Engine(rcfg, wp, 0)
    with pytest.raises(RuntimeError, match="no CTC head"):
        er.set_align_targets([[1]])
    with pytest.raises(RuntimeError, match="no CTC head"):
        er.transcribe_batch(pcms[:1], pkg.Decoder.CTC_ALIGN)
    er.close()
    tr = pkg.Transcriber(wp, tiny.vocab_path, rcfg)
    with pytest.raises(ValueError, match="CTC head"):
        tr.align(pcms[0], "a")
    tr.engine.close()


@gpu
def test_other_decodes_are_unchanged_after_alignment(pkg, synth, tiny):
    pcms = _pcms(synth)

    def dumps(eng):
        eng.set_ctc_beam(4)
        return [eng.transcribe_packed(*pkg.engine._pack(pcms), d) for d in (pkg.Decoder.CTC, pkg.Decoder.CTC_BEAM, pkg.Decoder.TDT)]

    fresh = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    want = [{k: v.copy() for k, v in a.items()} for a in dumps(fresh)]
    fresh.close()
    eng = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    eng.set_align_targets(_ids(eng.transcribe_batch(pcms, pkg.Decoder.CTC)))
    for _ in range(3):
        eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)
    for g, w in zip(dumps(eng), want):                      # targets still set
        for k in w:
            assert g[k].tobytes() == w[k].tobytes(), k
    eng.close()


@gpu
def test_device_memory_stays_flat(pkg, synth, tiny):
    import torch
    eng = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    pcms = _pcms(synth)
    greedy = _ids(eng.transcribe_batch(pcms, pkg.Decoder.CTC))
    rng = np.random.default_rng(4)

    def run(k):
        eng.set_align_targets([g[:max(0, len(g) - int(rng.integers(0, 3)))] for g in greedy])
        return eng.transcribe_batch(pcms, pkg.Decoder.CTC_ALIGN)

    for k in range(3):
        run(k)

    def free():
        eng.sync()
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]

    f0 = free()
    for k in range(50):
        run(k)
    assert f0 - free() < (2 << 20), "alignment runs with changing targets grew device memory"
    eng.close()


# ------------------------------------------------------------------ the C++ drop-in
@gpu
def test_cpp_transcriber_align_matches_python(pkg, synth, tiny, tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path / "cpp_align_check")
    libdir = os.path.dirname(pkg.lib_path())
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"),
                    os.path.join(ROOT, "tests", "cpp_align_check.cpp"), "-L" + libdir, "-lparakeet_b200", "-L" + os.path.join(cuda, "lib64"),
                    "-lcudart", "-Wl,-rpath," + libdir, "-o", exe], check=True)
    wav = str(tmp_path / "a.wav")
    synth_clip = synth.make_audio(30000, 21)
    pcm16 = np.clip(np.round(synth_clip * 32767), -32768, 32767).astype("<i2")
    import wave
    with wave.open(wav, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(pcm16.tobytes())
    tr = pkg.Transcriber(tiny.weights_path, tiny.vocab_path, tiny.cfg)
    text = tr.transcribe(wav, pkg.Decoder.CTC).text
    assert text
    texts = [text, text.split(" ")[-1] if " " in text else text[: max(1, len(text) // 2)]]
    want = tr.align_batch([wav, wav], texts)
    out = subprocess.run([exe, tiny.weights_path, tiny.vocab_path, wav] + texts, check=True, capture_output=True,
                         text=True).stdout.splitlines()
    for line, r in zip(out, want):
        f = line.split("\t")
        assert f[0] == ("1" if r.aligned else "0") and f[1] == r.text
        assert f[2].split() == [f"{t.token_id}:{t.start_frame}:{t.end_frame}" for t in r.timestamped_tokens]
        assert f[3].split() == [w.word for w in r.word_timestamps]
        assert float(f[4]) == pytest.approx(r.log_prob, rel=1e-12) and float(f[5]) == pytest.approx(r.ctc_log_likelihood, rel=1e-12)
    assert out[2:] == ["batch ok"]
    tr.engine.close()
