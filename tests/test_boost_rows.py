"""Phrase boosting per request: a phrase list and score for each utterance of a batch (pk_set_boost_rows) and for each stream
(pk_stream_set_boost), with the trie state carried across chunks on the device.

Offline rows are checked against the compiled reference's fixtures (tests/golden/golden_boost_v1.npz: each case is one clip
with its own list and score); streams against tests/boost_stream_oracle.py, the composition DESIGN.md section 8 defines; the
decode kernel against a float64 replay of the same decode through pk_kernel_tdt_decode_boosted."""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import boost_stream_oracle as BO  # noqa: E402
import nemotron_oracle as NO  # noqa: E402
import test_decode_fp64 as D  # noqa: E402

pytestmark = pytest.mark.gpu
MATH = {"bf16x3": 0, "fp32": 2}


def _tt(toks):
    return [(t.token_id, t.start_frame, t.end_frame) for t in toks]


def _full(toks):
    return [(t.token_id, t.start_frame, t.end_frame, np.float32(t.confidence).tobytes()) for t in toks]


@pytest.fixture(scope="module")
def cases(golden):
    """The golden_boost_v1 cases: (phrases, score, encoder rows, reference CTC / TDT tokens and confidences)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "golden_boost_v1.npz"))
    out = []
    for n in range(int(g["n_cases"][0])):
        k = f"boost.k{n}."
        ids, lens = g[k + "ph_ids"], g[k + "ph_len"]
        offs = np.concatenate([[0], np.cumsum(lens)])
        ci = int(g[k + "clip"][0])
        out.append(dict(phrases=[ids[offs[i]:offs[i + 1]].tolist() for i in range(len(lens))], boost=float(g[k + "boost"][0]), clip=ci,
                        enc=golden[f"tiny.c{ci}.enc"], ctc=g[k + "ctc_tok"].tolist(), ctc_conf=g[k + "ctc_conf"],
                        tdt=g[k + "tdt_tok"].tolist(), tdt_conf=g[k + "tdt_conf"], livelock=bool(int(g[k + "tdt_livelock"][0]))))
    return out


@pytest.fixture(scope="module", params=["bf16x3", "fp32"])
def eng_tiny(request, pkg, tiny):
    e = pkg.Engine(dataclasses.replace(tiny.cfg, math=MATH[request.param]), tiny.weights_path, 0)
    yield e
    e.close()


def _mixed_rows(cases, dec):
    """Rows of one batch: every usable case (the same clip appears under several lists), an unboosted row after every second."""
    rows = []
    for i, c in enumerate(cases):
        if dec == "tdt" and c["livelock"]:
            continue
        rows.append(c)
        if i % 2 == 1:
            rows.append(dict(phrases=[], boost=0.0, clip=c["clip"], enc=c["enc"], plain=True))
    return rows


@pytest.mark.parametrize("dec", ["ctc", "tdt"])
def test_mixed_batch_matches_reference_goldens(pkg, eng_tiny, golden, cases, dec):
    decoder = pkg.Decoder.CTC if dec == "ctc" else pkg.Decoder.TDT
    rows = _mixed_rows(cases, dec)[:eng_tiny.cfg.max_batch]
    assert sum(1 for r in rows if not r.get("plain")) >= 4 and any(r.get("plain") for r in rows)
    encs = [r["enc"] for r in rows]
    eng_tiny.set_boost_rows([], [])
    off = eng_tiny.decode(encs, decoder)
    eng_tiny.set_boost_rows([r["phrases"] for r in rows], [r["boost"] for r in rows])
    got = eng_tiny.decode(encs, decoder)
    changed = 0
    for i, r in enumerate(rows):
        if r.get("plain"):
            # an unboosted row of a boosted batch: the same bytes as with boosting off, and the plain golden
            assert _full(got[i]) == _full(off[i]), i
            assert [list(t) for t in _tt(got[i])] == golden[f"tiny.c{r['clip']}.{dec}_tok"].tolist()
        else:
            assert [list(t) for t in _tt(got[i])] == r[dec], i
            assert np.allclose([t.confidence for t in got[i]], r[dec + "_conf"], rtol=1e-3, atol=1e-6), i
            changed += _tt(got[i]) != _tt(off[i])
    assert changed >= 3
    # permuting the rows permutes the results
    perm = np.random.default_rng(1).permutation(len(rows))
    eng_tiny.set_boost_rows([rows[j]["phrases"] for j in perm], [rows[j]["boost"] for j in perm])
    again = eng_tiny.decode([encs[j] for j in perm], decoder)
    assert [_full(a) for a in again] == [_full(got[j]) for j in perm]
    eng_tiny.set_boost_rows([], [])
    assert [_full(a) for a in eng_tiny.decode(encs, decoder)] == [_full(a) for a in off]


@pytest.mark.parametrize("dec", ["ctc", "tdt"])
def test_equivalences_and_graph_replay(pkg, eng_tiny, synth, cases, dec):
    """The same list on every row is pk_set_boost; n_rows = 0 clears; rows past n_rows are unboosted; and new lists on a batch
    shape whose CUDA graph is already captured give the new lists' results."""
    decoder = pkg.Decoder.CTC if dec == "ctc" else pkg.Decoder.TDT
    use = [c for c in cases if not (dec == "tdt" and c["livelock"])]
    a, b = use[0], use[1]
    pcms = [synth.make_audio(n, 40 + i) for i, n in enumerate((32000, 20000, 26000, 32000))]
    run = lambda: [_full(t) for t in eng_tiny.transcribe_batch(pcms, decoder)]  # noqa: E731
    eng_tiny.set_boost_rows([], [])
    plain = run()
    assert run() == plain and run() == plain                  # (the batch shape has its graph now)
    eng_tiny.set_boost(a["phrases"], 12.0)
    shared = run()
    assert shared != plain
    eng_tiny.set_boost([], 0.0)
    eng_tiny.set_boost_rows([a["phrases"]] * 4, [12.0] * 4)
    rows_a = run()
    assert rows_a == shared and run() == rows_a
    eng_tiny.set_boost_rows([b["phrases"]] * 4, [12.0] * 4)
    eng_tiny.set_boost(b["phrases"], 12.0)                     # replaces the per-row lists ...
    shared_b = run()
    eng_tiny.set_boost_rows([b["phrases"], a["phrases"]], [12.0, 12.0])   # ... and is replaced by them
    mixed = run()
    assert mixed[0] == shared_b[0] and mixed[1] == rows_a[1] and mixed[2:] == plain[2:]
    eng_tiny.set_boost_rows([], [])
    assert run() == plain


def test_rows_no_call_has_named_decode_unboosted(pkg, tiny, synth):
    """The first pk_set_boost_rows of an engine names ONE row; a larger batch follows: rows 1.. have never been written by
    any call and must decode exactly as with boosting off."""
    pcms = [synth.make_audio(n, 60 + i) for i, n in enumerate((24000, 32000, 20000, 28000, 32000))]
    for dec in (pkg.Decoder.CTC, pkg.Decoder.TDT):
        e = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
        try:
            plain = [_full(t) for t in e.transcribe_batch(pcms, dec)]
            first = plain[0][0][0]
            e.set_boost_rows([[[first, 7], [9]]], [12.0])
            got = [_full(t) for t in e.transcribe_batch(pcms, dec)]
            assert got[1:] == plain[1:]
            assert got[0] != plain[0]
            e.set_boost([[first, 7], [9]], 12.0)
            assert [_full(t) for t in e.transcribe_batch(pcms[:1], dec)] == got[:1]
        finally:
            e.close()


# ------------------------------------------------------------------ the decode kernel against float64
def _ref_boosted(inp, lists, boosts, act0=None):
    """Float64 replay of the boosted decode for every row of `inp` (tests/test_decode_fp64.py's seeded inputs): the LSTM and
    joint in float64, the boosted first maximum over the labels, raw-log-prob confidence, ContextTrie on emissions."""
    import oracle as O
    P, V, Dn, L, n, cap, carry = inp["P"], inp["V"], inp["D"], inp["L"], inp["n"], inp["cap"], inp["carry"]
    f64 = lambda a: np.asarray(a, np.float64)  # noqa: E731
    sig = lambda x: 1 / (1 + np.exp(-x))  # noqa: E731
    out = []
    for b in range(n):
        T = int(inp["off"][b + 1] - inp["off"][b])
        trie = O.ContextTrie(lists[b])
        active = set(act0[b]) if act0 is not None else {0}
        h = [f64(inp["h0"][l][b]) if carry else np.zeros(P) for l in range(L)]
        c = [f64(inp["c0"][l][b]) if carry else np.zeros(P) for l in range(L)]
        tok = int(inp["tok0"][b]) if carry else V - 1
        base = int(inp["fbase"][b]) if carry else 0
        t, em, steps = 0, [], 0
        while t < T and len(em) < cap and steps < inp["max_steps"]:
            steps += 1
            nh, nc, x = [], [], None
            for l in range(L):
                g = f64(inp["Whh"][l]) @ h[l] + (f64(inp["G0"][tok]) if l == 0 else f64(inp["Wih"][l]) @ x + f64(inp["bih"][l]))
                gi, gf, gg, go = (g[k * P:(k + 1) * P] for k in range(4))
                c2 = sig(gf) * c[l] + sig(gi) * np.tanh(gg)
                x = sig(go) * np.tanh(c2)
                nh.append(x), nc.append(c2)
            z = np.maximum(f64(inp["Wp"]) @ x + f64(inp["EP"][inp["off"][b] + t]), 0)
            lg = f64(inp["Wout"]) @ z + f64(inp["bout"])
            lab = lg[:V]
            boosted = lab.copy()
            for tk in trie.boosted(active):
                if tk < V:
                    boosted[tk] += boosts[b]
            li, di = int(np.argmax(boosted)), int(np.argmax(lg[V:]))
            skip = inp["durations"][di]
            if li == V - 1:
                t += max(skip, 1)
                continue
            lse = lab.max() + np.log(np.exp(lab - lab.max()).sum())
            end = base + t + max(skip, 1) - 1 if carry else min(t + max(skip, 1) - 1, T - 1)
            em.append((li, base + t, end, float(np.exp(lab[li] - lse))))
            active = trie.advance(active, li)
            h, c, tok = nh, nc, li
            t += skip
        out.append(dict(em=em, active=active, bits=trie.boosted(active), trie=trie))
    return out


def _run_boost_hook(pkg, inp, lists, boosts, act0, cluster, max_ctas, no_stage):
    """pk_kernel_tdt_decode_boosted on the inputs of a tests/test_decode_fp64.py case -> every output as numpy arrays."""
    L, E = pkg.load_library(), pkg.engine
    n, P, J, V, Lh, cap = inp["n"], inp["P"], inp["J"], inp["V"], inp["L"], inp["cap"]
    keep = []

    def ptr(a, t=C.c_float):
        a = np.ascontiguousarray(a, {C.c_float: np.float32, C.c_int32: np.int32, C.c_uint32: np.uint32, C.c_double: np.float64}[t])
        keep.append(a)
        return a.ctypes.data_as(C.POINTER(t))

    bi, bo = E.TdtBoostHookIn(), E.TdtBoostHookOut()
    hi, ho = bi.dec, bo.dec
    hi.P, hi.J, hi.V, hi.n_dur, hi.L, hi.max_sym = P, J, V, inp["D"], Lh, inp["max_sym"]
    for i, d in enumerate(inp["durations"]):
        hi.durations[i] = d
    hi.n_utt, hi.rows, hi.row_off = n, inp["rows"], ptr(inp["off"], C.c_int32)
    hi.EP, hi.G0 = ptr(inp["EP"]), ptr(inp["G0"])
    for l in range(Lh):
        hi.W_hh[l] = ptr(inp["Whh"][l])
        if l:
            hi.W_ih[l], hi.b_ih[l] = ptr(inp["Wih"][l]), ptr(inp["bih"][l])
    hi.W_p, hi.W_out, hi.b_out = ptr(inp["Wp"]), ptr(inp["Wout"]), ptr(inp["bout"])
    hi.cap, hi.max_steps, hi.carry = cap, inp["max_steps"], int(inp["carry"])
    if inp["carry"]:
        hi.h0, hi.c0 = ptr(inp["h0"]), ptr(inp["c0"])
        hi.tok0, hi.frame_base = ptr(inp["tok0"], C.c_int32), ptr(inp["fbase"], C.c_int32)
    hi.cluster, hi.max_ctas, hi.no_stage = cluster, max_ctas, int(no_stage)
    ids, off, row = E.pack_phrase_lists(lists)
    bi.phrase_ids, bi.phrase_off, bi.row_off = ptr(ids, C.c_int32), ptr(off, C.c_int32), ptr(row, C.c_int32)
    bi.boost = ptr(np.asarray(boosts, np.float32))
    a0, n0 = np.zeros((n, 64), np.int32), np.ones(n, np.int32)
    if act0 is not None:
        for b, st in enumerate(act0):
            a0[b, :len(st)] = sorted(st)
            n0[b] = len(st)
    bi.trie_active0, bi.trie_nact0 = ptr(a0, C.c_int32), ptr(n0, C.c_int32)
    o = dict(tok=np.zeros((n, 1 + cap), np.int32), t_start=np.zeros((n, cap), np.int32), t_end=np.zeros((n, cap), np.int32),
             t_conf=np.zeros((n, cap), np.float32), overflow=np.zeros(n, np.int32), tok_state=np.zeros(n, np.int32))
    for k, a in o.items():
        setattr(ho, k, a.ctypes.data_as(C.POINTER(C.c_float if a.dtype == np.float32 else C.c_int32)))
    o.update(trie_active=np.full((n, 64), -7, np.int32), trie_nact=np.zeros(n, np.int32), boost_bits=np.zeros((n, (V + 31) // 32), np.uint32))
    bo.trie_active = o["trie_active"].ctypes.data_as(C.POINTER(C.c_int32))
    bo.trie_nact = o["trie_nact"].ctypes.data_as(C.POINTER(C.c_int32))
    bo.boost_bits = o["boost_bits"].ctypes.data_as(C.POINTER(C.c_uint32))
    gb = C.c_int64(-1)
    o["status"] = L.pk_kernel_tdt_decode_boosted(0, C.byref(bi), C.byref(bo), C.byref(gb))
    o["guard_bad"] = gb.value
    o["geom"] = {k: getattr(ho, k) for k in ("grid", "cl", "upc", "opc", "out_in_smem", "wih_in_smem", "staged_ih", "wstage_rows")}
    return o


BOOST_KERNEL_CASES = ["110m-n33-cl4", "110m-n33-cl2", "600m-n16", "600m-n16-nostage", "carry-tdt", "clamp-tdt"]


@pytest.mark.parametrize("name", BOOST_KERNEL_CASES)
def test_boosted_decode_kernel_against_fp64(pkg, name):
    c = D.BY_NAME[name]
    inp = D.case_inputs(c)
    n, V = inp["n"], inp["V"]
    rng = np.random.default_rng(c.seed + 100)
    plain = D.case_ref(c)
    lists, boosts = [], []
    for b in range(n):
        hyp = [e[0] for e in plain["emis"][b]]
        if b % 3 == 1:
            lists.append([])                                   # every third row is unboosted
        else:
            ph = [rng.integers(0, V - 1, int(rng.integers(1, 4))).tolist() for _ in range(int(rng.integers(1, 5)))]
            if len(hyp) >= 2:
                ph.append(hyp[:2] + [int(rng.integers(0, V - 1))])
            lists.append(ph)
        boosts.append(float(rng.uniform(1.0, 9.0)))
    act0 = None
    if c.carry:      # the state a stream is in after emitting the first token of its first phrase
        act0 = [({0} | ({1} if lst else set())) for lst in lists]
        # a row without frames in this chunk enters in a non-root state and must leave in it
        idle = [b for b in range(n) if inp["off"][b + 1] == inp["off"][b] and act0[b] != {0}]
        assert idle, "the case needs a zero-frame row that has a list"
    ref = _ref_boosted(inp, lists, boosts, act0)
    got = _run_boost_hook(pkg, inp, lists, boosts, act0, c.cluster, c.max_ctas, c.no_stage)
    assert got["status"] == 0 and got["guard_bad"] == 0
    for k, v in c.expect:
        assert got["geom"][k] == v, (k, got["geom"])
    changed = 0
    for b in range(n):
        em = ref[b]["em"]
        k = len(em)
        assert got["tok"][b, 0] == k, b
        assert got["tok"][b, 1:1 + k].tolist() == [e[0] for e in em], b
        assert got["t_start"][b, :k].tolist() == [e[1] for e in em] and got["t_end"][b, :k].tolist() == [e[2] for e in em], b
        assert np.allclose(got["t_conf"][b, :k], [e[3] for e in em], rtol=2e-3, atol=1e-7), b
        assert np.all(got["tok"][b, 1 + k:] == -1) and np.all(np.isnan(got["t_conf"][b, k:]))     # nothing past len was written
        na = int(got["trie_nact"][b])
        assert set(got["trie_active"][b, :na].tolist()) == ref[b]["active"], b
        bits = {w * 32 + i for w in range(got["boost_bits"].shape[1]) for i in range(32) if got["boost_bits"][b, w] >> i & 1}
        assert bits == {t for t in ref[b]["bits"] if t < V}, b
        if c.carry and inp["off"][b + 1] == inp["off"][b]:
            assert set(got["trie_active"][b, :na].tolist()) == act0[b] and k == 0, b       # idle: the entry state, untouched
        changed += [e[:3] for e in em] != [e[:3] for e in plain["emis"][b]]
        if not lists[b]:
            assert [e[:3] for e in em] == [e[:3] for e in plain["emis"][b]]
    assert changed >= 1                                        # the lists really alter the decode


# ------------------------------------------------------------------ streams
SCHED = [(2560, 2560, 1280, 0), (1280, 0, 2560, 4000), (2560, 2560, 0, 700), (0, 2560, 2560, 2560), (2560, 1280, 2560, 2560),
         (2560, 2560, 2560, 0), (1600, 2560, 0, 2560), (2560, 0, 2560, 2560)]


@pytest.fixture(scope="module", params=["eou", "nemotron"])
def stream_model(request, tmp_path_factory, pkg, O, synth):
    if request.param == "eou":
        ocfg, cfg = O.make_tiny_stream_config(), pkg.make_tiny_stream_config()
    else:
        ocfg, cfg = NO.make_tiny_nemotron_config(), pkg.make_tiny_nemotron_config()
    W = synth.make_weights(ocfg, seed=3)
    path = str(tmp_path_factory.mktemp("boost_stream") / (request.param + ".safetensors"))
    synth.save_safetensors(path, W)
    S = 4
    pcm = [synth.make_audio(sum(s[i] for s in SCHED), 90 + i) for i in range(S)]
    chunks, pos = [], [0] * S
    for s in SCHED:
        chunks.append([pcm[i][pos[i]:pos[i] + s[i]] for i in range(S)])
        pos = [pos[i] + s[i] for i in range(S)]
    # the encoder rows of every stream and step, from an unboosted run with the taps on
    e = pkg.Engine(cfg, path, 0)
    e.stream_open(S, 5120)
    enc, plain = [], []
    for ch in chunks:
        t, _, en = e.stream_step(ch, taps=True)
        enc.append(en)
        plain.append([_tt(x) for x in t])
    e.close()
    return dict(ocfg=ocfg, cfg=cfg, W=W, path=path, S=S, chunks=chunks, enc=enc, plain=plain)


def _oracle_stream(m, i, phrases, boost, reset_every_chunk=False, events=None):
    """Stream i of the model through tests/boost_stream_oracle.py on the device's encoder rows.  events: {step: (phrases, boost)}
    = a new list installed before that step (the trie restarts at the root)."""
    import oracle as O
    trie, st, out = O.ContextTrie(phrases), BO.BoostStreamDecodeState(m["ocfg"]), []
    for k, en in enumerate(m["enc"]):
        ev = (events or {}).get(k)
        if ev is not None:
            trie, boost = O.ContextTrie(ev[0]), ev[1]
            st.active = {0}
        if reset_every_chunk:
            st.active = {0}
        e = en[i]
        out.append([x for x in BO.boost_stream_decode_chunk(m["W"], e, st, m["ocfg"], trie, boost, max_steps=4000)] if len(e) else [])
    return out


def _straddling_phrase(m, i):
    """A phrase whose boost reaches across a chunk boundary of stream i: it starts with the last token the unboosted stream
    emits in some chunk and continues with a token the stream does not emit next, at a score where the carried trie state
    changes the decode and a trie restarted at every chunk does not give the same result."""
    V = m["ocfg"].vocab
    for k in range(len(m["plain"]) - 1):
        if not m["plain"][k][i]:
            continue
        a = m["plain"][k][i][-1][0]
        for boost in (3.0, 6.0, 12.0, 25.0, 50.0, 100.0):
            for x in range(V - 1):
                if x == a:
                    continue
                try:
                    carry = _oracle_stream(m, i, [[a, x]], boost)
                    fresh = _oracle_stream(m, i, [[a, x]], boost, reset_every_chunk=True)
                except RuntimeError:
                    continue
                if carry[:k + 1] == fresh[:k + 1] and carry != fresh:
                    return [[a, x]], boost, carry
    return None


def test_streams_with_their_own_lists(pkg, stream_model):
    m = stream_model
    S, V = m["S"], m["ocfg"].vocab
    found = _straddling_phrase(m, 0)
    assert found is not None, "no phrase straddles a chunk boundary: the case generator needs another schedule"
    ph0, b0, want0 = found
    rng = np.random.default_rng(3)
    hyp2 = [t[0] for step in m["plain"] for t in step[2]]
    lists = [ph0, [], [hyp2[:2] + [int(rng.integers(0, V - 1))], rng.integers(0, V - 1, 2).tolist()], [rng.integers(0, V - 1, 1).tolist()]]
    boosts = [b0, 0.0, 5.0, 3.0]
    want = [want0] + [_oracle_stream(m, i, lists[i], boosts[i]) for i in range(1, S)]
    e = pkg.Engine(m["cfg"], m["path"], 0)
    try:
        e.stream_open(S, 5120)
        for i in range(S):
            e.stream_set_boost(i, lists[i], boosts[i])
        got = [e.stream_step(ch) for ch in m["chunks"]]
        for k in range(len(SCHED)):
            for i in range(S):
                assert _tt(got[k][i]) == [w[:3] for w in want[i][k]], (k, i)
                assert np.allclose([t.confidence for t in got[k][i]], [w[3] for w in want[i][k]], rtol=1e-3, atol=1e-6), (k, i)
        # the unboosted stream is the unboosted run; the straddling phrase changed stream 0 after the boundary
        assert [_tt(got[k][1]) for k in range(len(SCHED))] == [m["plain"][k][1] for k in range(len(SCHED))]
        assert [_tt(got[k][0]) for k in range(len(SCHED))] != [m["plain"][k][0] for k in range(len(SCHED))]
        # a second pass after a reset of every stream: the lists stay, the trie states restart (graphs are replayed now)
        e.stream_reset(-1)
        again = [e.stream_step(ch) for ch in m["chunks"]]
        assert [[_full(t) for t in st] for st in again] == [[_full(t) for t in st] for st in got]
    finally:
        e.close()
    # each stream equals a solo engine running only that stream
    for i in (0, 2):
        solo = pkg.Engine(m["cfg"], m["path"], 0)
        try:
            solo.stream_open(1, 5120)
            solo.stream_set_boost(0, lists[i], boosts[i])
            for k, ch in enumerate(m["chunks"]):
                assert _tt(solo.stream_step([ch[i]])[0]) == _tt(got[k][i]), (i, k)
        finally:
            solo.close()


def test_set_boost_and_reset_mid_stream_touch_one_stream(pkg, stream_model):
    m = stream_model
    S, V = m["S"], m["ocfg"].vocab
    rng = np.random.default_rng(4)
    hyp = [[t[0] for step in m["plain"] for t in step[i]] for i in range(S)]
    lists = [[hyp[i][:2] + [int(rng.integers(0, V - 1))], rng.integers(0, V - 1, 2).tolist()] for i in range(S)]
    new0 = [rng.integers(0, V - 1, 2).tolist(), hyp[0][1:3]]
    want = [_oracle_stream(m, 0, lists[0], 6.0, events={3: (new0, 4.0)}), _oracle_stream(m, 1, lists[1], 6.0),
            _oracle_stream(m, 2, lists[2], 6.0, events={5: ([], 0.0)}), _oracle_stream(m, 3, lists[3], 6.0)]
    e = pkg.Engine(m["cfg"], m["path"], 0)
    try:
        e.stream_open(S, 5120)
        for i in range(S):
            e.stream_set_boost(i, lists[i], 6.0)
        for k, ch in enumerate(m["chunks"]):
            if k == 3:
                e.stream_set_boost(0, new0, 4.0)
            if k == 5:
                e.stream_set_boost(2, [], 0.0)
            got = e.stream_step(ch)
            for i in range(S):
                assert _tt(got[i]) == [w[:3] for w in want[i][k]], (k, i)
        # pk_stream_reset of one stream: that stream starts over (frames from 0, trie at the root, list kept), the others go on
        e.stream_reset(1)
        first = e.stream_step(m["chunks"][0])
        ref1 = _oracle_stream(m, 1, lists[1], 6.0)
        assert _tt(first[1]) == [w[:3] for w in ref1[0]]
    finally:
        e.close()


# ------------------------------------------------------------------ errors
def test_errors_leave_the_engine_usable(pkg, tiny, synth, tmp_path):
    e = pkg.Engine(tiny.cfg, tiny.weights_path, 0)
    try:
        pcms = [synth.make_audio(20000, 5), synth.make_audio(24000, 6)]
        e.set_boost_rows([[[1, 2]], []], [4.0, 0.0])
        before = [_full(t) for t in e.transcribe_batch(pcms, pkg.Decoder.TDT)]
        rng = np.random.default_rng(0)
        big = [rng.integers(0, tiny.cfg.vocab - 1, 40).tolist() for _ in range(40)]      # ~1600 trie nodes
        with pytest.raises(RuntimeError, match=r"\(5\).*row 1.*1024"):
            e.set_boost_rows([[[1, 2]], big], [4.0, 4.0])
        with pytest.raises(RuntimeError, match=r"\(5\)"):
            e.set_boost_rows([[]] * (tiny.cfg.max_batch + 1), [0.0] * (tiny.cfg.max_batch + 1))
        assert [_full(t) for t in e.transcribe_batch(pcms, pkg.Decoder.TDT)] == before      # the earlier lists are still in force
        with pytest.raises(RuntimeError, match="no streams are open"):
            e.stream_set_boost(0, [[1]], 3.0)
    finally:
        e.close()
    scfg = pkg.make_tiny_stream_config()
    import oracle as O
    wp = str(tmp_path / "s.safetensors")
    synth.save_safetensors(wp, synth.make_weights(O.make_tiny_stream_config(), seed=3))
    es = pkg.Engine(scfg, wp, 0)
    try:
        es.stream_open(2, 2560)
        for bad in (-1, 2):
            with pytest.raises(RuntimeError, match="bad stream index"):
                es.stream_set_boost(bad, [[1]], 3.0)
        es.stream_set_boost(1, [[1]], 3.0)
        assert len(es.stream_step([synth.make_audio(2560, 1), synth.make_audio(2560, 2)])) == 2
    finally:
        es.close()
    rcfg = pkg.make_tiny_rnnt_config()
    wr = str(tmp_path / "r.safetensors")
    synth.save_safetensors(wr, synth.make_weights(rcfg, seed=3, blank_bias=-1.0))
    er = pkg.Engine(rcfg, wr, 0)
    try:
        with pytest.raises(RuntimeError, match="RNN-T"):
            er.set_boost_rows([[[3, 4]]], [2.0])
        er.set_boost_rows([[]], [0.0])                         # no phrase: allowed, as pk_set_boost
        assert len(er.transcribe_batch([synth.make_audio(20000, 5)], pkg.Decoder.RNNT)) == 1
    finally:
        er.close()


def test_sortformer_engine_refuses(pkg, synth, tmp_path):
    import sortformer_oracle as SO
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "golden_sortformer_v1.npz")))
    cfg = pkg.make_tiny_sortformer_config()
    path = str(tmp_path / "sf.safetensors")
    synth.save_safetensors(path, SO.golden_weights(cfg, g, "tiny", synth))
    eng = pkg.Engine(cfg, path, 0)
    try:
        for call in (lambda: eng.set_boost_rows([[[1, 2]]], [3.0]), lambda: eng.stream_set_boost(0, [[1]], 3.0)):
            with pytest.raises(RuntimeError, match=r"\(1\)"):
                call()
    finally:
        eng.close()
