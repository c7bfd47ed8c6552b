"""The boosted streaming decode of tests/boost_stream_oracle.py pinned to the two reference functions it composes (no device)."""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import boost_stream_oracle as BO  # noqa: E402

SCHEDULE = (2560, 1280, 0, 4000, 2560, 700, 2560, 2560)


def _enc_chunks(O, synth, ocfg, W, seed):
    pcm = synth.make_audio(sum(SCHEDULE), seed)
    pre, cache = O.StreamingPreprocessor(ocfg.mel_bins), O.StreamEncoderCache(ocfg.n_layers)
    pos, out = 0, []
    for n in SCHEDULE:
        f = pre.process_chunk(pcm[pos:pos + n])
        pos += n
        out.append(O.stream_encoder_chunk(W, f, cache, ocfg) if f is not None else None)
    return out


def test_empty_list_is_the_stream_oracle(O, synth):
    ocfg = O.make_tiny_stream_config()
    W = synth.make_weights(ocfg, seed=3)
    chunks = _enc_chunks(O, synth, ocfg, W, 77)
    a, b = O.StreamDecodeState(ocfg), BO.BoostStreamDecodeState(ocfg)
    n = 0
    for e in chunks:
        if e is None:
            continue
        want = O.stream_decode_chunk(W, e, a, ocfg, max_steps=2000)
        got = BO.boost_stream_decode_chunk(W, e, b, ocfg, O.ContextTrie(), 7.0, max_steps=2000)
        assert got == want
        n += len(want)
    assert n >= 4 and b.active == {0} and b.token == a.token and b.frame_offset == a.frame_offset


def test_one_chunk_from_a_fresh_state_is_the_offline_boosted_decode(O, synth, golden):
    ocfg = O.make_tiny_stream_config()
    W = synth.make_weights(ocfg, seed=3)
    enc = np.concatenate([e for e in _enc_chunks(O, synth, ocfg, W, 78) if e is not None], axis=0)
    T = enc.shape[0]
    hyp = [x[0] for x in O.tdt_greedy_decode(W, enc, ocfg, with_timestamps=True, max_steps=3000)]
    # lists [hyp[0], x]: x is boosted only right after hyp[0] was emitted.  Scores are swept because the tiny model's logits
    # are far apart: a small score changes nothing and a large one makes the reference loop on zero-duration emissions.
    changed = compared = 0
    for boost in (3.0, 6.0, 12.0, 25.0, 50.0, 100.0):
        for x in range(0, ocfg.vocab - 1, 3):
            trie = O.ContextTrie([[hyp[0], x], [x, hyp[0]]])
            try:
                want = O.tdt_greedy_decode_with_timestamps_boosted(W, enc, ocfg, trie, boost, max_steps=400)
            except RuntimeError:
                continue
            got = BO.boost_stream_decode_chunk(W, enc, BO.BoostStreamDecodeState(ocfg), ocfg, trie, boost, max_steps=400)
            assert [g[:2] for g in got] == [w[:2] for w in want]
            assert [g[3] for g in got] == [w[3] for w in want]
            assert [min(g[2], T - 1) for g in got] == [w[2] for w in want]      # the offline decode clamps the end frame
            compared += 1
            changed += [w[0] for w in want] != hyp
    assert compared >= 10
    # the same property where the boosts are known to alter the decode: the compiled reference's boost cases on the tiny
    # offline model (the decode functions do not care which encoder made the rows)
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_boost_v1.npz"))
    tcfg = O.make_tiny_config()
    Wt = synth.make_weights(tcfg, seed=3)
    for n in range(int(g["n_cases"][0])):
        k = f"boost.k{n}."
        if int(g[k + "tdt_livelock"][0]):
            continue
        offs = np.concatenate([[0], np.cumsum(g[k + "ph_len"])])
        trie = O.ContextTrie([g[k + "ph_ids"][offs[i]:offs[i + 1]].tolist() for i in range(len(offs) - 1)])
        enc_t = golden[f"tiny.c{int(g[k + 'clip'][0])}.enc"]
        got = BO.boost_stream_decode_chunk(Wt, enc_t, BO.BoostStreamDecodeState(tcfg), tcfg, trie, float(g[k + "boost"][0]), max_steps=3000)
        assert [[x[0], x[1], min(x[2], len(enc_t) - 1)] for x in got] == g[k + "tdt_tok"].tolist(), n
        assert np.allclose([x[3] for x in got], g[k + "tdt_conf"], rtol=1e-3, atol=1e-6)
        changed += [x[0] for x in got] != [x[0] for x in golden[f"tiny.c{int(g[k + 'clip'][0])}.tdt_tok"].tolist()]
    assert changed >= 3


def test_new_entry_points_are_exported(pkg):
    L = pkg.load_library()
    for sym in ("pk_set_boost_rows", "pk_stream_set_boost", "pk_kernel_tdt_decode_boosted"):
        assert sym in pkg.engine.EXPORTS and getattr(L, sym)
    ids, off, row = pkg.engine.pack_phrase_lists([[[1, 2], [3]], [], [[4]]])
    assert ids.tolist() == [1, 2, 3, 4] and off.tolist() == [0, 2, 3, 4] and row.tolist() == [0, 2, 2, 3]
