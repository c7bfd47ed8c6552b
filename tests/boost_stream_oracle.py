"""Phrase-boosted streaming decode for the numpy oracle (test infrastructure, next to oracle/oracle.py).

The reference has no boosted streaming function.  The engine defines one (DESIGN.md section 8) as the composition of two
that exist, restated here from the oracle's own pieces:

    rnnt_streaming_decode_chunk                  src/eou.cpp:17-98         carried LSTM state and last token, absolute frame
                                                                            numbers, end frame not clamped to the chunk
    tdt_greedy_decode_with_timestamps_boosted    src/phrase_boost.cpp:266-352   boosted first maximum over the labels (durations
                                                                            are not boosted), ContextTrie::advance on every
                                                                            emission, confidence = exp(raw log-prob)

The active trie states live beside the decode state and are reset with it.  tests/test_boost_stream_oracle.py pins the
composition to what the reference does define: with an empty list it is stream_decode_chunk, and one chunk holding a whole
utterance from a fresh state is tdt_greedy_decode_with_timestamps_boosted up to the end-frame clamp.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import oracle as O  # noqa: E402


class BoostStreamDecodeState(O.StreamDecodeState):
    """StreamingDecodeState (eou.hpp:80-87) plus the active trie states (the root alone after a reset)."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.active = {0}


def boost_stream_decode_chunk(W, enc, st: BoostStreamDecodeState, cfg, trie: O.ContextTrie, boost=5.0, max_symbols=10,
                              max_steps=100000):
    """O.stream_decode_chunk with the label choice, trie advance and confidence of the boosted TDT decode."""
    C = enc.shape[0]
    blank = cfg.vocab - 1
    new, t, steps = [], 0, 0
    base = st.frame_offset
    while t < C:
        for _sym in range(max_symbols):
            steps += 1
            if steps > max_steps:
                raise RuntimeError("boost_stream_decode_chunk: livelock")
            saved = st.states
            pred, st.states = O.prediction_step(W, st.token, st.states, cfg)
            lab, dur = O.tdt_joint(W, enc[t], pred, cfg)
            tok = O._boosted_argmax(lab, trie.boosted(st.active), boost)
            di = O.first_argmax(dur)
            skip = cfg.durations[di] if di < len(cfg.durations) else 1
            if tok == blank:
                st.states = saved
                t += max(skip, 1)
                break
            new.append((tok, base + t, base + t + max(skip, 1) - 1, float(np.exp(O.F32(lab[tok])))))
            st.active = trie.advance(st.active, tok)
            st.tokens.append(tok)
            st.token = tok
            if skip > 0:
                t += skip
                break
    st.frame_offset += C
    return new
