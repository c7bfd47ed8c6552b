"""numpy restatement of the reference's RNN-T model family (test infrastructure, next to oracle/oracle.py whose
encoder, prediction net and helpers it reuses).

    RNNTJoint::forward                     src/rnnt.cpp:37-44
    rnnt_greedy_decode(_with_timestamps)   src/rnnt.cpp:56-177
    make_rnnt_600m_config                  include/parakeet/config.hpp:118-135
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import oracle as O  # noqa: E402

F32 = np.float32


def make_rnnt_600m_config() -> O.Config:
    """config.hpp:118-135: the 600m encoder with 80 mels, a 1025-token vocabulary, no duration head; ParakeetRNNT
    registers "joint_" (rnnt.cpp:48-52)."""
    return O.Config(mel_bins=80, d_model=1024, n_layers=24, n_heads=8, ff=4096, vocab=1025, lstm_layers=2,
                    durations=(), has_ctc=False, joint_prefix="joint_.", name="rnnt-600m")


def make_tiny_rnnt_config() -> O.Config:
    """Not a reference preset: a small RNN-T shape for fast unit tests only."""
    return O.Config(mel_bins=80, sub_channels=64, d_model=128, n_layers=2, n_heads=2, ff=256, vocab=33, pred_hidden=64,
                    joint_hidden=64, durations=(), has_ctc=False, joint_prefix="joint_.", name="tiny-rnnt")


def rnnt_joint(W, enc_t, pred, cfg):
    """RNNTJoint::forward, rnnt.cpp:37-44: log_softmax(out_proj(relu(enc_proj(enc) + pred_proj(pred)))), pred_proj_
    without bias."""
    p = cfg.joint_prefix
    z = O.linear(enc_t, W[p + "enc_proj_.weight"], W[p + "enc_proj_.bias"]) + O.linear(pred, W[p + "pred_proj_.weight"])
    z = np.maximum(z, 0).astype(F32)
    return O.log_softmax(O.linear(z, W[p + "out_proj_.weight"], W[p + "out_proj_.bias"]))


def rnnt_greedy_decode(W, enc, cfg, max_symbols=10, with_timestamps=False):
    """rnnt_greedy_decode(_with_timestamps), rnnt.cpp:56-177: zero LSTM state, token = blank; per frame at most
    max_symbols emissions; blank reverts the state and advances; after max_symbols emissions the frame advances with
    the state and token of the last emission.  Timestamps are (id, t, t, exp(lp))."""
    T = enc.shape[0]
    blank = cfg.vocab - 1
    H = cfg.pred_hidden
    states = [(np.zeros(H, F32), np.zeros(H, F32)) for _ in range(cfg.lstm_layers)]
    token, out = blank, []
    for t in range(T):
        for _sym in range(max_symbols):
            saved = states
            pred, states = O.prediction_step(W, token, states, cfg)
            lp = rnnt_joint(W, enc[t], pred, cfg)
            k = O.first_argmax(lp)
            if k == blank:
                states = saved
                break
            out.append((k, t, t, float(np.exp(F32(lp[k])))) if with_timestamps else k)
            token = k
    return out


def transcribe(W, pcm, cfg, max_symbols=10, timestamps=False):
    """Transcriber::transcribe for an RNN-T model: mel -> encoder -> rnnt_greedy_decode."""
    enc = O.encoder_forward(W, O.preprocess_audio(pcm, cfg.mel_bins), cfg)
    return rnnt_greedy_decode(W, enc, cfg, max_symbols=max_symbols, with_timestamps=timestamps)
