"""Numpy restatement of the reference's streaming Sortformer diarization (test infrastructure, next to sortformer_oracle.py):

    Sortformer::diarize_chunk                          src/sortformer.cpp:124-150
    AOSCCache                                          src/sortformer.cpp:9-38
    StreamingFastConformerEncoder::forward_chunk       src/streaming_encoder.cpp:430-472 (oracle.stream_encoder_chunk)
    preprocess_audio(chunk, {n_mels, normalize=false}) src/audio.cpp:100-158, per chunk (as diarize.cpp:82-85 calls it)

One call of diarize_chunk on one stream: the chunk's own centred log-mel; the NEST encoder's forward_chunk (leftover frames,
largest multiple of 8 subsampled, x sqrt(d), K/V caches of att_context_left rows, causal conv caches); if that yields no
frame the result is {} and the AOSC is NOT updated; else projection_ -> transformer_ -> speaker head on this chunk's
encoder rows only, the AOSC update, and probs_to_segments with chunk-local frame numbers.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sortformer_oracle as SO  # noqa: E402

O = SO.O
F32 = np.float32


class AOSCCache:
    """AOSCCache: a speaker arrives the first time its probability is > 0.5; within a frame in index order."""

    def __init__(self, max_speakers=4):
        self.active = [False] * max_speakers
        self.order = []

    def update(self, probs):
        for t in range(probs.shape[0]):
            for s in range(min(probs.shape[1], len(self.active))):
                if probs[t, s] > F32(0.5) and not self.active[s]:
                    self.active[s] = True
                    self.order.append(s)


def stream_cfg(scfg, att_context_left=70) -> O.Config:
    e = scfg.encoder
    return O.Config(mel_bins=e.mel_bins, sub_channels=e.sub_channels, d_model=e.d_model, n_layers=e.n_layers, n_heads=e.n_heads,
                    ff=e.ff, conv_k=e.conv_k, xscaling=True, att_context_left=att_context_left, att_context_right=0,
                    name="nest-encoder")


def encoder_weights(W):
    """The NEST encoder's weights under the oracle's "encoder_." prefix."""
    return {k[len("nest_"):]: v for k, v in W.items() if k.startswith("nest_encoder_.")}


class Stream:
    """One stream's EncoderCache and AOSCCache."""

    def __init__(self, scfg, att_context_left=70):
        self.cfg = stream_cfg(scfg, att_context_left)
        self.cache = O.StreamEncoderCache(self.cfg.n_layers)
        self.aosc = AOSCCache(scfg.max_speakers)
        self.frame_base = 0


def head(W, enc, scfg):
    """projection_ -> transformer_ -> speaker head on one chunk's encoder rows: (probs, logits)."""
    x = O.linear(enc, W["projection_.weight"], W["projection_.bias"]).astype(F32)
    for i in range(scfg.t_layers):
        x = SO.transformer_block(W, f"transformer_.layers_.{i}.", x, scfg.t_heads)
    h = np.maximum(x, 0).astype(F32)
    h = np.maximum(O.linear(h, W["first_hidden_.weight"], W["first_hidden_.bias"]), 0).astype(F32)
    logits = O.linear(h, W["output_proj_.weight"], W["output_proj_.bias"]).astype(F32)
    return O.sigmoid(logits), logits


def diarize_chunk(W, We, feats, st: Stream, scfg):
    """-> dict(probs [C][S] (C = 0: the reference's {}), enc [C][d], logits, segs (chunk-local), base)."""
    base = st.frame_base
    enc = O.stream_encoder_chunk(We, feats, st.cache, st.cfg)
    if enc is None:
        z = np.zeros((0, scfg.max_speakers), F32)
        return dict(probs=z, enc=np.zeros((0, scfg.d_model), F32), logits=z, segs=[], base=base)
    st.frame_base += enc.shape[0]
    probs, logits = head(W, enc, scfg)
    st.aosc.update(probs)
    return dict(probs=probs, enc=enc, logits=logits, segs=SO.probs_to_segments(probs, scfg.activity_threshold), base=base)


def chunk_features(pcm, scfg):
    """preprocess_audio(chunk, {n_mels = mel_bins, normalize = false}); an empty chunk has no frames."""
    if len(pcm) == 0:
        return np.zeros((0, scfg.mel_bins), F32)
    return SO.features(pcm, scfg)


def run_schedule(W, scfg, clips, sched, att_context_left=70):
    """sched[s] = chunk lengths of stream s (all the same count); clips[s] its audio.  -> per step a list over streams of
    diarize_chunk results, plus the final AOSC orders."""
    We = encoder_weights(W)
    streams = [Stream(scfg, att_context_left) for _ in clips]
    pos = [0] * len(clips)
    steps = []
    for k in range(len(sched[0])):
        row = []
        for s, c in enumerate(clips):
            n = sched[s][k]
            pcm = c[pos[s]:pos[s] + n]
            pos[s] += n
            r = diarize_chunk(W, We, chunk_features(pcm, scfg), streams[s], scfg)
            r["order"] = list(streams[s].aosc.order)
            row.append(r)
        steps.append(row)
    return steps


def split(n_total, chunk):
    """A clip of n_total samples as chunks of `chunk` samples (the last one shorter)."""
    return [min(chunk, n_total - o) for o in range(0, n_total, chunk)]


def calibrated_weights(scfg, seed, runs, synth, att_context_left=70):
    """sortformer_oracle.calibrated_weights on STREAMING logits: runs = [(clips, sched)]; output_proj_'s bias puts every
    speaker's threshold in the widest gap of its streaming logits inside their 30-70 % band.  Returns (W, smallest |logit|)."""
    W = synth.make_sortformer_weights(scfg, seed=seed)
    W["output_proj_.bias"] = np.zeros(scfg.max_speakers, F32)

    def logits():
        out = []
        for clips, sched in runs:
            for row in run_schedule(W, scfg, clips, sched, att_context_left):
                out += [r["logits"] for r in row if len(r["logits"])]
        return np.concatenate(out, axis=0)

    lg = logits()
    b = np.zeros(scfg.max_speakers, F32)
    for s in range(scfg.max_speakers):
        v = np.sort(lg[:, s].astype(np.float64))
        lo, hi = int(0.3 * len(v)), max(int(0.7 * len(v)), int(0.3 * len(v)) + 1)
        k = lo + int(np.argmax(np.diff(v[lo:hi + 1])))
        b[s] = F32(-(v[k] + v[k + 1]) / 2)
    W["output_proj_.bias"] = b
    return W, float(np.abs(logits()).min())

