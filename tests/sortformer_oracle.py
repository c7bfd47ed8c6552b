"""Numpy restatement of the reference's Sortformer diarization model (test infrastructure, next to oracle/oracle.py whose
offline FastConformer it reuses unchanged):

    Sortformer::forward / diarize / probs_to_segments     src/sortformer.cpp:50-122
    StreamingFastConformerEncoder::forward (xscaling)     src/streaming_encoder.cpp:399-423
    TransformerBlock::forward (pre_ln = false)            src/transformer.cpp:15-62
    preprocess_audio with normalize = false               src/audio.cpp:100-158, src/main.cpp:514-517

Configs are parakeet_cpp_b200.SortformerConfig objects (make_sortformer_117m_config / make_tiny_sortformer_config).
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import oracle as O  # noqa: E402

F32 = np.float32
FRAME_DURATION_S = F32(0.08)      # timestamp.hpp:31


def features(pcm, scfg):
    """preprocess_audio(normalize = false): log-mel (n_frames, mel_bins)."""
    return np.ascontiguousarray(O.log_mel_unnormalised(pcm, scfg.mel_bins).T)


def _enc_cfg(scfg) -> O.Config:
    e = scfg.encoder
    return O.Config(mel_bins=e.mel_bins, sub_channels=e.sub_channels, d_model=e.d_model, n_layers=e.n_layers, n_heads=e.n_heads,
                    ff=e.ff, conv_k=e.conv_k, xscaling=True, name="nest-encoder")


def nest_encoder(W, feats, scfg):
    """The offline FastConformer under "nest_encoder_." with the subsampling output times sqrt(d_model) (the reference
    scales after proj_'s bias)."""
    We = {k[len("nest_"):]: v for k, v in W.items() if k.startswith("nest_encoder_.")}
    cfg = _enc_cfg(scfg)
    x = O.conv_subsampling(We, feats, cfg)
    x = (x * F32(math.sqrt(float(cfg.d_model)))).astype(F32)
    pos = O.sinusoidal_position_embedding(x.shape[0], x.shape[1])
    for i in range(cfg.n_layers):
        x = O.conformer_block(We, i, x, pos, cfg)
    return x


def transformer_block(W, p, x, n_heads):
    """TransformerBlock::forward, post-norm (transformer.cpp:15-62)."""
    T, d = x.shape
    hd = d // n_heads
    q = O.linear(x, W[p + "mha_.q_proj.weight"], W[p + "mha_.q_proj.bias"]).reshape(T, n_heads, hd).transpose(1, 0, 2)
    k = O.linear(x, W[p + "mha_.k_proj.weight"], W[p + "mha_.k_proj.bias"]).reshape(T, n_heads, hd).transpose(1, 0, 2)
    v = O.linear(x, W[p + "mha_.v_proj.weight"], W[p + "mha_.v_proj.bias"]).reshape(T, n_heads, hd).transpose(1, 0, 2)
    scores = ((q @ k.transpose(0, 2, 1)) * F32(1.0 / math.sqrt(float(hd)))).astype(F32)
    o = (O.softmax(scores, axis=-1) @ v).transpose(1, 0, 2).reshape(T, d)
    o = O.linear(o, W[p + "mha_.out_proj.weight"], W[p + "mha_.out_proj.bias"])
    x = O.layer_norm((x + o).astype(F32), W[p + "norm1_.weight"], W[p + "norm1_.bias"])
    h = np.maximum(O.linear(x, W[p + "fc1_.weight"], W[p + "fc1_.bias"]), 0).astype(F32)
    h = O.linear(h, W[p + "fc2_.weight"], W[p + "fc2_.bias"])
    return O.layer_norm((x + h).astype(F32), W[p + "norm2_.weight"], W[p + "norm2_.bias"])


def forward(W, feats, scfg, taps=False):
    """Sortformer::forward of one utterance: features -> probs (T', max_speakers); taps: also the NEST encoder output, the
    transformer output and the speaker logits."""
    enc = nest_encoder(W, feats, scfg)
    x = O.linear(enc, W["projection_.weight"], W["projection_.bias"]).astype(F32)
    for i in range(scfg.t_layers):
        x = transformer_block(W, f"transformer_.layers_.{i}.", x, scfg.t_heads)
    h = np.maximum(x, 0).astype(F32)
    h = np.maximum(O.linear(h, W["first_hidden_.weight"], W["first_hidden_.bias"]), 0).astype(F32)
    logits = O.linear(h, W["output_proj_.weight"], W["output_proj_.bias"]).astype(F32)
    probs = O.sigmoid(logits)
    if taps:
        return probs, dict(enc=enc, trans=x, logits=logits)
    return probs


def probs_to_segments(probs, threshold=0.5):
    """Sortformer::probs_to_segments (sortformer.cpp:70-113) -> [(speaker, start s, end s)], sorted by start; equal starts
    keep speaker order (libstdc++'s std::sort for <= 16 segments)."""
    T, S = probs.shape
    segs = []
    for s in range(S):
        start = None
        for t in range(T):
            active = probs[t, s] > F32(threshold)
            if active and start is None:
                start = t
            elif not active and start is not None:
                segs.append((s, F32(start) * FRAME_DURATION_S, F32(t - 1) * FRAME_DURATION_S))
                start = None
        if start is not None:
            segs.append((s, F32(start) * FRAME_DURATION_S, F32(T - 1) * FRAME_DURATION_S))
    segs.sort(key=lambda g: g[1])            # Python's sort is stable
    return [(int(s), float(a), float(b)) for s, a, b in segs]


def diarize(W, pcm, scfg):
    return probs_to_segments(forward(W, features(pcm, scfg), scfg), scfg.activity_threshold)


def calibrated_weights(scfg, seed, clips, synth):
    """Seeded synthetic weights (synth.make_sortformer_weights) whose speaker activity changes over `clips` (16 kHz PCM):
    output_proj_'s bias puts every speaker's threshold (logit 0) in the middle of the widest gap between its logits inside
    their 30-70 % quantile band, so each speaker is active on some frames and inactive on others.  Returns (W, smallest
    |logit| over all frames and speakers): a threshold decision that close to 0 could flip under device rounding, so
    callers reject seeds whose margin is below theirs."""
    W = synth.make_sortformer_weights(scfg, seed=seed)
    W["output_proj_.bias"] = np.zeros(scfg.max_speakers, F32)
    lg = np.concatenate([forward(W, features(c, scfg), scfg, taps=True)[1]["logits"] for c in clips], axis=0)
    b = np.zeros(scfg.max_speakers, F32)
    for s in range(scfg.max_speakers):
        v = np.sort(lg[:, s].astype(np.float64))
        lo, hi = int(0.3 * len(v)), max(int(0.7 * len(v)), int(0.3 * len(v)) + 1)
        k = lo + int(np.argmax(np.diff(v[lo:hi + 1])))
        b[s] = F32(-(v[k] + v[k + 1]) / 2)
    W["output_proj_.bias"] = b
    # the reference adds the bias in fp32 after the product: recompute instead of shifting
    lg = np.concatenate([forward(W, features(c, scfg), scfg, taps=True)[1]["logits"] for c in clips], axis=0)
    return W, float(np.abs(lg).min())


def golden_weights(scfg, g, tag, synth):
    """The weights a golden file was made with: synth.make_sortformer_weights(seed) with the recorded output_proj_ bias."""
    W = synth.make_sortformer_weights(scfg, seed=int(g[tag + ".seed"]))
    W["output_proj_.bias"] = g[tag + ".spk_bias"].astype(F32)
    return W
