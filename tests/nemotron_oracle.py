"""Configs of the reference's Nemotron streaming model for the numpy oracle (test infrastructure, next to oracle/oracle.py
whose streaming restatement -- StreamingPreprocessor, stream_encoder_chunk, stream_decode_chunk -- runs them unchanged:
NemotronTranscriber::transcribe_chunk takes the same steps as StreamingTranscriber::transcribe_chunk).

    make_nemotron_600m_config       include/parakeet/nemotron.hpp:33-54
"""
from __future__ import annotations

import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import oracle as O  # noqa: E402


def make_nemotron_600m_config(latency_frames=0) -> O.Config:
    """nemotron.hpp:33-54: d 1024, 24 layers, 8 heads (head_dim 128), ff 4096, 8193 labels, two LSTM layers; mel_bins is
    left at EncoderConfig's 80.  ParakeetNemotron registers "encoder_" / "prediction_" / "joint_" (nemotron.cpp:7-12)."""
    return O.Config(d_model=1024, n_layers=24, n_heads=8, ff=4096, vocab=8193, lstm_layers=2, has_ctc=False,
                    joint_prefix="joint_.", att_context_left=70, att_context_right=latency_frames, name="nemotron-600m")


def make_tiny_nemotron_config() -> O.Config:
    """Not a reference preset: a small streaming shape with Nemotron's head_dim 128 and two LSTM layers."""
    return O.Config(mel_bins=80, sub_channels=64, d_model=256, n_layers=2, n_heads=2, ff=512, vocab=33, pred_hidden=64,
                    lstm_layers=2, joint_hidden=64, has_ctc=False, joint_prefix="joint_.", att_context_left=12,
                    att_context_right=0, name="tiny-nemotron")
