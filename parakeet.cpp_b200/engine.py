"""ctypes binding of libparakeet_b200.so and a Python mirror of the reference's
high-level API (include/parakeet/transcribe.hpp:23-190 in the reference):

    Transcriber(weights_path, vocab_path, config=make_110m_config())
    .to_gpu()
    .transcribe(samples | path, decoder=Decoder.TDT, timestamps=False) -> TranscribeResult
    .transcribe(samples | path, TranscribeOptions(...))

plus `transcribe_batch`, which the reference lacks (it is batch-1 only,
transcribe.hpp:170-171).  There is no CPU path: if the CUDA library or a device
is missing, construction raises.
"""
from __future__ import annotations

import ctypes as C
import enum
import os
import struct
from dataclasses import dataclass, field, replace
from typing import List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))


def lib_path() -> str:
    # PK_LIB: a developer knob to load a variant build of the same sources (scratch/build_variant.py)
    return os.environ.get("PK_LIB") or os.path.join(_HERE, "libparakeet_b200.so")


class _PkConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "mel_bins", "sub_channels", "d_model", "n_layers", "n_heads", "ff", "conv_kernel", "vocab",
        "pred_hidden", "lstm_layers", "joint_hidden", "n_durations")] + [("durations", C.c_int32 * 8)] + \
        [(n, C.c_int32) for n in ("has_ctc", "joint_prefix_tdt", "max_symbols", "max_batch", "max_samples", "math",
                                  "local_att_left", "local_att_right")]


class _PkSortformerConfig(C.Structure):
    _fields_ = [("enc", _PkConfig)] + [(n, C.c_int32) for n in ("t_hidden", "t_layers", "t_heads", "t_ff", "max_speakers")]


class _PkTokens(C.Structure):
    _fields_ = [("cap", C.c_int32), ("ids", C.POINTER(C.c_int32)), ("start", C.POINTER(C.c_int32)),
                ("end", C.POINTER(C.c_int32)), ("conf", C.POINTER(C.c_float)), ("len", C.POINTER(C.c_int32))]


class TdtHookIn(C.Structure):
    """pk_tdt_hook_in (include/parakeet_b200.h)."""
    _fields_ = [(n, C.c_int32) for n in ("P", "J", "V", "n_dur")] + [("durations", C.c_int32 * 8)] + \
        [(n, C.c_int32) for n in ("L", "max_sym", "n_utt", "rows")] + \
        [("row_off", C.POINTER(C.c_int32)), ("EP", C.POINTER(C.c_float)), ("G0", C.POINTER(C.c_float)),
         ("W_hh", C.POINTER(C.c_float) * 4), ("W_ih", C.POINTER(C.c_float) * 4), ("b_ih", C.POINTER(C.c_float) * 4),
         ("W_p", C.POINTER(C.c_float)), ("W_out", C.POINTER(C.c_float)), ("b_out", C.POINTER(C.c_float)),
         ("cap", C.c_int32), ("max_steps", C.c_int32), ("carry", C.c_int32),
         ("h0", C.POINTER(C.c_float)), ("c0", C.POINTER(C.c_float)), ("tok0", C.POINTER(C.c_int32)),
         ("frame_base", C.POINTER(C.c_int32)), ("cluster", C.c_int32), ("max_ctas", C.c_int32), ("no_stage", C.c_int32)]


class TdtHookOut(C.Structure):
    """pk_tdt_hook_out (include/parakeet_b200.h)."""
    _fields_ = [("tok", C.POINTER(C.c_int32)), ("t_start", C.POINTER(C.c_int32)), ("t_end", C.POINTER(C.c_int32)),
                ("t_conf", C.POINTER(C.c_float)), ("overflow", C.POINTER(C.c_int32))] + \
        [(n, C.POINTER(C.c_float)) for n in ("h_hi", "h_lo", "z_hi", "z_lo", "lab_val", "dur_val")] + \
        [("lab_idx", C.POINTER(C.c_int32)), ("dur_idx", C.POINTER(C.c_int32)), ("lse", C.POINTER(C.c_double)),
         ("c_state", C.POINTER(C.c_float)), ("tok_state", C.POINTER(C.c_int32))] + \
        [(n, C.c_int32) for n in ("steps", "grid", "cl", "upc", "opc", "out_in_smem", "wih_in_smem", "staged_ih", "wstage_rows")]


class TdtBoostHookIn(C.Structure):
    """pk_tdt_boost_hook_in (include/parakeet_b200.h)."""
    _fields_ = [("dec", TdtHookIn), ("phrase_ids", C.POINTER(C.c_int32)), ("phrase_off", C.POINTER(C.c_int32)),
                ("row_off", C.POINTER(C.c_int32)), ("boost", C.POINTER(C.c_float)),
                ("trie_active0", C.POINTER(C.c_int32)), ("trie_nact0", C.POINTER(C.c_int32))]


class TdtBoostHookOut(C.Structure):
    """pk_tdt_boost_hook_out (include/parakeet_b200.h)."""
    _fields_ = [("dec", TdtHookOut), ("trie_active", C.POINTER(C.c_int32)), ("trie_nact", C.POINTER(C.c_int32)),
                ("boost_bits", C.POINTER(C.c_uint32))]


BOOST_ROW_NODES = 1024   # PK_BOOST_ROW_NODES: trie nodes (root included) one row's phrase list may make

EXPORTS = ["pk_config_110m", "pk_config_tdt_600m", "pk_config_rnnt_600m", "pk_config_nemotron_600m", "pk_engine_create", "pk_engine_destroy", "pk_last_error",
           "pk_mel_frames", "pk_encoder_frames", "pk_mel", "pk_encode", "pk_decode", "pk_ctc_logprobs",
           "pk_transcribe_batch", "pk_stage_pcm", "pk_prefetch_pcm", "pk_run_staged", "pk_fetch_tokens", "pk_sync",
           "pk_token_buffer", "pk_stream", "pk_launch_count", "pk_profile_begin", "pk_profile_end",
           "pk_profile_names", "pk_flush_l2", "pk_selftest_gemm",
           "pk_kernel_gemm", "pk_kernel_attention", "pk_kernel_attention_local", "pk_kernel_layernorm", "pk_kernel_dwconv", "pk_kernel_ctc_argmax", "pk_kernel_tdt_decode", "pk_kernel_stream_attention", "pk_kernel_stream_dwconv",
           "pk_debug_tdt_phases", "pk_vocab_load", "pk_vocab_free", "pk_vocab_size",
           "pk_detokenize", "pk_group_words", "pk_tokenize", "pk_ctc_decode_boosted",
           "pk_resample_len", "pk_resample",
           "pk_job_begin", "pk_job_append", "pk_nccl_unique_id", "pk_comm_init_rank", "pk_allgather_tokens",
           "pk_job_fetch", "pk_job_stage_pcm", "pk_job_select", "pk_truncated_count",
           "pk_stream_open", "pk_stream_reset", "pk_stream_step", "pk_stream_count", "pk_stage_pcm_rate", "pk_resample_batch",
           "pk_set_boost", "pk_vocab_max_piece_bytes", "pk_safetensors_probe", "pk_debug_tdt_passes",
           "pk_config_sortformer_117m", "pk_sortformer_create", "pk_sortformer_forward", "pk_diarize_batch", "pk_run_diarize_staged",
           "pk_fetch_probs", "pk_diar_segments", "pk_kernel_mha", "pk_kernel_speaker_head",
           "pk_diar_stream_open", "pk_diar_stream_reset", "pk_diar_stream_step", "pk_diar_stream_step_feats", "pk_diar_stream_speakers",
           "pk_diar_stream_count", "pk_set_boost_rows", "pk_stream_set_boost", "pk_kernel_tdt_decode_boosted",
           "pk_transcribe_diarize_batch", "pk_run_transcribe_diarize_staged", "pk_diarize_transcription", "pk_diarize_words",
           "pk_lm_load", "pk_lm_free", "pk_lm_order", "pk_lm_count", "pk_lm_sentence_log10", "pk_set_ctc_beam", "pk_kernel_ctc_beam",
           "pk_kernel_mel", "pk_kernel_mel_stream", "pk_kernel_subsample_conv1", "pk_kernel_subsample_dw",
           "pk_set_align_targets", "pk_fetch_align_scores", "pk_kernel_ctc_align"]

_lib = None


def load_library():
    """Load the CUDA extension; fails loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise RuntimeError(f"{p} is missing: build it with `python parakeet.cpp_b200/build.py` "
                           "(there is no CPU fallback)")
    L = C.CDLL(p)
    vp, i32p, f32p, i64p = C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int64)
    L.pk_config_110m.argtypes = [C.POINTER(_PkConfig)]
    L.pk_config_tdt_600m.argtypes = [C.POINTER(_PkConfig)]
    L.pk_config_rnnt_600m.argtypes = [C.POINTER(_PkConfig)]
    L.pk_config_nemotron_600m.argtypes = [C.POINTER(_PkConfig)]
    L.pk_engine_create.argtypes = [C.POINTER(_PkConfig), C.c_char_p, C.c_int, C.POINTER(vp)]
    L.pk_engine_destroy.argtypes = [vp]
    L.pk_last_error.argtypes = [vp]
    L.pk_last_error.restype = C.c_char_p
    L.pk_mel_frames.argtypes = [C.c_int64]
    L.pk_encoder_frames.argtypes = [C.c_int32]
    L.pk_mel.argtypes = [vp, f32p, i64p, C.c_int32, f32p, i32p]
    L.pk_encode.argtypes = [vp, f32p, i32p, C.c_int32, f32p, i32p, f32p, f32p]
    L.pk_decode.argtypes = [vp, f32p, i32p, C.c_int32, C.c_int, C.POINTER(_PkTokens)]
    L.pk_ctc_logprobs.argtypes = [vp, f32p, C.c_int32, f32p]
    L.pk_transcribe_batch.argtypes = [vp, f32p, i64p, C.c_int32, C.c_int, C.POINTER(_PkTokens)]
    L.pk_stage_pcm.argtypes = [vp, f32p, i64p, C.c_int32]
    L.pk_resample_len.argtypes = [C.c_int64, C.c_int32, C.c_int32]
    L.pk_resample_len.restype = C.c_int64
    L.pk_resample.argtypes = [f32p, C.c_int64, C.c_int32, C.c_int32, f32p, C.c_int64]
    L.pk_resample.restype = C.c_int64
    L.pk_tokenize.argtypes = [vp, C.c_char_p, i32p, C.c_int32]
    L.pk_tokenize.restype = C.c_int32
    L.pk_ctc_decode_boosted.argtypes = [f32p, C.c_int32, C.c_int32, C.c_int32, i32p, i32p, C.c_int32, C.c_float, i32p, i32p, i32p,
                                        f32p, C.c_int32]
    L.pk_ctc_decode_boosted.restype = C.c_int32
    L.pk_prefetch_pcm.argtypes = [vp, f32p, i64p, C.c_int32]
    L.pk_run_staged.argtypes = [vp, C.c_int]
    L.pk_fetch_tokens.argtypes = [vp, C.POINTER(_PkTokens)]
    L.pk_sync.argtypes = [vp]
    L.pk_token_buffer.argtypes = [vp, C.POINTER(vp), i32p, i32p]
    L.pk_stream.argtypes = [vp]
    L.pk_stream.restype = vp
    L.pk_launch_count.argtypes = [vp]
    L.pk_launch_count.restype = C.c_int64
    L.pk_profile_begin.argtypes = [vp]
    L.pk_profile_end.argtypes = [vp, C.POINTER(C.c_double), i64p, C.POINTER(C.c_double), C.c_int32]
    L.pk_profile_names.restype = C.c_char_p
    L.pk_flush_l2.argtypes = [vp]
    L.pk_debug_tdt_phases.argtypes = [vp, i64p]
    L.pk_debug_tdt_passes.argtypes = [vp, i64p]
    L.pk_selftest_gemm.argtypes = [C.c_int] * 6 + [C.c_uint32, f32p, f32p]
    L.pk_kernel_gemm.argtypes = [C.c_int] * 10 + [C.c_float, C.c_int] + [f32p] * 7 + [i64p]
    L.pk_kernel_attention.argtypes = [C.c_int] * 4 + [i32p] + [C.c_int] * 4 + [f32p] * 7 + [i64p]
    L.pk_kernel_attention_local.argtypes = [C.c_int] * 4 + [i32p] + [C.c_int] * 6 + [f32p] * 7 + [i64p]
    L.pk_kernel_layernorm.argtypes = [C.c_int] * 3 + [f32p] * 5 + [C.c_int] * 2 + [f32p] * 4 + [i64p]
    L.pk_kernel_dwconv.argtypes = [C.c_int] * 3 + [i32p] + [C.c_int] * 3 + [f32p] * 6 + [i64p]
    L.pk_kernel_ctc_argmax.argtypes = [C.c_int] * 4 + [f32p, i32p, f32p, f32p, i64p]
    L.pk_kernel_tdt_decode.argtypes = [C.c_int, C.POINTER(TdtHookIn), C.POINTER(TdtHookOut), i64p]
    L.pk_kernel_stream_attention.argtypes = [C.c_int] * 4 + [i32p, i32p, C.c_int, i32p, i32p] + [C.c_int] * 4 + [f32p] * 11 + [i64p]
    L.pk_kernel_stream_dwconv.argtypes = [C.c_int] * 4 + [i32p, i32p] + [C.c_int] * 3 + [f32p] * 8 + [i64p]
    L.pk_vocab_load.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.pk_vocab_free.argtypes = [vp]
    L.pk_vocab_size.argtypes = [vp]
    L.pk_vocab_max_piece_bytes.argtypes = [vp]
    L.pk_detokenize.argtypes = [vp, i32p, C.c_int32, C.c_char_p, C.c_int32]
    L.pk_group_words.argtypes = [vp, i32p, i32p, i32p, f32p, C.c_int32, C.c_char_p, C.c_int32, f32p, f32p, f32p]
    L.pk_job_begin.argtypes = [vp, C.c_int64, C.c_int32]
    L.pk_job_append.argtypes = [vp]
    L.pk_nccl_unique_id.argtypes = [C.c_char_p]
    L.pk_comm_init_rank.argtypes = [vp, C.c_char_p, C.c_int32, C.c_int32]
    L.pk_allgather_tokens.argtypes = [vp, vp]
    L.pk_job_fetch.argtypes = [vp, C.c_int32, i32p, C.c_int64, i32p]
    L.pk_job_stage_pcm.argtypes = [vp, f32p, i64p, C.c_int32]
    L.pk_job_select.argtypes = [vp, C.c_int32, C.c_int32]
    L.pk_truncated_count.argtypes = [vp]
    L.pk_stream_open.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    L.pk_stream_reset.argtypes = [vp, C.c_int32]
    L.pk_stream_step.argtypes = [vp, f32p, i64p, C.POINTER(_PkTokens), f32p, i32p, f32p, i32p]
    L.pk_stream_count.argtypes = [vp]
    L.pk_set_boost.argtypes = [vp, i32p, i32p, C.c_int32, C.c_float]
    L.pk_set_boost_rows.argtypes = [vp, i32p, i32p, i32p, f32p, C.c_int32]
    L.pk_stream_set_boost.argtypes = [vp, C.c_int32, i32p, i32p, C.c_int32, C.c_float]
    L.pk_kernel_tdt_decode_boosted.argtypes = [C.c_int, C.POINTER(TdtBoostHookIn), C.POINTER(TdtBoostHookOut), i64p]
    L.pk_safetensors_probe.argtypes = [C.c_char_p, C.c_char_p, f32p, C.c_int64, i64p]
    L.pk_stage_pcm_rate.argtypes = [vp, f32p, i64p, C.c_int32, C.c_int32]
    L.pk_resample_batch.argtypes = [vp, f32p, i64p, C.c_int32, C.c_int32, C.c_int32, f32p, i64p]
    L.pk_config_sortformer_117m.argtypes = [C.POINTER(_PkSortformerConfig)]
    L.pk_sortformer_create.argtypes = [C.POINTER(_PkSortformerConfig), C.c_char_p, C.c_int, C.POINTER(vp)]
    L.pk_sortformer_forward.argtypes = [vp, f32p, i32p, C.c_int32, f32p, i32p]
    L.pk_diarize_batch.argtypes = [vp, f32p, i64p, C.c_int32, f32p, i32p]
    L.pk_run_diarize_staged.argtypes = [vp]
    L.pk_fetch_probs.argtypes = [vp, f32p, i32p]
    L.pk_diar_segments.argtypes = [f32p, C.c_int32, C.c_int32, C.c_float, i32p, f32p, f32p, C.c_int32]
    L.pk_diar_segments.restype = C.c_int32
    L.pk_kernel_mha.argtypes = [C.c_int] * 3 + [i32p] + [C.c_int] * 3 + [f32p] * 4 + [i64p]
    L.pk_kernel_speaker_head.argtypes = [C.c_int] * 4 + [f32p] * 6 + [i64p]
    L.pk_diar_stream_open.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32]
    L.pk_diar_stream_reset.argtypes = [vp, C.c_int32]
    L.pk_diar_stream_step.argtypes = [vp, f32p, i64p, f32p, i32p, i32p, f32p]
    L.pk_diar_stream_step_feats.argtypes = [vp, f32p, i32p, f32p, i32p, i32p, f32p]
    L.pk_diar_stream_speakers.argtypes = [vp, C.c_int32, i32p, C.c_int32]
    L.pk_diar_stream_speakers.restype = C.c_int32
    L.pk_diar_stream_count.argtypes = [vp]
    L.pk_diar_stream_count.restype = C.c_int32
    L.pk_transcribe_diarize_batch.argtypes = [vp, vp, f32p, i64p, C.c_int32, C.c_int, C.POINTER(_PkTokens), f32p, i32p]
    L.pk_run_transcribe_diarize_staged.argtypes = [vp, vp, C.c_int]
    L.pk_diarize_transcription.argtypes = [f32p, f32p, C.c_int32, i32p, f32p, f32p, C.c_int32, i32p]
    L.pk_diarize_words.argtypes = [f32p, C.c_int32, C.c_int32, C.c_float, f32p, f32p, C.c_int32, i32p, i32p, f32p, f32p, C.c_int32]
    L.pk_diarize_words.restype = C.c_int32
    L.pk_lm_load.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.pk_lm_free.argtypes = [vp]
    L.pk_lm_order.argtypes = [vp]
    L.pk_lm_order.restype = C.c_int32
    L.pk_lm_count.argtypes = [vp, C.c_int32]
    L.pk_lm_count.restype = C.c_int64
    L.pk_lm_sentence_log10.argtypes = [vp, C.c_char_p]
    L.pk_lm_sentence_log10.restype = C.c_double
    L.pk_set_ctc_beam.argtypes = [vp, C.c_int32, vp, vp, C.c_float, C.c_float]
    L.pk_kernel_ctc_beam.argtypes = [C.c_int, C.c_int, i32p, C.c_int, C.c_int, f32p, C.c_int, vp, vp, C.c_float, C.c_float, C.c_int,
                                     i32p, i32p, i32p, f32p, i32p, f32p, f32p, i32p, i64p]
    f64p = C.POINTER(C.c_double)
    L.pk_set_align_targets.argtypes = [vp, i32p, i32p, C.c_int32]
    L.pk_fetch_align_scores.argtypes = [vp, f64p, f64p]
    L.pk_kernel_ctc_align.argtypes = [C.c_int, C.c_int, i32p, C.c_int, C.c_int, f32p, i32p, i32p, C.c_int, i32p, i32p, i32p, f32p,
                                      f64p, f64p, i32p, i64p]
    L.pk_kernel_mel.argtypes = [C.c_int, C.c_int, i64p, f32p, C.c_int, C.c_int, f32p, f32p, i64p]
    L.pk_kernel_mel_stream.argtypes = [C.c_int, C.c_int, i64p, f32p, i32p, i32p, C.c_int, C.c_int, f32p, i64p]
    L.pk_kernel_subsample_conv1.argtypes = [C.c_int] * 3 + [i32p, C.c_int, f32p, C.c_int, C.c_int] + [f32p] * 7 + [i64p]
    L.pk_kernel_subsample_dw.argtypes = [C.c_int] * 3 + [i32p, C.c_int, C.c_int] + [f32p] * 6 + [i64p]
    _lib = L
    return L


# ------------------------------------------------------------------ configs (config.hpp)
class Math(enum.IntEnum):
    BF16X3 = 0
    BF16X1 = 1
    FP32 = 2


@dataclass
class ModelConfig:
    """EncoderConfig + PredictionConfig + JointConfig (reference config.hpp:9-75)."""
    mel_bins: int = 80
    sub_channels: int = 256
    d_model: int = 512
    n_layers: int = 17
    n_heads: int = 8
    ff: int = 2048
    conv_k: int = 9
    vocab: int = 1025
    pred_hidden: int = 640
    lstm_layers: int = 1
    joint_hidden: int = 640
    durations: tuple = (0, 1, 2, 3, 4)    # () = RNN-T joint (ParakeetRNNT: out_proj_, no duration head)
    has_ctc: bool = True
    joint_prefix: str = "tdt_joint_."
    max_symbols: int = 10                 # max_symbols_per_step (RNN-T: forced advance after this many)
    name: str = "tdt-ctc-110m"
    # streaming encoder only (StreamingEncoderConfig, streaming_encoder.hpp:18-24)
    att_context_left: int = 70
    att_context_right: int = 0
    # engine capacity
    max_batch: int = 64
    max_samples: int = 160000
    math: int = int(Math.BF16X3)
    # offline limited-context attention (left, right) for long utterances, NeMo's rel_pos_local_attn: frame i attends to
    # frame j only when -right <= i - j <= left.  (0, 0) = full attention.  With a band, max_batch * max_samples may reach
    # 3 h of audio (DESIGN.md section 16).  Separate from att_context_left / _right, which only pk_stream_open reads.
    local_attention: tuple = (0, 0)

    def to_c(self) -> _PkConfig:
        c = _PkConfig()
        c.mel_bins, c.sub_channels, c.d_model, c.n_layers = self.mel_bins, self.sub_channels, self.d_model, self.n_layers
        c.n_heads, c.ff, c.conv_kernel, c.vocab = self.n_heads, self.ff, self.conv_k, self.vocab
        c.pred_hidden, c.lstm_layers, c.joint_hidden = self.pred_hidden, self.lstm_layers, self.joint_hidden
        c.n_durations = len(self.durations)
        for i, d in enumerate(self.durations):
            c.durations[i] = d
        c.has_ctc = int(self.has_ctc)
        c.joint_prefix_tdt = int(self.joint_prefix == "tdt_joint_.")
        c.max_symbols = self.max_symbols
        c.max_batch, c.max_samples, c.math = self.max_batch, self.max_samples, int(self.math)
        c.local_att_left, c.local_att_right = (int(v) for v in self.local_attention)
        return c

    @property
    def is_rnnt(self) -> bool:
        return len(self.durations) == 0


def make_110m_config(**kw) -> ModelConfig:           # config.hpp:77-95
    return ModelConfig(**kw)


def make_tdt_600m_config(**kw) -> ModelConfig:       # config.hpp:98-116
    base = dict(mel_bins=128, d_model=1024, n_layers=24, ff=4096, vocab=8193, lstm_layers=2, has_ctc=False,
                joint_prefix="joint_.", name="tdt-600m", max_batch=16, max_samples=480000)
    base.update(kw)
    return ModelConfig(**base)


def make_rnnt_600m_config(**kw) -> ModelConfig:      # config.hpp:118-135 (ParakeetRNNT registers "joint_", rnnt.cpp:48-52)
    base = dict(d_model=1024, n_layers=24, ff=4096, vocab=1025, lstm_layers=2, durations=(), has_ctc=False,
                joint_prefix="joint_.", name="rnnt-600m", max_batch=16, max_samples=480000)
    base.update(kw)
    return ModelConfig(**base)


def make_eou_120m_config(**kw) -> ModelConfig:       # eou.hpp:32-55 (streaming; ParakeetEOU registers "joint_", eou.cpp:9-13)
    base = dict(has_ctc=False, joint_prefix="joint_.", name="eou-120m", att_context_left=70, att_context_right=1,
                max_batch=64, max_samples=102400)
    base.update(kw)
    return ModelConfig(**base)


def make_nemotron_600m_config(latency_frames: int = 0, **kw) -> ModelConfig:   # nemotron.hpp:33-54
    """The multilingual streaming model (ParakeetNemotron registers "encoder_" / "prediction_" / "joint_", the eou layout).
    latency_frames is att_context_right; like the reference's CPU path, it does not change the output (DESIGN.md)."""
    base = dict(d_model=1024, n_layers=24, ff=4096, vocab=8193, lstm_layers=2, has_ctc=False, joint_prefix="joint_.",
                name="nemotron-600m", att_context_left=70, att_context_right=latency_frames, max_batch=64, max_samples=102400)
    base.update(kw)
    return ModelConfig(**base)


def make_tiny_nemotron_config(**kw) -> ModelConfig:
    """Small test-only streaming shape with the Nemotron preset's head_dim 128 and two LSTM layers
    (mirrors tests/nemotron_oracle.make_tiny_nemotron_config; not a reference preset)."""
    base = dict(sub_channels=64, d_model=256, n_layers=2, n_heads=2, ff=512, vocab=33, pred_hidden=64, lstm_layers=2,
                joint_hidden=64, has_ctc=False, joint_prefix="joint_.", name="tiny-nemotron", att_context_left=12,
                att_context_right=0, max_batch=8, max_samples=102400)
    base.update(kw)
    return ModelConfig(**base)


def make_tiny_stream_config(**kw) -> ModelConfig:
    """Small test-only streaming shape (mirrors oracle.make_tiny_stream_config; not a reference preset)."""
    base = dict(sub_channels=64, d_model=128, n_layers=2, n_heads=2, ff=256, vocab=33, pred_hidden=64, joint_hidden=64,
                has_ctc=False, joint_prefix="joint_.", name="tiny-stream", att_context_left=12, att_context_right=1,
                max_batch=8, max_samples=102400)
    base.update(kw)
    return ModelConfig(**base)


def make_tiny_config(**kw) -> ModelConfig:
    """Small test-only shape (not a reference preset)."""
    base = dict(sub_channels=64, d_model=128, n_layers=2, n_heads=2, ff=256, vocab=33, pred_hidden=64,
                joint_hidden=64, name="tiny", max_batch=8, max_samples=64000)
    base.update(kw)
    return ModelConfig(**base)


def make_tiny_rnnt_config(**kw) -> ModelConfig:
    """Small test-only RNN-T shape (not a reference preset)."""
    base = dict(sub_channels=64, d_model=128, n_layers=2, n_heads=2, ff=256, vocab=33, pred_hidden=64,
                joint_hidden=64, durations=(), has_ctc=False, joint_prefix="joint_.", name="tiny-rnnt",
                max_batch=8, max_samples=64000)
    base.update(kw)
    return ModelConfig(**base)


@dataclass
class SortformerConfig:
    """SortformerConfig (reference sortformer.hpp:28-41): the NEST encoder (an offline FastConformer under "nest_encoder_."
    with xscaling and un-normalised features) plus the post-norm transformer and the speaker head.  `encoder` also carries
    the engine capacity and math."""
    encoder: ModelConfig
    t_hidden: int = 192
    t_layers: int = 18
    t_heads: int = 8
    t_ff: int = 768
    max_speakers: int = 4
    activity_threshold: float = 0.5
    name: str = "sortformer-117m"

    @property
    def mel_bins(self) -> int:
        return self.encoder.mel_bins

    @property
    def d_model(self) -> int:
        return self.encoder.d_model

    @property
    def n_layers(self) -> int:
        return self.encoder.n_layers

    @property
    def max_samples(self) -> int:
        return self.encoder.max_samples

    def to_c(self) -> _PkSortformerConfig:
        c = _PkSortformerConfig()
        c.enc = self.encoder.to_c()
        c.t_hidden, c.t_layers, c.t_heads, c.t_ff, c.max_speakers = (self.t_hidden, self.t_layers, self.t_heads, self.t_ff,
                                                                      self.max_speakers)
        return c


def make_sortformer_117m_config(**kw) -> SortformerConfig:   # sortformer.hpp:43-72
    """kw: capacity and math of the engine (max_batch, max_samples, math)."""
    enc = dict(mel_bins=128, sub_channels=256, d_model=512, n_layers=17, n_heads=8, ff=2048, vocab=0, pred_hidden=0, lstm_layers=0,
               joint_hidden=0, durations=(), has_ctc=False, joint_prefix="", max_symbols=0, name="nest-encoder", max_batch=16, max_samples=1440000)
    enc.update(kw)
    return SortformerConfig(encoder=ModelConfig(**enc))


def make_tiny_sortformer_config(**kw) -> SortformerConfig:
    """Small test-only Sortformer (not a reference preset): a 2-layer d 128 NEST encoder and a 2-layer post-norm transformer
    that keeps the preset's head_dim 24 (d 192, 8 heads), ff 384, 4 speakers."""
    enc = dict(mel_bins=128, sub_channels=64, d_model=128, n_layers=2, n_heads=2, ff=256, vocab=0, pred_hidden=0, lstm_layers=0,
               joint_hidden=0, durations=(), has_ctc=False, joint_prefix="", max_symbols=0, name="tiny-nest", max_batch=16, max_samples=64000)
    enc.update(kw)
    return SortformerConfig(encoder=ModelConfig(**enc), t_layers=2, t_ff=384, name="tiny-sortformer")


@dataclass
class DiarizationSegment:             # sortformer.hpp:20-24
    speaker_id: int
    start: float                      # seconds
    end: float


def diar_segments(probs: np.ndarray, threshold: float = 0.5) -> List[DiarizationSegment]:
    """Sortformer::probs_to_segments (sortformer.cpp:70-113) of one utterance's probs [T][S] (pk_diar_segments)."""
    L = load_library()
    p = np.ascontiguousarray(probs, np.float32)
    T, S = p.shape
    n = L.pk_diar_segments(_f32p(p), T, S, float(threshold), None, None, None, 0)
    if n < 0:
        raise RuntimeError("pk_diar_segments: invalid arguments")
    spk, st, en = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.float32)
    L.pk_diar_segments(_f32p(p), T, S, float(threshold), _i32p(spk), _f32p(st), _f32p(en), n)
    return [DiarizationSegment(int(spk[i]), float(st[i]), float(en[i])) for i in range(n)]


class AOSCCache:
    """AOSCCache (reference sortformer.cpp:9-38): arrival-order speaker tracking.  A speaker arrives the first time its
    probability is > 0.5 (fixed, not activity_threshold); within a frame speakers arrive in index order; a speaker is never
    forgotten until reset()."""

    def __init__(self, max_speakers: int = 4):
        self.max_speakers = max_speakers
        self.reset()

    def update(self, probs: np.ndarray):
        p = np.asarray(probs, np.float32)
        for t in range(p.shape[0]):
            for s in range(min(p.shape[1], self.max_speakers)):
                if p[t, s] > np.float32(0.5) and not self._active[s]:
                    self._active[s] = True
                    self._order.append(s)

    def speaker_order(self) -> List[int]:
        return list(self._order)

    def reset(self):
        self._active = [False] * self.max_speakers
        self._order = []


# ------------------------------------------------------------------ result types (timestamp.hpp, transcribe.hpp)
class Decoder(enum.IntEnum):          # transcribe.hpp:34
    CTC = 0
    TDT = 1
    RNNT = 2
    CTC_BEAM = 3                      # CTC prefix beam search (Engine.set_ctc_beam; DESIGN.md section 14)
    CTC_ALIGN = 4                     # CTC forced alignment of known tokens (Engine.set_align_targets; DESIGN.md section 15)


@dataclass
class TimestampedToken:               # timestamp.hpp:11-18
    token_id: int
    start_frame: int
    end_frame: int
    confidence: float = 1.0


@dataclass
class WordTimestamp:                  # timestamp.hpp:20-27
    word: str
    start: float
    end: float
    confidence: float = 1.0


@dataclass
class TranscribeResult:               # transcribe.hpp:23-30
    text: str = ""
    token_ids: List[int] = field(default_factory=list)
    timestamped_tokens: List[TimestampedToken] = field(default_factory=list)
    word_timestamps: List[WordTimestamp] = field(default_factory=list)


@dataclass
class AlignResult:
    """Transcriber.align: the tokens of the text (what was aligned, detokenised), their frames, the words, whether the
    audio could be aligned at all, the alignment (best path) score and the CTC log-likelihood log p(tokens | audio)."""
    text: str = ""
    token_ids: List[int] = field(default_factory=list)
    timestamped_tokens: List[TimestampedToken] = field(default_factory=list)
    word_timestamps: List[WordTimestamp] = field(default_factory=list)
    aligned: bool = False
    log_prob: float = float("-inf")
    ctc_log_likelihood: float = float("-inf")


@dataclass
class TranscribeOptions:              # transcribe.hpp:38-43
    decoder: Decoder = Decoder.TDT
    timestamps: bool = False
    boost_phrases: List[str] = field(default_factory=list)
    boost_score: float = 5.0


def safetensors_probe(path: str, name: Optional[str] = None, cap: int = 0):
    """Host-only check of the checkpoint reader: -> (status, message, values | None)."""
    L = load_library()
    out = np.zeros(max(cap, 1), np.float32)
    n = C.c_int64(0)
    st = L.pk_safetensors_probe(path.encode(), name.encode() if name else None, _f32p(out), cap, C.byref(n))
    msg = L.pk_last_error(None).decode() if st != 0 else ""
    return st, msg, (out[:min(cap, n.value)].copy() if (st == 0 and name) else None)


def selftest_gemm(M, N, K, epi_kind, math=0, seed=1, device=0):
    """-> (max_abs_err, max_abs_ref) of the wgmma GEMM vs the fp32 CUDA-core GEMM."""
    L = load_library()
    e, r = C.c_float(), C.c_float()
    st = L.pk_selftest_gemm(device, M, N, K, epi_kind, math, seed, C.byref(e), C.byref(r))
    if st != 0:
        raise RuntimeError(f"pk_selftest_gemm failed ({st})")
    return e.value, r.value


def _f32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _i32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _i64p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def _pack(arrs: Sequence[np.ndarray]):
    arrs = [np.ascontiguousarray(a, np.float32).reshape(-1) for a in arrs]
    off = np.zeros(len(arrs) + 1, np.int64)
    off[1:] = np.cumsum([len(a) for a in arrs])
    return (np.concatenate(arrs) if arrs else np.zeros(0, np.float32)), off


def read_wav(path: str) -> np.ndarray:
    """16 kHz mono PCM16 / float32 WAV -> fp32 in [-1, 1] (the subset of read_audio,
    src/audio_io.cpp:453-483, the configs need; int16 is divided by 32768 like dr_wav)."""
    with open(path, "rb") as f:
        data = f.read()
    if data[:4] != b"RIFF" or data[8:12] != b"WAVE":
        raise RuntimeError("Unsupported audio format (only RIFF/WAVE here): " + path)
    pos, fmt, pcm = 12, None, None
    while pos + 8 <= len(data):
        cid, size = data[pos:pos + 4], struct.unpack("<I", data[pos + 4:pos + 8])[0]
        body = data[pos + 8:pos + 8 + size]
        if cid == b"fmt ":
            fmt = struct.unpack("<HHIIHH", body[:16])
        elif cid == b"data":
            pcm = body
        pos += 8 + size + (size & 1)
    if fmt is None or pcm is None:
        raise RuntimeError("malformed WAV: " + path)
    tag, ch, sr, _, _, bits = fmt
    if sr != 16000:
        raise RuntimeError(f"Sample rate mismatch: audio={sr} expected=16000")
    if tag == 1 and bits == 16:
        x = np.frombuffer(pcm, "<i2").astype(np.float32) / np.float32(32768.0)
    elif tag == 3 and bits == 32:
        x = np.frombuffer(pcm, "<f4").astype(np.float32)
    else:
        raise RuntimeError("unsupported WAV encoding")
    if ch > 1:
        x = x.reshape(-1, ch).mean(axis=1).astype(np.float32)
    return x


class Engine:
    """Thin object wrapper over the C-ABI (one engine per device)."""

    def __init__(self, cfg: ModelConfig, weights_path: str, device: int = 0):
        self.L = load_library()
        self.cfg = cfg
        self.h = C.c_void_p()
        cc = cfg.to_c()
        create = self.L.pk_sortformer_create if isinstance(cfg, SortformerConfig) else self.L.pk_engine_create
        st = create(C.byref(cc), weights_path.encode(), device, C.byref(self.h))
        if st != 0:
            raise RuntimeError(f"{create.__name__} failed ({st}): " + self.L.pk_last_error(None).decode())
        self.Tmax = self.L.pk_encoder_frames(self.L.pk_mel_frames(cfg.max_samples))
        self.cap = self.token_buffer()[2] - 1       # the engine's token row capacity (2 T'max + 8; RNN-T: max_symbols T'max + 8)

    def close(self):
        if self.h:
            self.L.pk_engine_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st, what):
        if st != 0:
            raise RuntimeError(f"{what} failed ({st}): " + self.L.pk_last_error(self.h).decode())

    # -- stage-level entry points (parity taps)
    def mel(self, pcms: Sequence[np.ndarray]) -> List[np.ndarray]:
        buf, off = _pack(pcms)
        nfr = np.zeros(len(pcms), np.int32)
        total = sum(1 + len(p) // 160 for p in pcms)
        out = np.zeros((total, self.cfg.mel_bins), np.float32)
        self._check(self.L.pk_mel(self.h, _f32p(buf), _i64p(off), len(pcms), _f32p(out), _i32p(nfr)), "pk_mel")
        res, o = [], 0
        for n in nfr:
            res.append(out[o:o + n].copy())
            o += n
        return res

    def encode(self, feats: Sequence[np.ndarray], taps: bool = False):
        nfr = np.array([f.shape[0] for f in feats], np.int32)
        buf = np.ascontiguousarray(np.concatenate([np.asarray(f, np.float32) for f in feats], axis=0))
        lens = [self.L.pk_encoder_frames(int(n)) for n in nfr]
        Mx, d = sum(lens), self.cfg.d_model
        out = np.zeros((Mx, d), np.float32)
        olen = np.zeros(len(feats), np.int32)
        sub = np.zeros((Mx, d), np.float32) if taps else None
        lay = np.zeros((self.cfg.n_layers, Mx, d), np.float32) if taps else None
        self._check(self.L.pk_encode(self.h, _f32p(buf), _i32p(nfr), len(feats), _f32p(out), _i32p(olen),
                                     _f32p(sub) if taps else None, _f32p(lay) if taps else None), "pk_encode")
        offs = np.concatenate([[0], np.cumsum(olen)])
        encs = [out[offs[i]:offs[i + 1]].copy() for i in range(len(feats))]
        if taps:
            return encs, [sub[offs[i]:offs[i + 1]].copy() for i in range(len(feats))], \
                [lay[:, offs[i]:offs[i + 1]].copy() for i in range(len(feats))]
        return encs

    def _tokens(self, n):
        cap = self.cap
        arrs = dict(ids=np.zeros((n, cap), np.int32), start=np.zeros((n, cap), np.int32),
                    end=np.zeros((n, cap), np.int32), conf=np.zeros((n, cap), np.float32), len=np.zeros(n, np.int32))
        t = _PkTokens(cap, _i32p(arrs["ids"]), _i32p(arrs["start"]), _i32p(arrs["end"]), _f32p(arrs["conf"]),
                      _i32p(arrs["len"]))
        return t, arrs

    @staticmethod
    def _unpack(arrs, n):
        out = []
        for b in range(n):
            k = int(arrs["len"][b])
            out.append([TimestampedToken(int(arrs["ids"][b, i]), int(arrs["start"][b, i]), int(arrs["end"][b, i]),
                                         float(arrs["conf"][b, i])) for i in range(k)])
        return out

    def decode(self, encs: Sequence[np.ndarray], decoder: Decoder) -> List[List[TimestampedToken]]:
        lens = np.array([e.shape[0] for e in encs], np.int32)
        buf = np.ascontiguousarray(np.concatenate([np.asarray(e, np.float32) for e in encs], axis=0))
        t, arrs = self._tokens(len(encs))
        self._check(self.L.pk_decode(self.h, _f32p(buf), _i32p(lens), len(encs), int(decoder), C.byref(t)), "pk_decode")
        return self._unpack(arrs, len(encs))

    def ctc_logprobs(self, enc: np.ndarray) -> np.ndarray:
        enc = np.ascontiguousarray(enc, np.float32)
        out = np.zeros((enc.shape[0], self.cfg.vocab), np.float32)
        self._check(self.L.pk_ctc_logprobs(self.h, _f32p(enc), enc.shape[0], _f32p(out)), "pk_ctc_logprobs")
        return out

    # -- the whole path
    def transcribe_batch(self, pcms: Sequence[np.ndarray], decoder: Decoder) -> List[List[TimestampedToken]]:
        buf, off = _pack(pcms)
        t, arrs = self._tokens(len(pcms))
        self._check(self.L.pk_transcribe_batch(self.h, _f32p(buf), _i64p(off), len(pcms), int(decoder), C.byref(t)),
                    "pk_transcribe_batch")
        return self._unpack(arrs, len(pcms))

    def transcribe_packed(self, buf: np.ndarray, off: np.ndarray, decoder: Decoder, out=None):
        """Same call on an already packed host buffer (fp32 samples back to back + int64 offsets;
        page-locked buffers are DMA'd directly).  Returns the raw token arrays
        (ids, start, end, conf, len) without building Python objects."""
        n = len(off) - 1
        if out is None:
            out = self._tokens(n)
        t, arrs = out
        self._check(self.L.pk_transcribe_batch(self.h, _f32p(buf), _i64p(off), n, int(decoder), C.byref(t)),
                    "pk_transcribe_batch")
        return arrs

    # -- device-resident variant (bench)
    def stage(self, buf: np.ndarray, off: np.ndarray):
        self._check(self.L.pk_stage_pcm(self.h, _f32p(buf), _i64p(off), len(off) - 1), "pk_stage_pcm")

    def prefetch(self, buf: np.ndarray, off: np.ndarray):
        """Start the H2D copy of the NEXT batch (page-locked packed buffer) under the current batch's kernels;
        the following stage() / transcribe_packed() with the same arguments adopts it."""
        self._check(self.L.pk_prefetch_pcm(self.h, _f32p(buf), _i64p(off), len(off) - 1), "pk_prefetch_pcm")

    def fetch_into(self, out):
        """pk_fetch_tokens into preallocated arrays (see _tokens)."""
        t, arrs = out
        self._check(self.L.pk_fetch_tokens(self.h, C.byref(t)), "pk_fetch_tokens")
        return arrs

    def run_staged(self, decoder: Decoder):
        self._check(self.L.pk_run_staged(self.h, int(decoder)), "pk_run_staged")

    def fetch(self, n) -> List[List[TimestampedToken]]:
        t, arrs = self._tokens(n)
        self._check(self.L.pk_fetch_tokens(self.h, C.byref(t)), "pk_fetch_tokens")
        return self._unpack(arrs, n)

    def sync(self):
        self._check(self.L.pk_sync(self.h), "pk_sync")

    def flush_l2(self):
        self._check(self.L.pk_flush_l2(self.h), "pk_flush_l2")

    def profile_begin(self):
        self._check(self.L.pk_profile_begin(self.h), "pk_profile_begin")

    def profile_end(self):
        """-> {class: (ms, launches, gemm_flops)} summed since profile_begin()."""
        names = self.L.pk_profile_names().decode().split(",")
        n = len(names)
        ms = (C.c_double * n)(); cnt = (C.c_int64 * n)(); fl = (C.c_double * n)()
        self._check(self.L.pk_profile_end(self.h, ms, cnt, fl, n), "pk_profile_end")
        return {names[i]: (ms[i], int(cnt[i]), fl[i]) for i in range(n)}

    def tdt_phases(self):
        a = np.zeros(8, np.int64)
        self._check(self.L.pk_debug_tdt_phases(self.h, _i64p(a)), "pk_debug_tdt_phases")
        return a

    def tdt_passes(self):
        a = np.zeros(8, np.int64)
        self._check(self.L.pk_debug_tdt_passes(self.h, _i64p(a)), "pk_debug_tdt_passes")
        return a

    def launch_count(self) -> int:
        return int(self.L.pk_launch_count(self.h))

    def stream(self) -> int:
        return int(self.L.pk_stream(self.h) or 0)

    # -- Sortformer diarization (an engine made from a SortformerConfig)
    def _probs(self, lens_out: np.ndarray, out: np.ndarray) -> List[np.ndarray]:
        offs = np.concatenate([[0], np.cumsum(lens_out)])
        return [out[offs[i]:offs[i + 1]].copy() for i in range(len(lens_out))]

    def sortformer_forward(self, feats: Sequence[np.ndarray]) -> List[np.ndarray]:
        """Sortformer::forward per utterance: features [frames][mel_bins] -> sigmoid activities [T'][max_speakers]."""
        nfr = np.array([f.shape[0] for f in feats], np.int32)
        buf = np.ascontiguousarray(np.concatenate([np.asarray(f, np.float32) for f in feats], axis=0))
        M = sum(self.L.pk_encoder_frames(int(n)) for n in nfr)
        out = np.zeros((M, self.cfg.max_speakers), np.float32)
        lens = np.zeros(len(feats), np.int32)
        self._check(self.L.pk_sortformer_forward(self.h, _f32p(buf), _i32p(nfr), len(feats), _f32p(out), _i32p(lens)),
                    "pk_sortformer_forward")
        return self._probs(lens, out)

    def diarize_probs(self, pcms: Sequence[np.ndarray]) -> List[np.ndarray]:
        """The whole path from 16 kHz PCM: activities [T'][max_speakers] per utterance."""
        buf, off = _pack(pcms)
        M = sum(self.L.pk_encoder_frames(self.L.pk_mel_frames(len(p))) for p in pcms)
        out = np.zeros((M, self.cfg.max_speakers), np.float32)
        lens = np.zeros(len(pcms), np.int32)
        self._check(self.L.pk_diarize_batch(self.h, _f32p(buf), _i64p(off), len(pcms), _f32p(out), _i32p(lens)), "pk_diarize_batch")
        return self._probs(lens, out)

    def diarize_batch(self, pcms: Sequence[np.ndarray]) -> List[List[DiarizationSegment]]:
        """Sortformer::diarize for a batch of PCM utterances."""
        return [diar_segments(p, self.cfg.activity_threshold) for p in self.diarize_probs(pcms)]

    def run_diarize_staged(self):
        self._check(self.L.pk_run_diarize_staged(self.h), "pk_run_diarize_staged")

    def fetch_probs(self, out: np.ndarray, lens: np.ndarray):
        self._check(self.L.pk_fetch_probs(self.h, _f32p(out), _i32p(lens)), "pk_fetch_probs")

    # -- speaker-attributed transcription: this ASR engine and a Sortformer engine over one staged batch
    def transcribe_diarize_batch(self, diar_engine: "Engine", pcms: Sequence[np.ndarray], decoder: Decoder):
        """pk_transcribe_diarize_batch -> (tokens per utterance, activities [T'][max_speakers] per utterance)."""
        buf, off = _pack(pcms)
        t, arrs = self._tokens(len(pcms))
        M = sum(self.L.pk_encoder_frames(self.L.pk_mel_frames(len(p))) for p in pcms)
        probs = np.zeros((max(M, 1), diar_engine.cfg.max_speakers), np.float32)
        lens = np.zeros(max(len(pcms), 1), np.int32)
        self._check(self.L.pk_transcribe_diarize_batch(self.h, diar_engine.h, _f32p(buf), _i64p(off), len(pcms), int(decoder),
                                                        C.byref(t), _f32p(probs), _i32p(lens)), "pk_transcribe_diarize_batch")
        return self._unpack(arrs, len(pcms)), self._probs(lens[:len(pcms)], probs)

    def run_transcribe_diarize_staged(self, diar_engine: "Engine", decoder: Decoder):
        """After stage() on this engine: both models on the staged batch (then fetch / fetch_probs on each engine)."""
        self._check(self.L.pk_run_transcribe_diarize_staged(self.h, diar_engine.h, int(decoder)), "pk_run_transcribe_diarize_staged")

    # -- streaming diarization (a Sortformer engine): Sortformer::diarize_chunk for n_streams streams in lock step
    def diar_stream_open(self, n_streams: int, max_chunk_samples: int = 16000, att_context_left: int = 70):
        self._check(self.L.pk_diar_stream_open(self.h, n_streams, max_chunk_samples, att_context_left), "pk_diar_stream_open")
        self.n_diar_streams = n_streams
        self.diar_max_chunk = max_chunk_samples

    def diar_stream_reset(self, stream: int = -1):
        self._check(self.L.pk_diar_stream_reset(self.h, stream), "pk_diar_stream_reset")

    def diar_stream_step(self, chunks: Sequence[np.ndarray], feats: bool = False, taps: bool = False):
        """chunks[s] = stream s's input this step: 16 kHz PCM, or with feats=True its log-mel features [frames][mel_bins]
        (an empty chunk = no input).  Returns (probs, frame_base): probs[s] the chunk-local activities [C_s][max_speakers]
        of this step (C_s = 0 where the reference returns {}), frame_base[s] the absolute encoder frame of its first row;
        with taps also the NEST encoder rows [C_s][d_model] per stream."""
        S, SP = self.n_diar_streams, self.cfg.max_speakers
        assert len(chunks) == S
        nf_max = 1 + self.diar_max_chunk // 160
        rows = S * (((7 + nf_max) // 8) * 8 // 8 + 1)
        probs = np.zeros((rows, SP), np.float32)
        n_out, base = np.zeros(S, np.int32), np.zeros(S, np.int32)
        enc = np.zeros((rows, self.cfg.d_model), np.float32) if taps else None
        encp = _f32p(enc) if taps else None
        if feats:
            fs = [np.asarray(f, np.float32).reshape(-1, self.cfg.mel_bins) for f in chunks]
            nfr = np.array([f.shape[0] for f in fs], np.int32)
            buf = np.ascontiguousarray(np.concatenate(fs, axis=0)) if nfr.sum() else np.zeros((1, self.cfg.mel_bins), np.float32)
            st = self.L.pk_diar_stream_step_feats(self.h, _f32p(buf), _i32p(nfr), _f32p(probs), _i32p(n_out), _i32p(base), encp)
            self._check(st, "pk_diar_stream_step_feats")
        else:
            buf, off = _pack(chunks)
            self._check(self.L.pk_diar_stream_step(self.h, _f32p(buf), _i64p(off), _f32p(probs), _i32p(n_out), _i32p(base), encp),
                        "pk_diar_stream_step")
        o = np.concatenate([[0], np.cumsum(n_out)])
        out = [probs[o[i]:o[i + 1]].copy() for i in range(S)]
        if taps:
            return out, base, [enc[o[i]:o[i + 1]].copy() for i in range(S)]
        return out, base

    def diar_stream_speakers(self, stream: int) -> List[int]:
        """AOSCCache::speaker_order of one stream."""
        order = np.zeros(max(self.cfg.max_speakers, 1), np.int32)
        n = self.L.pk_diar_stream_speakers(self.h, stream, _i32p(order), len(order))
        if n < 0:
            raise RuntimeError("pk_diar_stream_speakers: invalid arguments")
        return [int(v) for v in order[:n]]

    # -- phrase boosting on the device (SURVEY.md section 8f row 3)
    def set_boost(self, phrases: Sequence[Sequence[int]], boost: float = 5.0):
        """phrases: token-id sequences; an empty list clears the boost."""
        ids = np.array([t for ph in phrases for t in ph], np.int32)
        off = np.zeros(len(phrases) + 1, np.int32)
        off[1:] = np.cumsum([len(ph) for ph in phrases])
        if len(ids) == 0:
            ids = np.zeros(1, np.int32)
        self._check(self.L.pk_set_boost(self.h, _i32p(ids), _i32p(off), len(phrases), float(boost)), "pk_set_boost")

    def set_boost_rows(self, lists: Sequence[Sequence[Sequence[int]]], boosts: Sequence[float]):
        """lists[i] = the phrases (token-id sequences) of utterance i of the following batches, boosts[i] its score; an
        empty list leaves that utterance unboosted; no lists at all clears.  Replaces, and is replaced by, set_boost."""
        assert len(lists) == len(boosts)
        ids, off, row = pack_phrase_lists(lists)
        self._check(self.L.pk_set_boost_rows(self.h, _i32p(ids), _i32p(off), _i32p(row), _f32p(np.asarray(list(boosts) or [0], np.float32)),
                                             len(lists)), "pk_set_boost_rows")

    def stream_set_boost(self, stream: int, phrases: Sequence[Sequence[int]], boost: float = 5.0):
        """The phrase list of one open stream from its next step on (an empty list: none); its trie state restarts."""
        ids, off, _ = pack_phrase_lists([phrases])
        self._check(self.L.pk_stream_set_boost(self.h, stream, _i32p(ids), _i32p(off), len(phrases), float(boost)), "pk_stream_set_boost")

    def set_ctc_beam(self, width: int, lm: Optional["LanguageModel"] = None, vocab=None, alpha: float = 0.5, beta: float = 1.0):
        """Beam width and optional word n-gram LM for Decoder.CTC_BEAM (pk_set_ctc_beam).  vocab: a Tokenizer or a vocab
        path, needed with an LM (word boundaries come from its pieces)."""
        tok = Tokenizer(vocab) if isinstance(vocab, str) else vocab
        self._check(self.L.pk_set_ctc_beam(self.h, int(width), lm.h if lm is not None else None, tok.h if tok is not None else None,
                                           float(alpha), float(beta)), "pk_set_ctc_beam")

    # -- non-16 kHz input: converted on the device (SURVEY.md section 8f row 4)
    def set_align_targets(self, token_lists: Sequence[Sequence[int]]):
        """The token ids to align in each row of the next Decoder.CTC_ALIGN run (pk_set_align_targets); [] clears them."""
        flat = np.array([t for ids in token_lists for t in ids] or [0], np.int32)
        off = np.zeros(len(token_lists) + 1, np.int32)
        off[1:] = np.cumsum([len(ids) for ids in token_lists])
        self._check(self.L.pk_set_align_targets(self.h, _i32p(flat), _i32p(off), len(token_lists)), "pk_set_align_targets")

    def align_scores(self, n: int):
        """(alignment score, log p(tokens | audio)) of each of the n rows of the last alignment run; -inf: not alignable."""
        sc, ll = np.zeros(max(n, 1), np.float64), np.zeros(max(n, 1), np.float64)
        self._check(self.L.pk_fetch_align_scores(self.h, sc.ctypes.data_as(C.POINTER(C.c_double)),
                                                 ll.ctypes.data_as(C.POINTER(C.c_double))), "pk_fetch_align_scores")
        return [(float(sc[i]), float(ll[i])) for i in range(n)]

    def stage_rate(self, pcms: Sequence[np.ndarray], src_rate: int):
        buf, off = _pack(pcms)
        self._check(self.L.pk_stage_pcm_rate(self.h, _f32p(buf), _i64p(off), len(pcms), src_rate), "pk_stage_pcm_rate")

    def transcribe_batch_rate(self, pcms: Sequence[np.ndarray], src_rate: int, decoder: Decoder) -> List[List[TimestampedToken]]:
        self.stage_rate(pcms, src_rate)
        self.run_staged(decoder)
        return self.fetch(len(pcms))

    def resample_batch(self, pcms: Sequence[np.ndarray], src_rate: int, dst_rate: int) -> List[np.ndarray]:
        buf, off = _pack(pcms)
        lens = [int(self.L.pk_resample_len(len(p), src_rate, dst_rate)) for p in pcms]
        ooff = np.zeros(len(pcms) + 1, np.int64)
        ooff[1:] = np.cumsum(lens)
        out = np.zeros(int(ooff[-1]), np.float32)
        self._check(self.L.pk_resample_batch(self.h, _f32p(buf), _i64p(off), len(pcms), src_rate, dst_rate, _f32p(out), _i64p(ooff)),
                    "pk_resample_batch")
        return [out[ooff[i]:ooff[i + 1]].copy() for i in range(len(pcms))]

    # -- jobs: many micro-batches, one exchange (SURVEY.md section 8e)
    def job_begin(self, rows_local: int, world: int = 1):
        self._check(self.L.pk_job_begin(self.h, rows_local, world), "pk_job_begin")

    def job_append(self):
        self._check(self.L.pk_job_append(self.h), "pk_job_append")

    def job_stage(self, buf: np.ndarray, off: np.ndarray):
        self._check(self.L.pk_job_stage_pcm(self.h, _f32p(buf), _i64p(off), len(off) - 1), "pk_job_stage_pcm")

    def job_select(self, first: int, n: int):
        self._check(self.L.pk_job_select(self.h, first, n), "pk_job_select")

    def nccl_unique_id(self) -> bytes:
        buf = C.create_string_buffer(128)
        if self.L.pk_nccl_unique_id(buf) != 0:
            raise RuntimeError("pk_nccl_unique_id failed: " + self.L.pk_last_error(None).decode())
        return buf.raw

    def comm_init_rank(self, uid: bytes, rank: int, world: int):
        self._check(self.L.pk_comm_init_rank(self.h, uid, rank, world), "pk_comm_init_rank")

    def allgather_tokens(self, comm=None):
        self._check(self.L.pk_allgather_tokens(self.h, comm), "pk_allgather_tokens")

    def job_fetch(self, n_rows: int, gathered: bool = False) -> np.ndarray:
        """-> int32 [n_rows, 1 + cap] rows (len, ids...) of this rank's job (or of all ranks, rank-major)."""
        out = np.zeros((n_rows, 1 + self.cap), np.int32)
        w = C.c_int32()
        self._check(self.L.pk_job_fetch(self.h, int(gathered), _i32p(out), n_rows, C.byref(w)), "pk_job_fetch")
        assert w.value == 1 + self.cap
        return out

    # -- streaming (eou path): n_streams streams advanced in lock step, one chunk per stream and step
    def stream_open(self, n_streams: int, max_chunk_samples: int = 5120):
        self._check(self.L.pk_stream_open(self.h, n_streams, max_chunk_samples, self.cfg.att_context_left,
                                          self.cfg.att_context_right), "pk_stream_open")
        self.n_streams = n_streams

    def stream_reset(self, stream: int = -1):
        self._check(self.L.pk_stream_reset(self.h, stream), "pk_stream_reset")

    def stream_step(self, chunks: Sequence[np.ndarray], taps: bool = False, out=None, raw: bool = False):
        """chunks[s] = the samples stream s receives in this step (may be empty).  Returns the tokens each stream emitted
        in this step (absolute frames); with taps also the new log-mel frames and the encoder rows per stream."""
        S = self.n_streams
        assert len(chunks) == S
        buf, off = _pack(chunks)
        if out is None:
            out = self._tokens(S)
        t, arrs = out
        if not taps:
            self._check(self.L.pk_stream_step(self.h, _f32p(buf), _i64p(off), C.byref(t), None, None, None, None), "pk_stream_step")
            return arrs if raw else self._unpack(arrs, S)
        max_nf = 8 + max(len(c) for c in chunks) // 160 + 4
        mel = np.zeros((S * max_nf, self.cfg.mel_bins), np.float32)
        enc = np.zeros((S * (max_nf // 8 + 2), self.cfg.d_model), np.float32)
        n_mel, n_enc = np.zeros(S, np.int32), np.zeros(S, np.int32)
        self._check(self.L.pk_stream_step(self.h, _f32p(buf), _i64p(off), C.byref(t), _f32p(mel), _i32p(n_mel), _f32p(enc), _i32p(n_enc)),
                    "pk_stream_step")
        mo, eo = np.concatenate([[0], np.cumsum(n_mel)]), np.concatenate([[0], np.cumsum(n_enc)])
        return self._unpack(arrs, S), [mel[mo[i]:mo[i + 1]].copy() for i in range(S)], [enc[eo[i]:eo[i + 1]].copy() for i in range(S)]

    def truncated_count(self) -> int:
        return int(self.L.pk_truncated_count(self.h))

    def token_buffer(self):
        p, rows, ints = C.c_void_p(), C.c_int32(), C.c_int32()
        self._check(self.L.pk_token_buffer(self.h, C.byref(p), C.byref(rows), C.byref(ints)), "pk_token_buffer")
        return int(p.value), rows.value, ints.value


def pack_phrase_lists(lists):
    """Phrase lists (one per row, each a list of token-id sequences) -> (phrase_ids, phrase_off, row_off) int32 arrays in the
    layout of pk_set_boost_rows."""
    phrases = [ph for lst in lists for ph in lst]
    ids = np.array([t for ph in phrases for t in ph] or [0], np.int32)
    off = np.zeros(len(phrases) + 1, np.int32)
    off[1:] = np.cumsum([len(ph) for ph in phrases])
    row = np.zeros(len(lists) + 1, np.int32)
    row[1:] = np.cumsum([len(lst) for lst in lists])
    return ids, off, row


class LanguageModel:
    """A word n-gram LM read from an ARPA file (pk_lm_load), for Engine.set_ctc_beam."""

    def __init__(self, arpa_path: str):
        self.L = load_library()
        self.h = C.c_void_p()
        if self.L.pk_lm_load(arpa_path.encode(), C.byref(self.h)) != 0:
            raise RuntimeError("pk_lm_load: " + self.L.pk_last_error(None).decode())

    @property
    def order(self) -> int:
        return self.L.pk_lm_order(self.h)

    def count(self, order: int) -> int:
        return self.L.pk_lm_count(self.h, order)

    def sentence_log10(self, words: str) -> float:
        """log10 p(words </s> | <s>) by ARPA back-off."""
        return self.L.pk_lm_sentence_log10(self.h, words.encode("utf-8"))

    def close(self):
        if self.h:
            self.L.pk_lm_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Tokenizer:
    """Tokenizer::load / decode (src/vocab.cpp:10-64) via the C-ABI host helpers."""

    def __init__(self, vocab_path: Optional[str] = None):
        self.L = load_library()
        self.h = C.c_void_p()
        if vocab_path:
            self.load(vocab_path)

    def load(self, vocab_path: str):
        if self.L.pk_vocab_load(vocab_path.encode(), C.byref(self.h)) != 0:
            raise RuntimeError("Cannot open vocab file: " + vocab_path)      # vocab.cpp:13

    def loaded(self) -> bool:
        return bool(self.h) and self.L.pk_vocab_size(self.h) > 0

    def decode(self, ids: Sequence[int]) -> str:
        a = np.ascontiguousarray(ids, np.int32)
        buf = C.create_string_buffer(2 + (self.L.pk_vocab_max_piece_bytes(self.h) + 1) * max(len(a), 1))
        self.L.pk_detokenize(self.h, _i32p(a), len(a), buf, len(buf))
        return buf.value.decode("utf-8")

    def encode(self, text: str) -> List[int]:
        """Tokenizer::encode (src/vocab.cpp:76-117)."""
        raw = text.encode("utf-8")
        ids = np.zeros(2 * len(raw) + 8, np.int32)
        n = self.L.pk_tokenize(self.h, raw, _i32p(ids), len(ids))
        return ids[:n].tolist()

    def group_words(self, toks: Sequence[TimestampedToken]) -> List[WordTimestamp]:
        n = len(toks)
        ids = np.array([t.token_id for t in toks], np.int32)
        st = np.array([t.start_frame for t in toks], np.int32)
        en = np.array([t.end_frame for t in toks], np.int32)
        cf = np.array([t.confidence for t in toks], np.float32)
        buf = C.create_string_buffer(64 + 64 * max(n, 1))
        ws, we, wc = (np.zeros(max(n, 1), np.float32) for _ in range(3))
        k = self.L.pk_group_words(self.h, _i32p(ids), _i32p(st), _i32p(en), _f32p(cf), n, buf, len(buf), _f32p(ws),
                                  _f32p(we), _f32p(wc))
        words = buf.value.decode("utf-8").split("\n")[:k]
        return [WordTimestamp(words[i], float(ws[i]), float(we[i]), float(wc[i])) for i in range(k)]


def resample(samples: np.ndarray, src_rate: int, dst_rate: int = 16000) -> np.ndarray:
    """parakeet::resample (src/audio_io.cpp:238-251): Kaiser-windowed sinc, host code behind pk_resample."""
    L = load_library()
    x = np.ascontiguousarray(samples, np.float32)
    m = L.pk_resample_len(len(x), src_rate, dst_rate)
    if m < 0:
        raise ValueError("pk_resample: invalid arguments")
    out = np.zeros(max(m, 1), np.float32)
    L.pk_resample(_f32p(x if len(x) else np.zeros(1, np.float32)), len(x), src_rate, dst_rate, _f32p(out), m)
    return out[:m]


def ctc_greedy_decode_boosted(logprobs: np.ndarray, phrases: Sequence[Sequence[int]], boost_score: float = 5.0,
                              blank_id: Optional[int] = None) -> List[TimestampedToken]:
    """ctc_greedy_decode_with_timestamps_boosted (src/phrase_boost.cpp:122-176) on one utterance's log-probs
    (Engine.ctc_logprobs); phrases are token-id sequences (Tokenizer.encode).  Host code behind pk_ctc_decode_boosted."""
    L = load_library()
    lp = np.ascontiguousarray(logprobs, np.float32)
    T, V = lp.shape
    blank = V - 1 if blank_id is None else blank_id
    flat = np.array([t for ph in phrases for t in ph] or [0], np.int32)
    off = np.zeros(len(phrases) + 1, np.int32)
    off[1:] = np.cumsum([len(ph) for ph in phrases])
    ids, st, en = (np.zeros(max(T, 1), np.int32) for _ in range(3))
    cf = np.zeros(max(T, 1), np.float32)
    n = L.pk_ctc_decode_boosted(_f32p(lp), T, V, blank, _i32p(flat), _i32p(off), len(phrases), float(boost_score), _i32p(ids),
                                _i32p(st), _i32p(en), _f32p(cf), len(ids))
    if n < 0:
        raise ValueError("pk_ctc_decode_boosted: invalid arguments")
    return [TimestampedToken(int(ids[i]), int(st[i]), int(en[i]), float(cf[i])) for i in range(n)]


class Transcriber:
    """Python mirror of parakeet::Transcriber / TDTTranscriber (transcribe.hpp:55-299)."""

    def __init__(self, weights_path: str, vocab_path: str, config: Optional[ModelConfig] = None, device: int = 0):
        self.config = config or make_110m_config()
        self.engine = Engine(self.config, weights_path, device)
        self.tokenizer = Tokenizer(vocab_path) if vocab_path else Tokenizer()

    def to_gpu(self):
        """The reference moves the module tree to Metal here (transcribe.hpp:68-71); this
        engine only ever lives on the CUDA device, so this is a checked no-op."""
        return self

    def _result(self, toks, timestamps):
        r = TranscribeResult()
        r.token_ids = [t.token_id for t in toks]
        if timestamps:
            r.timestamped_tokens = list(toks)
        if self.tokenizer.loaded():
            r.text = self.tokenizer.decode(r.token_ids)
            if timestamps:
                r.word_timestamps = self.tokenizer.group_words(toks)
        return r

    def _decoder(self, decoder):
        """An RNN-T model always decodes with RNNT; a model without a CTC head always with TDT."""
        if self.config.is_rnnt:
            return Decoder.RNNT
        return decoder if self.config.has_ctc else Decoder.TDT

    def transcribe(self, audio, decoder=Decoder.TDT, timestamps: bool = False) -> TranscribeResult:
        if isinstance(decoder, TranscribeOptions):
            opts = decoder
        else:
            opts = TranscribeOptions(decoder=decoder, timestamps=timestamps)
        if opts.boost_phrases:
            raise NotImplementedError("phrase boosting is outside the H100 hot path (SURVEY.md section 8f.3)")
        samples = read_wav(audio) if isinstance(audio, str) else np.asarray(audio, np.float32)
        toks = self.engine.transcribe_batch([samples], self._decoder(opts.decoder))[0]
        return self._result(toks, opts.timestamps)

    def align(self, audio, text: str) -> AlignResult:
        """CTC forced alignment (DESIGN.md section 15): the frames of each token of `text` (tokenised by Tokenizer.encode,
        which skips bytes no piece covers) and its words in `audio` (a 16 kHz WAV path or samples)."""
        return self.align_batch([audio], [text])[0]

    def align_batch(self, audios, texts: Sequence[str]) -> List[AlignResult]:
        if not self.config.has_ctc:
            raise ValueError("alignment needs a CTC head; this model has none")
        if len(audios) != len(texts):
            raise ValueError("align_batch: one text per utterance")
        pcms = [read_wav(a) if isinstance(a, str) else np.asarray(a, np.float32) for a in audios]
        targets = [self.tokenizer.encode(t) for t in texts]
        out = []
        B = self.config.max_batch
        for i in range(0, len(pcms), B):
            self.engine.set_align_targets(targets[i:i + B])
            rows = self.engine.transcribe_batch(pcms[i:i + B], Decoder.CTC_ALIGN)
            for ids, toks, (sc, ll) in zip(targets[i:i + B], rows, self.engine.align_scores(len(rows))):
                r = AlignResult(text=self.tokenizer.decode(ids), token_ids=list(ids), timestamped_tokens=toks,
                                aligned=sc != float("-inf"), log_prob=sc, ctc_log_likelihood=ll)
                r.word_timestamps = self.tokenizer.group_words(toks)
                out.append(r)
        return out

    def transcribe_batch(self, audios, decoder=Decoder.TDT, timestamps: bool = False,
                         options: Optional[Sequence[TranscribeOptions]] = None) -> List[TranscribeResult]:
        """options: one TranscribeOptions per utterance (decoder and timestamps must agree across the batch); each
        utterance is decoded with its own boost_phrases / boost_score, as transcribe() would on it alone."""
        pcms = [read_wav(a) if isinstance(a, str) else np.asarray(a, np.float32) for a in audios]
        lists = None
        if options is not None:
            if len(options) != len(pcms):
                raise ValueError("transcribe_batch: one TranscribeOptions per utterance")
            if any(o.decoder != options[0].decoder or o.timestamps != options[0].timestamps for o in options):
                raise ValueError("transcribe_batch: decoder and timestamps must agree across the batch")
            if options:
                decoder, timestamps = options[0].decoder, options[0].timestamps
            if any(o.boost_phrases for o in options):
                if self.config.is_rnnt:
                    raise ValueError("phrase boosting covers CTC and TDT decodes; this is an RNN-T model")
                lists = [[self.tokenizer.encode(ph) for ph in o.boost_phrases] for o in options]
                lists = [[ph for ph in lst if ph] for lst in lists]           # (ContextTrie::build skips phrases without tokens)
        out = []
        B = self.config.max_batch
        for i in range(0, len(pcms), B):
            if lists is not None:
                self.engine.set_boost_rows(lists[i:i + B], [o.boost_score for o in options[i:i + B]])
            try:
                for toks in self.engine.transcribe_batch(pcms[i:i + B], self._decoder(decoder)):
                    out.append(self._result(toks, timestamps))
            finally:
                if lists is not None:
                    self.engine.set_boost_rows([], [])
        return out


@dataclass
class DiarizedWord:                   # diarize.hpp:19-25
    word: str
    start: float                      # seconds
    end: float
    speaker_id: int = -1              # -1: no overlapping segment
    confidence: float = 1.0


@dataclass
class DiarizedResult:                 # diarize.hpp:27-32
    text: str = ""
    words: List[DiarizedWord] = field(default_factory=list)
    segments: List[DiarizationSegment] = field(default_factory=list)
    word_timestamps: List[WordTimestamp] = field(default_factory=list)


def diarize_transcription(words: Sequence[WordTimestamp], segments: Sequence[DiarizationSegment]) -> List[DiarizedWord]:
    """diarize_transcription (reference diarize.cpp:10-48), pk_diarize_transcription: each word gets the speaker with the
    largest summed overlap over the segments in list order (ties as the reference's std::unordered_map), or -1."""
    L = load_library()
    ws = np.array([w.start for w in words] or [0], np.float32)
    we = np.array([w.end for w in words] or [0], np.float32)
    spk = np.array([s.speaker_id for s in segments] or [0], np.int32)
    ss = np.array([s.start for s in segments] or [0], np.float32)
    se = np.array([s.end for s in segments] or [0], np.float32)
    out = np.zeros(max(len(words), 1), np.int32)
    if L.pk_diarize_transcription(_f32p(ws), _f32p(we), len(words), _i32p(spk), _f32p(ss), _f32p(se), len(segments), _i32p(out)) != 0:
        raise RuntimeError("pk_diarize_transcription: invalid arguments")
    return [DiarizedWord(w.word, w.start, w.end, int(out[i]), w.confidence) for i, w in enumerate(words)]


def diarize_words(probs: np.ndarray, words: Sequence[WordTimestamp], threshold: float = 0.5):
    """pk_diarize_words on one utterance: -> (segments in the reference's order, [DiarizedWord])."""
    L = load_library()
    p = np.ascontiguousarray(probs, np.float32)
    T, S = p.shape
    ws = np.array([w.start for w in words] or [0], np.float32)
    we = np.array([w.end for w in words] or [0], np.float32)
    spk = np.zeros(max(len(words), 1), np.int32)
    cap = T * S // 2 + S
    ss, st, en = np.zeros(cap, np.int32), np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    n = L.pk_diarize_words(_f32p(p), T, S, float(threshold), _f32p(ws), _f32p(we), len(words), _i32p(spk), _i32p(ss), _f32p(st),
                           _f32p(en), cap)
    if n < 0:
        raise RuntimeError("pk_diarize_words: invalid arguments")
    segs = [DiarizationSegment(int(ss[i]), float(st[i]), float(en[i])) for i in range(n)]
    return segs, [DiarizedWord(w.word, w.start, w.end, int(spk[i]), w.confidence) for i, w in enumerate(words)]


class DiarizedTranscriber:
    """Python mirror of parakeet::DiarizedTranscriber (include/parakeet/diarize.hpp): a TDT-CTC ASR engine and a Sortformer
    engine with one capacity (max_batch utterances of max_samples), run over one staged batch (pk_transcribe_diarize_batch)."""

    def __init__(self, asr_weights: str, sortformer_weights: str, vocab_path: str, config: Optional[ModelConfig] = None,
                 sf_config: Optional[SortformerConfig] = None, device: int = 0, max_batch: int = 16, max_samples: int = 30 * 16000,
                 math: int = 0):
        cap = dict(max_batch=max_batch, max_samples=max_samples, math=math)
        self.config = replace(config or make_110m_config(), **cap)
        if self.config.is_rnnt:
            raise ValueError("DiarizedTranscriber: the ASR model must be a TDT-CTC or TDT model")
        sf = sf_config or make_sortformer_117m_config()
        self.sf_config = replace(sf, encoder=replace(sf.encoder, **cap))
        self.asr = Engine(self.config, asr_weights, device)
        self.diar = Engine(self.sf_config, sortformer_weights, device)
        self.tokenizer = Tokenizer(vocab_path)

    def to_gpu(self):
        """A no-op: both models only ever live on the CUDA device."""
        return self

    def close(self):
        self.asr.close()
        self.diar.close()

    def transcribe(self, audio, decoder=Decoder.TDT) -> DiarizedResult:
        return self.transcribe_batch([audio], decoder)[0]

    def transcribe_batch(self, audios, decoder=Decoder.TDT) -> List[DiarizedResult]:
        pcms = [read_wav(a) if isinstance(a, str) else np.asarray(a, np.float32) for a in audios]
        dec = decoder if self.config.has_ctc else Decoder.TDT
        out = []
        B = self.config.max_batch
        for i in range(0, len(pcms), B):
            toks, probs = self.asr.transcribe_diarize_batch(self.diar, pcms[i:i + B], dec)
            for tk, p in zip(toks, probs):
                wts = self.tokenizer.group_words(tk)
                segs, words = diarize_words(p, wts, self.sf_config.activity_threshold)
                out.append(DiarizedResult(self.tokenizer.decode([t.token_id for t in tk]), words, segs, wts))
        return out


TDTTranscriber = Transcriber   # transcribe.hpp:200-299 (same surface, TDT only)
RNNTTranscriber = Transcriber  # same surface; an RNN-T config (make_rnnt_600m_config) decodes with Decoder.RNNT
