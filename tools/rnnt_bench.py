"""Throughput of the rnnt-600m model: 16 x 30 s synthetic clips per step, RNN-T greedy decode in lock step.

    python tools/rnnt_bench.py [--steps 20] [--warmup 3] [--tmp DIR]

Prints one JSON line: device-resident RTFx (the batch's PCM staged on the device once; every step runs mel ->
encoder -> RNN-T decode with an L2 flush in between) and end-to-end RTFx (pk_transcribe_batch: host PCM in, host
tokens out), ms per step, per-class device time and launches of one step, the encoder's algorithmic GFLOP per clip
(SURVEY.md section 8d formula), and the card name, power limit and SM clock sampled during the timed region.

The synthetic checkpoint (seed 0, blank bias 7: ~0.25 tokens per encoder frame, the rate of real speech) and clip 0
are those of tests/golden/golden_rnnt_600m_long_v1.npz, so the line also reports whether clip 0's tokens equal the
compiled reference's.  The checkpoint is written under --tmp; nothing is written into the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import __graft_entry__ as ge  # noqa: E402

BATCH, CLIP_SAMPLES = 16, 480000
BLANK_BIAS = 7.0                      # as tests/golden/make_golden_rnnt.py (M600_BLANK_BIAS)
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_rnnt_600m_long_v1.npz")


def conv_len(n):
    return (n + 2 - 3) // 2 + 1


def encoder_gflop(n_samples, mel=80, C=256, d=1024, ff=4096, layers=24):
    """SURVEY.md section 8d: F_sub + layers * F_layer, without the input-independent pos_proj."""
    n = 1 + n_samples // 160
    t1, t2 = conv_len(n), conv_len(conv_len(n))
    T = conv_len(t2)
    f1, f2 = conv_len(mel), conv_len(conv_len(mel))
    F = conv_len(f2)
    f_sub = 2 * C * 9 * (t1 * f1) + 2 * C * 9 * (t2 * f2) + 2 * C * C * (t2 * f2) + 2 * C * 9 * (T * F) + 2 * C * C * (T * F) + 2 * T * (C * F) * d
    f_layer = 8 * T * d * ff + 8 * T * d * d + 4 * T * T * d + 2 * T * (2 * T - 1) * d + (6 * T * d * d + 18 * T * d)
    return (f_sub + layers * f_layer) / 1e9, F


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception:
        return ""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tmp", default=os.environ.get("PK_BENCH_TMP", "/tmp/pk_bench"))
    args = ap.parse_args()
    args.steps, args.warmup = max(args.steps, 20), max(args.warmup, 3)
    os.makedirs(args.tmp, exist_ok=True)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("rnnt_bench.py: no CUDA device (the engine has no CPU fallback)")
    pkg = ge.load_package()
    from parakeet_cpp_b200 import synth
    cfg = pkg.make_rnnt_600m_config()
    wp = os.path.join(args.tmp, "pkrnnt600m_seed0_blank7.safetensors")
    if not os.path.exists(wp):
        synth.save_safetensors(wp + ".tmp", synth.make_weights(cfg, seed=0, blank_bias=BLANK_BIAS))
        os.replace(wp + ".tmp", wp)
    eng = pkg.Engine(cfg, wp, 0)
    dec = pkg.Decoder.RNNT
    gold = np.load(GOLDEN)
    n0, seed0 = (int(v) for v in gold["m600l.c0.n_samples"])
    assert n0 == CLIP_SAMPLES
    clips = [synth.make_audio(CLIP_SAMPLES, seed0)] + [synth.make_audio(CLIP_SAMPLES, 3000 + i) for i in range(1, BATCH)]
    buf = torch.empty(BATCH * CLIP_SAMPLES, dtype=torch.float32).pin_memory().numpy()
    for i, c in enumerate(clips):
        buf[i * CLIP_SAMPLES:(i + 1) * CLIP_SAMPLES] = c
    off = np.arange(BATCH + 1, dtype=np.int64) * CLIP_SAMPLES
    stream = torch.cuda.ExternalStream(eng.stream(), device=0)

    # device-resident: the batch's PCM is staged once; each step re-runs the whole path on it
    eng.job_stage(buf, off)
    eng.job_select(0, BATCH)

    def steps(k):
        for _ in range(k):
            eng.flush_l2()
            eng.run_staged(dec)

    steps(args.warmup)
    first = eng.fetch(BATCH)
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.3)
    eng.sync()
    l0 = eng.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    steps(args.steps)
    e1.record(stream)
    eng.sync()
    ms = e0.elapsed_time(e1)
    launches = (eng.launch_count() - l0) // args.steps
    last = eng.fetch(BATCH)
    assert [[t.token_id for t in u] for u in last] == [[t.token_id for t in u] for u in first], "rnnt_bench: steps differ"
    assert eng.truncated_count() == 0

    # end to end: pk_transcribe_batch from page-locked host PCM, tokens back to the host every step
    tok_out = eng._tokens(BATCH)
    eng.transcribe_packed(buf, off, dec, tok_out)
    w0 = time.perf_counter()
    for _ in range(args.steps):
        eng.transcribe_packed(buf, off, dec, tok_out)
    e2e_wall = time.perf_counter() - w0
    clocks = sampler.stop()

    eng.job_select(0, BATCH)
    eng.profile_begin()
    P = 3
    steps(P)
    prof = eng.profile_end()
    audio_s = args.steps * BATCH * CLIP_SAMPLES / 16000.0
    gflop, fprime = encoder_gflop(CLIP_SAMPLES)
    line = {"config": "rnnt-600m-16x30s", "workload": "rnnt-600m RNN-T greedy decode (max_symbols 10), 16 x 30 s synthetic clips per step, lock step",
            "rtfx_device": audio_s / (ms / 1e3), "rtfx_e2e": audio_s / e2e_wall, "ms_per_step": ms / args.steps,
            "e2e_ms_per_step": 1e3 * e2e_wall / args.steps, "steps": args.steps, "warmup": args.warmup, "n_clips": BATCH,
            "clip_s": CLIP_SAMPLES / 16000.0, "tokens_per_step": int(sum(len(u) for u in last)),
            "gpu_launches": int(launches),
            "per_class_ms": {k: v[0] / P for k, v in prof.items()}, "per_class_launches": {k: v[1] // P for k, v in prof.items()},
            "encoder_gflop_per_clip": gflop, "encoder_gflop_formula": f"SURVEY.md section 8d, F' = {fprime}, T' = 376, without pos_proj",
            "dtype": {0: "bf16x3", 1: "bf16", 2: "f32"}[int(cfg.math)],
            "gpu_name": gpu_name(), "power_limit_w": clocks["power_limit_w"], "sm_clock_mhz": clocks["sm_mhz"], "clocks": clocks,
            "clip0_tokens_match_reference": [(t.token_id, t.start_frame, t.end_frame) for t in first[0]] ==
                                            [tuple(int(v) for v in r) for r in gold["m600l.c0.tok"]]}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
