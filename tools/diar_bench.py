"""Sortformer offline diarization throughput on one GPU (sortformer-117m, seeded synthetic weights and audio).

    python tools/diar_bench.py --batch 64 --seconds 10 --steps 20 --warmup 3 [--out FILE]

One step = one batch of PCM staged on the device (pk_stage_pcm), the whole model after the front end replayed as a CUDA graph
(pk_run_diarize_staged) and the activities fetched (pk_fetch_probs, which synchronises the engine stream).  Prints one JSON
line: ms per step (host clock around the steps; every step ends in that synchronise), x real time, per-kernel-class device times from a separate profiled pass, and the card
name, power limit and SM clock read in the same run.  Writes nothing into the repository tree unless --out says so.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    v = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")] if r.returncode == 0 and r.stdout.strip() else ["?"] * 4
    return {"name": v[0], "power_limit_w": v[1], "sm_clock_mhz": v[2], "sm_clock_max_mhz": v[3]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--math", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = ge.load_package()
    from parakeet_cpp_b200 import synth
    n = int(a.seconds * 16000)
    cfg = pkg.make_sortformer_117m_config(max_batch=a.batch, max_samples=n, math=a.math)
    W = synth.make_sortformer_weights(cfg, seed=0)
    pcms = [synth.make_audio(n, 1000 + i) for i in range(a.batch)]
    buf = np.concatenate(pcms).astype(np.float32)
    off = np.arange(a.batch + 1, dtype=np.int64) * n
    with tempfile.TemporaryDirectory() as td:
        wp = os.path.join(td, "sortformer.safetensors")
        synth.save_safetensors(wp, W)
        eng = pkg.Engine(cfg, wp, 0)
    T = eng.L.pk_encoder_frames(eng.L.pk_mel_frames(n))
    probs = np.zeros((a.batch * T, cfg.max_speakers), np.float32)
    lens = np.zeros(a.batch, np.int32)

    def step():
        eng.stage(buf, off)
        eng.run_diarize_staged()
        eng.fetch_probs(probs, lens)

    for _ in range(a.warmup):
        step()
    c0 = card()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        step()
    ms = (time.perf_counter() - t0) * 1e3 / a.steps
    eng.profile_begin()
    for _ in range(3):
        step()
    prof = {k: round(v[0] / 3, 4) for k, v in eng.profile_end().items() if v[1]}
    eng.close()
    res = {"model": "sortformer-117m", "batch": a.batch, "seconds": a.seconds, "math": a.math, "steps": a.steps,
           "ms_per_step": round(ms, 3), "x_real_time": round(a.batch * a.seconds * 1e3 / ms, 1),
           "device_ms_per_class": prof, "card": c0}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
