"""Speaker-attributed transcription throughput on one GPU: tdt-ctc-110m (TDT decode) and sortformer-117m over one batch,
seeded synthetic weights and audio.

    python tools/diarized_bench.py [--steps 20] [--warmup 3] [--configs 64x10,16x60] [--out FILE]

For each configuration (utterances x seconds) three runs are timed, each as ms per batch:
  joint     pk_transcribe_diarize_batch: the PCM copied once, both models on their own streams
  separate  pk_transcribe_batch on the ASR engine, then pk_diarize_batch on the Sortformer engine (the PCM copied twice)
  asr       pk_transcribe_batch alone
in two forms: `pinned` (every step stages the batch from a page-locked host buffer, runs, and fetches the results) and
`resident` (the batch staged once; every step runs from the device buffer and fetches).  Every step ends in the fetches,
which synchronise the engines; the window is timed with CUDA events on the engines' streams after the warm-up steps.
Prints one JSON line with the card name and power limit read in the same run.  Writes nothing into the repository tree
unless --out says so.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    v = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")] if r.returncode == 0 and r.stdout.strip() else ["?"] * 4
    return {"name": v[0], "power_limit_w": v[1], "sm_clock_mhz": v[2], "sm_clock_max_mhz": v[3]}


def timed(torch, streams, step, steps, warmup):
    """ms per step over `steps` steps after `warmup`, CUDA events on the engine streams (every stream joins the last one)."""
    for _ in range(warmup):
        step()
    ext = [torch.cuda.ExternalStream(s) for s in streams]
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(ext[0])
    for s in ext[1:]:
        s.wait_stream(ext[0])
    for _ in range(steps):
        step()
    for s in ext[1:]:
        ext[0].wait_stream(s)
    b.record(ext[0])
    b.synchronize()
    return a.elapsed_time(b) / steps


def run_config(pkg, torch, synth, O, td, B, seconds, steps, warmup):
    n = int(seconds * 16000)
    acfg = pkg.make_110m_config(max_batch=B, max_samples=n)
    scfg = pkg.make_sortformer_117m_config(max_batch=B, max_samples=n)
    wa, ws = os.path.join(td, "asr.safetensors"), os.path.join(td, "sf.safetensors")
    synth.save_safetensors(wa, synth.make_weights(O.make_110m_config(), seed=0))
    synth.save_safetensors(ws, synth.make_sortformer_weights(scfg, seed=0))
    asr, diar = pkg.Engine(acfg, wa, 0), pkg.Engine(scfg, ws, 0)
    pin = torch.empty(B * n, dtype=torch.float32, pin_memory=True).numpy()
    pin[:] = np.concatenate([synth.make_audio(n, 1000 + i) for i in range(B)])
    off = np.arange(B + 1, dtype=np.int64) * n
    T = asr.L.pk_encoder_frames(asr.L.pk_mel_frames(n))
    probs, lens = np.zeros((B * T, scfg.max_speakers), np.float32), np.zeros(B, np.int32)
    toks = asr._tokens(B)
    L, dec = asr.L, int(pkg.Decoder.TDT)

    def joint_pinned():
        asr._check(L.pk_transcribe_diarize_batch(asr.h, diar.h, pkg.engine._f32p(pin), pkg.engine._i64p(off), B, dec,
                                                 toks[0], pkg.engine._f32p(probs), pkg.engine._i32p(lens)), "joint")

    def separate_pinned():
        asr.transcribe_packed(pin, off, pkg.Decoder.TDT, toks)
        diar.stage(pin, off)
        diar.run_diarize_staged()
        diar.fetch_probs(probs, lens)

    def asr_pinned():
        asr.transcribe_packed(pin, off, pkg.Decoder.TDT, toks)

    def joint_resident():
        asr.run_transcribe_diarize_staged(diar, pkg.Decoder.TDT)
        asr.fetch_into(toks)
        diar.fetch_probs(probs, lens)

    def separate_resident():
        asr.run_staged(pkg.Decoder.TDT)
        diar.run_diarize_staged()
        asr.fetch_into(toks)
        diar.fetch_probs(probs, lens)

    def asr_resident():
        asr.run_staged(pkg.Decoder.TDT)
        asr.fetch_into(toks)

    streams = [asr.stream(), diar.stream()]
    res = {"utterances": B, "seconds": seconds}
    for name, fn in (("joint", joint_pinned), ("separate", separate_pinned), ("asr", asr_pinned)):
        res[f"{name}_pinned_ms"] = round(timed(torch, streams, fn, steps, warmup), 3)
    asr.stage(pin, off)
    asr.run_transcribe_diarize_staged(diar, pkg.Decoder.TDT)
    asr.sync()
    res["joint_resident_ms"] = round(timed(torch, streams, joint_resident, steps, warmup), 3)
    asr.stage(pin, off)
    diar.stage(pin, off)
    for name, fn in (("separate", separate_resident), ("asr", asr_resident)):
        res[f"{name}_resident_ms"] = round(timed(torch, streams, fn, steps, warmup), 3)
    res["x_real_time_joint_pinned"] = round(B * seconds * 1e3 / res["joint_pinned_ms"], 1)
    asr.close()
    diar.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="64x10,16x60")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("diarized_bench: no CUDA device")
    pkg = ge.load_package()
    from parakeet_cpp_b200 import synth
    O = ge.load_oracle()
    c0 = card()
    out = {"models": "tdt-ctc-110m (TDT) + sortformer-117m", "math": "bf16x3", "steps": a.steps, "warmup": a.warmup, "runs": []}
    with tempfile.TemporaryDirectory() as td:
        for c in a.configs.split(","):
            B, s = c.split("x")
            out["runs"].append(run_config(pkg, torch, synth, O, td, int(B), float(s), a.steps, a.warmup))
    out["card"] = c0
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
