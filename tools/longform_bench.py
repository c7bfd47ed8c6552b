"""Long-form offline transcription with limited-context attention (DESIGN.md section 16).

    python tools/longform_bench.py [--runs all|110m-60|600m-60|110m-8x20|110m-5-ab|600m-180-mem] [--reps 2] [--tmp DIR]

One JSON line per run: card name and power limit (read in the same call), model, band, audio minutes, the time per call
from CUDA events on the engine stream after one warm-up call (PCM staged on the device once, mel -> encoder -> TDT greedy,
tokens fetched), RTFx, the per-class device times of one profiled call (attention vs GEMM, the TDT decode), and the engine's
own device memory (cudaMemGetInfo before its creation and after its warm-up call; its workspace is allocated once, so this is
also its peak, as long as nothing else on the card allocates in between).  Runs:
  110m-60     110m, one 60-minute utterance, band (256, 256)
  600m-60     tdt-600m, one 60-minute utterance, band (256, 256)
  110m-8x20   110m, 8 x 20 minutes, band (256, 256)
  110m-5-ab   110m, one 5-minute utterance, full attention and band (256, 256) alternated on two engines in one process
  600m-180-mem  tdt-600m engine with max_samples = 3 h, band (256, 256): device memory of the engine only
Synthetic seeded checkpoints go under --tmp; nothing is written into the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

SR = 16000
BAND = (256, 256)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=60).stdout.strip().split(",")
    return {"gpu_name": r[0].strip(), "power_limit_w": float(r[1])}


def weights(pkg, synth, cfg, tmp, tag):
    wp = os.path.join(tmp, f"longform_{tag}_seed0.safetensors")
    if not os.path.exists(wp):
        synth.save_safetensors(wp + ".tmp", synth.make_weights(cfg, seed=0))
        os.replace(wp + ".tmp", wp)
    return wp


def used_gb(torch):
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2 ** 30


class Run:
    """One engine with one staged batch: timed calls and a profiled call."""

    def __init__(self, pkg, torch, cfg, wp, pcms):
        self.pkg, self.torch = pkg, torch
        m0 = used_gb(torch)
        self.eng = pkg.Engine(cfg, wp, 0)
        self.n = len(pcms)
        lens = [len(p) for p in pcms]
        self.buf = torch.empty(sum(lens), dtype=torch.float32).pin_memory().numpy()
        self.off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        for i, p in enumerate(pcms):
            self.buf[self.off[i]:self.off[i + 1]] = p
        self.stream = torch.cuda.ExternalStream(self.eng.stream(), device=0)
        self.eng.stage(self.buf, self.off)
        self.call()                                      # warm-up: first sight of the shape, lazy initialisation
        self.mem_gb = used_gb(torch) - m0                # this engine's device memory (its workspace is allocated once)

    def call(self):
        self.eng.run_staged(self.pkg.Decoder.TDT)
        return self.eng.fetch(self.n)

    def timed(self, reps):
        ms = []
        for _ in range(reps):
            e0, e1 = self.torch.cuda.Event(enable_timing=True), self.torch.cuda.Event(enable_timing=True)
            e0.record(self.stream)
            self.eng.run_staged(self.pkg.Decoder.TDT)
            e1.record(self.stream)
            self.eng.sync()
            ms.append(e0.elapsed_time(e1))
        self.tokens = self.eng.fetch(self.n)
        return ms

    def profile(self):
        self.eng.profile_begin()
        self.eng.run_staged(self.pkg.Decoder.TDT)
        prof = self.eng.profile_end()
        return {k: round(v[0], 3) for k, v in prof.items() if v[1]}

    def close(self):
        self.eng.close()


def line(c, name, model, band, minutes, n_utt, ms, prof, mem, extra=None):
    audio_s = minutes * 60 * n_utt
    d = dict(c, run=name, model=model, band=list(band), audio_minutes=minutes, n_utterances=n_utt, ms_per_call=[round(x, 2) for x in ms],
             ms_per_call_median=round(float(np.median(ms)), 2), rtfx=round(audio_s / (float(np.median(ms)) / 1e3), 1),
             per_class_ms=prof, engine_device_mem_gb=round(mem, 2), decoder="tdt greedy", math="bf16x3")
    d.update(extra or {})
    print(json.dumps(d), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", default="all")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--tmp", default=os.environ.get("PK_BENCH_TMP", "/tmp/pk_bench"))
    args = ap.parse_args()
    os.makedirs(args.tmp, exist_ok=True)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("longform_bench.py: no CUDA device (the engine has no CPU fallback)")
    pkg = ge.load_package()
    from parakeet_cpp_b200 import synth
    runs = args.runs.split(",") if args.runs != "all" else ["110m-5-ab", "110m-60", "110m-8x20", "600m-60", "600m-180-mem"]
    c = card()
    base = {"110m": pkg.make_110m_config(), "600m": pkg.make_tdt_600m_config()}
    wps = {}

    def wp(m):
        if m not in wps:
            wps[m] = weights(pkg, synth, base[m], args.tmp, m)
        return wps[m]

    import dataclasses
    for name in runs:
        if name == "110m-5-ab":
            n = 5 * 60 * SR
            pcm = synth.make_audio(n, 5)
            r = {}
            for b in ((0, 0), BAND):                       # created one after the other: each memory delta is that engine's own
                r[b] = Run(pkg, torch, dataclasses.replace(base["110m"], max_batch=1, max_samples=n, local_attention=b), wp("110m"), [pcm])
            ms = {b: [] for b in r}
            for _ in range(max(args.reps, 3)):             # alternated: the two engines see the same card state
                for b in r:
                    ms[b] += r[b].timed(1)
            for b in r:
                line(c, name, "tdt-ctc-110m", b, 5, 1, ms[b], r[b].profile(), r[b].mem_gb)
                r[b].close()
        elif name in ("110m-60", "600m-60", "110m-8x20"):
            m = name.split("-")[0]
            minutes, n_utt = (20, 8) if name == "110m-8x20" else (60, 1)
            n = minutes * 60 * SR
            pcms = [synth.make_audio(n, 60 + i) for i in range(n_utt)]
            cfg = dataclasses.replace(base[m], max_batch=n_utt, max_samples=n, local_attention=BAND)
            r = Run(pkg, torch, cfg, wp(m), pcms)
            ms = r.timed(args.reps)
            T = r.eng.L.pk_encoder_frames(r.eng.L.pk_mel_frames(n))
            ok = all(len(u) <= r.eng.cap and all(0 <= t.start_frame <= t.end_frame < T for t in u) for u in r.tokens)
            line(c, name, base[m].name, BAND, minutes, n_utt, ms, r.profile(), r.mem_gb,
                 {"encoder_frames_per_utterance": T, "tokens": [len(u) for u in r.tokens], "timestamps_in_range": ok})
            r.close()
        elif name == "600m-180-mem":
            m0 = used_gb(torch)
            e = pkg.Engine(dataclasses.replace(base["600m"], max_batch=1, max_samples=3 * 3600 * SR, local_attention=BAND), wp("600m"), 0)
            m1 = used_gb(torch)
            e.close()
            print(json.dumps(dict(c, run=name, model="tdt-600m", band=list(BAND), audio_minutes=180, n_utterances=1,
                                  engine_device_mem_gb=round(m1 - m0, 2))), flush=True)
        else:
            raise SystemExit(f"unknown run {name}")


if __name__ == "__main__":
    main()
