"""What phrase boosting costs: each workload with boosting off, with one list shared by every row (pk_set_boost; streams:
the same list on every stream) and with a different list on every row (pk_set_boost_rows before EVERY batch, as a server
that batches different requests would call it; streams: pk_stream_set_boost per stream).  A fourth arm, "rows-same", sends
the shared list through the per-row path, so that the cost of the mechanism (a trie slot per row, the upload) can be told from
the cost of the lists being different (the batch decodes in lock step, so its length is that of its slowest row).  Streams
only have the per-stream form, so there "shared" and "rows-same" are the same arm measured twice.

    python tools/boost_bench.py [--workloads 110m-tdt,110m-ctc,nemotron-600m,eou-120m] [--rounds 3] [--steps 20]

Workloads: tdt-ctc-110m, 64 x 10 s clips, TDT and CTC (device-resident PCM, the whole path per step); nemotron-600m and
eou-120m, 64 streams of 160 ms chunks through pk_stream_step (host PCM in, host tokens out).  The arms are alternated
--rounds times inside this one call; a line reports the time of every round, so the spread is in the line.  Per-class
device time (pk_profile_*) comes from a separate profiled pass per arm.  One JSON line per workload and arm, with the card
name and power limit read in the same call.

Lists: 20 phrases of 3 random token ids per list (seeded), score 5; "rows" gives row i the list of seed i.  Synthetic
seeded weights are written under --tmp; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import __graft_entry__ as ge  # noqa: E402
from rnnt_bench import gpu_name  # noqa: E402

ROWS, CLIP, CH, SCORE = 64, 160000, 2560, 5.0
ARMS = ("off", "shared", "rows-same", "rows")


def phrase_list(vocab, seed):
    r = np.random.default_rng(9000 + seed)
    return [r.integers(0, vocab - 1, 3).tolist() for _ in range(20)]


def weights(pkg, synth, cfg, tmp, name):
    wp = os.path.join(tmp, f"pk{name}_seed0.safetensors")
    if not os.path.exists(wp):
        synth.save_safetensors(wp + ".tmp", synth.make_weights(cfg, seed=0))
        os.replace(wp + ".tmp", wp)
    return wp


def offline(pkg, synth, args, dec_name):
    import torch
    cfg = pkg.make_110m_config(max_batch=ROWS)
    eng = pkg.Engine(cfg, weights(pkg, synth, cfg, args.tmp, "110m"), 0)
    dec = pkg.Decoder.TDT if dec_name == "tdt" else pkg.Decoder.CTC
    buf = torch.empty(ROWS * CLIP, dtype=torch.float32).pin_memory().numpy()
    for i in range(ROWS):
        buf[i * CLIP:(i + 1) * CLIP] = synth.make_audio(CLIP, 5000 + i)
    off = np.arange(ROWS + 1, dtype=np.int64) * CLIP
    eng.job_stage(buf, off)
    eng.job_select(0, ROWS)
    lists = [phrase_list(cfg.vocab, i) for i in range(ROWS)]
    scores = [SCORE] * ROWS
    stream = torch.cuda.ExternalStream(eng.stream(), device=0)

    def arm_on(arm):
        eng.set_boost([], 0.0)
        eng.set_boost_rows([], [])
        if arm == "shared":
            eng.set_boost(lists[0], SCORE)

    def steps(arm, k):
        for _ in range(k):
            if arm == "rows":
                eng.set_boost_rows(lists, scores)          # a new set of lists for every batch
            elif arm == "rows-same":
                eng.set_boost_rows([lists[0]] * ROWS, scores)
            eng.run_staged(dec)

    times = {a: [] for a in ARMS}
    host = {a: [] for a in ARMS}
    tokens = {}
    for a in ARMS:                                         # warm-up: graphs captured for every arm
        arm_on(a)
        steps(a, 3)
        tokens[a] = int(sum(len(u) for u in eng.fetch(ROWS)))
    for _ in range(args.rounds):
        for a in ARMS:
            arm_on(a)
            steps(a, 2)
            eng.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            w0 = time.perf_counter()
            e0.record(stream)
            steps(a, args.steps)
            e1.record(stream)
            eng.sync()
            host[a].append(1e3 * (time.perf_counter() - w0) / args.steps)
            times[a].append(e0.elapsed_time(e1) / args.steps)
    prof = {}
    for a in ARMS:
        arm_on(a)
        steps(a, 2)
        eng.profile_begin()
        steps(a, 3)
        prof[a] = {k: v[0] / 3 for k, v in eng.profile_end().items() if v[1]}
    arm_on("off")
    eng.close()
    wl = f"tdt-ctc-110m {dec_name.upper()} decode, {ROWS} x {CLIP // 16000} s synthetic clips per step, device-resident PCM"
    return wl, times, host, prof, tokens, "ms_per_step_device"


def streaming(pkg, synth, args, model):
    make = {"nemotron-600m": "make_nemotron_600m_config", "eou-120m": "make_eou_120m_config"}[model]
    cfg = getattr(pkg, make)(max_batch=ROWS)
    eng = pkg.Engine(cfg, weights(pkg, synth, cfg, args.tmp, model.replace("-", "")), 0)
    eng.stream_open(ROWS, CH)
    K = args.steps
    pcm = [synth.make_audio((K + 4) * CH, 1200 + i) for i in range(ROWS)]
    lists = [phrase_list(cfg.vocab, i) for i in range(ROWS)]
    out = eng._tokens(ROWS)

    def arm_on(arm):
        for i in range(ROWS):
            eng.stream_set_boost(i, [] if arm == "off" else lists[i if arm == "rows" else 0], SCORE)
        eng.stream_reset(-1)

    def run(k):
        n = 0
        for j in range(k):
            n += int(eng.stream_step([x[j * CH:(j + 1) * CH] for x in pcm], out=out, raw=True)["len"].sum())
        return n

    times = {a: [] for a in ARMS}
    tokens = {}
    for a in ARMS:
        arm_on(a)
        run(K + 4)
    for _ in range(args.rounds):
        for a in ARMS:
            arm_on(a)
            run(4)
            eng.sync()
            w0 = time.perf_counter()
            tokens[a] = run(K)
            eng.sync()
            times[a].append(1e3 * (time.perf_counter() - w0) / K)
    prof = {}
    for a in ARMS:
        arm_on(a)
        run(2)
        eng.profile_begin()
        for j in range(2, 10):
            eng.stream_step([x[j * CH:(j + 1) * CH] for x in pcm], out=out, raw=True)
        prof[a] = {k: v[0] / 8 for k, v in eng.profile_end().items() if v[1]}
    eng.close()
    wl = f"{model} streaming TDT decode, {ROWS} streams in lock step, {CH}-sample (160 ms) chunks, host PCM in and tokens out every step"
    return wl, times, None, prof, tokens, "ms_per_step_wall"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="110m-tdt,110m-ctc,nemotron-600m,eou-120m")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--tmp", default=os.environ.get("PK_BENCH_TMP", "/tmp/pk_bench"))
    args = ap.parse_args()
    os.makedirs(args.tmp, exist_ok=True)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("boost_bench.py: no CUDA device (the engine has no CPU fallback)")
    pkg = ge.load_package()
    from parakeet_cpp_b200 import synth
    sampler = bench.ClockSampler(0)
    sampler.start()
    results = []
    for w in args.workloads.split(","):
        results.append((w, offline(pkg, synth, args, w.split("-")[1]) if w.startswith("110m-") else streaming(pkg, synth, args, w)))
    clocks = sampler.stop()
    for w, (wl, times, host, prof, tokens, what) in results:
        for a in ARMS:
            line = {"bench": "boost", "workload_id": w, "arm": a, "workload": wl, what: float(np.median(times[a])),
                    "rounds_ms": times[a], "steps_per_round": args.steps, "tokens_per_round": tokens[a],
                    "vs_off": float(np.median(times[a]) / np.median(times["off"])), "per_class_ms": prof[a],
                    "lists": "none" if a == "off" else f"20 phrases x 3 tokens, score {SCORE}" + (", one per row" if a == "rows" else "") + (", re-sent every batch" if a.startswith("rows") and host else ""),
                    "gpu_name": gpu_name(), "power_limit_w": clocks.get("power_limit_w"), "sm_clock_mhz": clocks.get("sm_mhz")}
            if host:
                line["rounds_host_ms"] = host[a]
            print(json.dumps(line))


if __name__ == "__main__":
    main()
