"""Throughput and latency of lock-step streaming: S streams of 160 ms chunks through pk_stream_step.

    python tools/stream_bench.py --model {eou-120m,nemotron-600m} [--streams 64] [--latency 0] [--steps 125] [--warmup 24]

Prints one JSON line shaped like `bench.py --config eou-120m-stream`: `value` = audio seconds per wall second over the
timed steps (host PCM in, host tokens out every step), ms per step (= the chunk latency of every stream in it), the
single-stream latency on a one-stream engine (the reference's operating point), per-class device time and launches of
one step (pk_profile_*), and the card name, power limit and SM clock sampled during the timed region.

Synthetic seeded weights (seed 0) are written under --tmp; nothing is read from outside the tree and nothing is written
into it.  Stream i gets make_audio(seed = base + i) with base 1200 (eou-120m) or 1400 (nemotron-600m).  The one-stream
engine also replays the golden fixture's stream (golden_stream_v1.npz / golden_nemotron_v1.npz: 14 chunks of the same
seed, same weights), so the line says whether it gave the reference's tokens.
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

CH = 2560                    # 160 ms at 16 kHz
MODELS = {"eou-120m": ("make_eou_120m_config", 1200, "golden_stream_v1.npz", "eou120"),
          "nemotron-600m": ("make_nemotron_600m_config", 1400, "golden_nemotron_v1.npz", "nemo600")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=sorted(MODELS), default="nemotron-600m")
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--latency", type=int, default=None,
                    help="att_context_right (nemotron-600m latency mode, default 0; eou-120m default 1); no effect on the output")
    ap.add_argument("--steps", type=int, default=125, help="timed chunk steps (125 = 20 s per stream)")
    ap.add_argument("--warmup", type=int, default=24)
    ap.add_argument("--tmp", default=os.environ.get("PK_BENCH_TMP", "/tmp/pk_bench"))
    args = ap.parse_args()
    args.steps, args.warmup = max(args.steps, 14), max(args.warmup, 2)
    os.makedirs(args.tmp, exist_ok=True)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("stream_bench.py: no CUDA device (the engine has no CPU fallback)")
    pkg = ge.load_package()
    from parakeet_cpp_b200 import synth
    make, seed_base, golden, tag = MODELS[args.model]
    S, K = args.streams, args.steps

    def config(n):
        kw = dict(max_batch=max(n, 8))
        if args.latency is not None:
            kw["att_context_right"] = args.latency
        return getattr(pkg, make)(**kw)

    cfg = config(S)
    wp = os.path.join(args.tmp, f"pk{args.model.replace('-', '')}_seed0.safetensors")
    if not os.path.exists(wp):
        synth.save_safetensors(wp + ".tmp", synth.make_weights(cfg, seed=0))
        os.replace(wp + ".tmp", wp)
    streams = [synth.make_audio(K * CH, seed_base + i) for i in range(S)]
    eng = pkg.Engine(cfg, wp, 0)
    eng.stream_open(S, CH)
    out = eng._tokens(S)

    def run(e, o, rows, steps):
        ntok = 0
        for k in range(steps):
            arrs = e.stream_step([x[k * CH:(k + 1) * CH] for x in rows], out=o, raw=True)
            ntok += int(arrs["len"].sum())
        return ntok

    run(eng, out, streams, min(args.warmup, K))            # warm-up: every chunk pattern seen, graphs instantiated
    eng.stream_reset(-1)
    eng.sync()
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.2)
    l0 = eng.launch_count()
    t0 = time.perf_counter()
    ntok = run(eng, out, streams, K)
    eng.sync()
    wall = time.perf_counter() - t0
    clocks = sampler.stop()
    launches = (eng.launch_count() - l0) / K
    # per-class device time of one step (a separate, profiled pass over the first chunks)
    eng.stream_reset(-1)
    P = 8
    run(eng, out, streams, 2)
    eng.profile_begin()
    for k in range(2, 2 + P):
        eng.stream_step([x[k * CH:(k + 1) * CH] for x in streams], out=out, raw=True)
    prof = eng.profile_end()
    eng.close()
    # single-stream latency (the reference's case)
    e1 = pkg.Engine(config(1), wp, 0)
    e1.stream_open(1, CH)
    o1 = e1._tokens(1)
    run(e1, o1, streams[:1], min(args.warmup, K))
    e1.stream_reset(-1)
    e1.sync()
    k1 = min(K, 125)
    t1 = time.perf_counter()
    run(e1, o1, streams[:1], k1)
    e1.sync()
    lat1 = (time.perf_counter() - t1) / k1
    g = np.load(os.path.join(ROOT, "tests", "golden", golden))
    sched = [int(v) for v in g[tag + ".schedule"]]
    gpcm = synth.make_audio(sum(sched), int(g[tag + ".seeds"][1]))
    e1.stream_reset(-1)
    got, pos = [], 0
    for n in sched:
        got.append([[t.token_id, t.start_frame, t.end_frame] for t in e1.stream_step([gpcm[pos:pos + n]])[0]])
        pos += n
    match = got == [g[f"{tag}.k{ci}.tok"].tolist() for ci in range(len(sched))]
    e1.close()
    audio_s = S * K * CH / 16000.0
    value = audio_s / wall
    line = {"metric": f"audio-seconds/sec (RTFx) {args.model} streaming, 160 ms chunks", "value": value, "unit": "x real-time",
            "n_gpus": 1, "steps": K, "warmup": min(args.warmup, K), "ms_per_step": 1e3 * wall / K, "higher_is_better": True,
            "dtype": {0: "bf16x3", 1: "bf16", 2: "f32"}[int(cfg.math)], "data": "synthetic",
            "config": {"model": args.model, "workload": f"{args.model} streaming TDT decode, {S} concurrent 16 kHz streams in lock step, "
                       f"{CH}-sample (160 ms) chunks, {K} chunks per stream ({K * CH / 16000.0:g} s)", "streams": S, "chunk_samples": CH,
                       "latency_frames": cfg.att_context_right, "max_batch": cfg.max_batch, "tokens_emitted": ntok},
            "latency": {"ms_per_chunk_step_all_streams": 1e3 * wall / K, "ms_per_chunk_single_stream": 1e3 * lat1, "real_time_budget_ms": 160.0},
            "per_class_ms": {k: v[0] / P for k, v in prof.items() if v[1]}, "per_class_launches": {k: v[1] / P for k, v in prof.items() if v[1]},
            "gpu_launches": launches, "wall_s": wall,
            "golden_stream_matches_reference": match,
            "gpu_name": gpu_name(), "power_limit_w": clocks.get("power_limit_w"), "sm_clock_mhz": clocks.get("sm_mhz"), "clocks": clocks}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
