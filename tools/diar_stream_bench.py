"""Throughput and latency of lock-step streaming diarization: S sortformer-117m streams through pk_diar_stream_step.

    python tools/diar_stream_bench.py [--streams 64] [--chunk 2560] [--seconds 60] [--warmup 16]

Prints one JSON line: `value` = audio seconds per wall second over the timed steps (host PCM in, host activities out
every step), ms per step (= the chunk latency of every stream in it), the single-stream chunk latency on a one-stream
engine against the chunk's duration, per-class device time and launches of one step (pk_profile_*, a separate pass),
the weight bytes a step reads (bf16 hi + lo planes of every matrix of the loaded checkpoint) over the step time against
the H100 SXM's 3.35 TB/s, and the card name, power limit and SM clock sampled during the timed region.

Synthetic seeded weights (seed 0) are written under --tmp; nothing is read from outside the tree and nothing is written
into it.  Stream i gets make_audio(seed = 1600 + i).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import __graft_entry__ as ge  # noqa: E402
from rnnt_bench import gpu_name  # noqa: E402

HBM_PEAK = 3.35e12           # H100 SXM data sheet, bytes/s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--chunk", type=int, default=2560, help="samples per chunk (2560 = 160 ms)")
    ap.add_argument("--seconds", type=float, default=60.0, help="audio per stream")
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--tmp", default=os.environ.get("PK_BENCH_TMP", "/tmp/pk_bench"))
    args = ap.parse_args()
    os.makedirs(args.tmp, exist_ok=True)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("diar_stream_bench.py: no CUDA device (the engine has no CPU fallback)")
    pkg = ge.load_package()
    from parakeet_cpp_b200 import synth
    S, CH = args.streams, args.chunk
    K = int(args.seconds * 16000) // CH

    def config(n):
        return pkg.make_sortformer_117m_config(max_batch=max(n, 1), max_samples=160000)

    cfg = config(S)
    W = synth.make_sortformer_weights(cfg, seed=0)
    wbytes = sum(4 * v.size for k, v in W.items() if v.ndim >= 2 and not k.startswith("hidden_to_spks_"))
    wp = os.path.join(args.tmp, "pksortformer117m_seed0.safetensors")
    if not os.path.exists(wp):
        synth.save_safetensors(wp + ".tmp", W)
        os.replace(wp + ".tmp", wp)
    streams = [synth.make_audio(K * CH, 1600 + i) for i in range(S)]

    def run(e, rows, k0, k1):
        frames = 0
        for k in range(k0, k1):
            p, _ = e.diar_stream_step([x[k * CH:(k + 1) * CH] for x in rows])
            frames += sum(len(q) for q in p)
        return frames

    eng = pkg.Engine(cfg, wp, 0)
    eng.diar_stream_open(S, CH)
    run(eng, streams, 0, min(args.warmup, K))     # every chunk pattern seen, graphs instantiated
    eng.diar_stream_reset(-1)
    eng.sync()
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.2)
    l0 = eng.launch_count()
    t0 = time.perf_counter()
    frames = run(eng, streams, 0, K)
    eng.sync()
    wall = time.perf_counter() - t0
    clocks = sampler.stop()
    launches = (eng.launch_count() - l0) / K
    eng.diar_stream_reset(-1)
    P = 8
    run(eng, streams, 0, 2)
    eng.profile_begin()
    run(eng, streams, 2, 2 + P)
    prof = eng.profile_end()
    eng.close()
    e1 = pkg.Engine(config(1), wp, 0)                 # single-stream latency (the reference's case)
    e1.diar_stream_open(1, CH)
    run(e1, streams[:1], 0, min(args.warmup, K))
    e1.diar_stream_reset(-1)
    e1.sync()
    k1 = min(K, 200)
    t1 = time.perf_counter()
    run(e1, streams[:1], 0, k1)
    e1.sync()
    lat1 = (time.perf_counter() - t1) / k1
    e1.close()
    step_s = wall / K
    per_class = {k: v[0] / P for k, v in prof.items() if v[1]}
    dev_ms = sum(per_class.values())
    line = {"metric": "audio-seconds/sec (RTFx) sortformer-117m streaming diarization", "value": S * K * CH / 16000.0 / wall,
            "unit": "x real-time", "n_gpus": 1, "steps": K, "warmup": min(args.warmup, K), "ms_per_step": 1e3 * step_s,
            "higher_is_better": True, "dtype": "bf16x3", "data": "synthetic",
            "config": {"model": "sortformer-117m", "workload": f"sortformer-117m streaming diarization, {S} concurrent 16 kHz streams in "
                       f"lock step, {CH}-sample ({CH / 16:g} ms) chunks, {K} chunks per stream ({K * CH / 16000.0:g} s)",
                       "streams": S, "chunk_samples": CH, "encoder_frames": frames},
            "latency": {"ms_per_chunk_step_all_streams": 1e3 * step_s, "ms_per_chunk_single_stream": 1e3 * lat1,
                        "chunk_duration_ms": CH / 16.0},
            "per_class_ms": per_class, "per_class_launches": {k: v[1] / P for k, v in prof.items() if v[1]},
            "mha_share_of_device_time": per_class.get("mha", 0.0) / dev_ms if dev_ms else None,
            "weight_bytes_per_step": wbytes, "weight_bandwidth_share_of_hbm_peak": wbytes / step_s / HBM_PEAK,
            "gpu_launches_per_step": launches, "wall_s": wall,
            "gpu_name": gpu_name(), "power_limit_w": clocks.get("power_limit_w"), "sm_clock_mhz": clocks.get("sm_mhz"), "clocks": clocks}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
