"""What CTC forced alignment costs: tdt-ctc-110m on 64 x 10 s clips per step, greedy CTC against PK_DECODER_CTC_ALIGN of each
clip's greedy transcript (so both arms decode the same audio and the alignment has the greedy transcript's length).

    python tools/ctc_align_bench.py [--rounds 5] [--steps 20] [--out FILE]

The two arms are alternated --rounds times inside this one call after a warm-up of each (device-resident PCM, the whole
path per step, device events around the timed steps); the line reports every round, so the spread is in it.  The CTC
decode-class device time (pk_profile_*: the frame pass, and for the alignment its kernel and the collapse) comes from a
separate profiled pass per arm.  One JSON line, with the card name and power limit read in the same call; --out also writes
it to a file.  Synthetic weights are written under --tmp.
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

ROWS, CLIP = 64, 160000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception:
        return "", ""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--tmp", default=os.environ.get("PK_BENCH_TMP", "/tmp/pk_bench"))
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("ctc_align_bench.py needs a CUDA device")
    os.makedirs(args.tmp, exist_ok=True)
    pkg = ge.load_package()
    O = ge.load_oracle()
    from parakeet_cpp_b200 import synth
    cfg = pkg.make_110m_config(max_batch=ROWS)
    wp = os.path.join(args.tmp, "pk110m_seed0.safetensors")
    if not os.path.exists(wp):
        synth.save_safetensors(wp + ".tmp", synth.make_weights(O.make_110m_config(), seed=0))
        os.replace(wp + ".tmp", wp)

    eng = pkg.Engine(cfg, wp, 0)
    buf = torch.empty(ROWS * CLIP, dtype=torch.float32).pin_memory().numpy()
    for i in range(ROWS):
        buf[i * CLIP:(i + 1) * CLIP] = synth.make_audio(CLIP, 5000 + i)
    off = np.arange(ROWS + 1, dtype=np.int64) * CLIP
    eng.job_stage(buf, off)
    eng.job_select(0, ROWS)
    stream = torch.cuda.ExternalStream(eng.stream(), device=0)
    eng.run_staged(pkg.Decoder.CTC)
    greedy = eng.fetch(ROWS)
    eng.set_align_targets([[t.token_id for t in r] for r in greedy])
    arms = {"greedy": pkg.Decoder.CTC, "align": pkg.Decoder.CTC_ALIGN}

    def steps(dec, k):
        for _ in range(k):
            eng.run_staged(dec)

    for dec in arms.values():                          # warm-up: a graph per arm
        steps(dec, 3)
    key = lambda rows: [[(t.token_id, t.start_frame, t.end_frame) for t in r] for r in rows]
    same = key(eng.fetch(ROWS)) == key(greedy)         # (the last warm-up step was the alignment)
    times = {a: [] for a in arms}
    for _ in range(args.rounds):
        for a, dec in arms.items():
            steps(dec, 2)
            eng.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            steps(dec, args.steps)
            e1.record(stream)
            eng.sync()
            times[a].append(round(e0.elapsed_time(e1) / args.steps, 3))
    ctc_ms = {}
    for a, dec in arms.items():
        steps(dec, 2)
        eng.profile_begin()
        steps(dec, 3)
        ctc_ms[a] = round(eng.profile_end()["ctc"][0] / 3, 4)
    eng.close()
    name, limit = card()
    extra = [round(x - y, 3) for x, y in zip(times["align"], times["greedy"])]
    line = dict(tool="ctc_align_bench", workload=f"tdt-ctc-110m, {ROWS} x {CLIP // 16000} s synthetic clips per step, device-resident PCM; "
                "alignment targets = the greedy transcripts", gpu=name, power_limit=limit, rounds=args.rounds, steps=args.steps,
                ms_per_step_device=times, align_minus_greedy_ms=extra, ctc_class_ms=ctc_ms,
                tokens_per_step=int(sum(len(r) for r in greedy)), align_rows_equal_greedy=same)
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
