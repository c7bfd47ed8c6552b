"""What the CTC prefix beam search costs: tdt-ctc-110m on 64 x 10 s clips per step, greedy CTC against PK_DECODER_CTC_BEAM at
widths 4, 8, 16 and 32, each without a language model and with a seeded generated 3-gram of about 10^5 n-grams over words
spelled from the synthetic vocabulary's pieces (nothing is downloaded).

    python tools/ctc_beam_bench.py [--rounds 3] [--steps 10] [--out FILE]

The arms are alternated --rounds times inside this one call (device-resident PCM, the whole path per step, device events
around the timed steps); the line reports every round, so the spread is in it.  The CTC decode-class device time
(pk_profile_*: the frame pass, top-W and beam kernels) comes from a separate profiled pass per arm.  One JSON line, with
the card name and power limit read in the same call.  Synthetic weights, vocabulary and LM are written under --tmp.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__ as ge  # noqa: E402
import ctc_beam_oracle as CB  # noqa: E402

ROWS, CLIP = 64, 160000
WIDTHS = (4, 8, 16, 32)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception:
        return "", ""


def lm_words(pieces, n, seed):
    rng = np.random.default_rng(seed)
    starts = [p[1:] for p in pieces if p.startswith(CB.SP_MARK) and len(p) > 1]
    conts = [p for p in pieces if not p.startswith(CB.SP_MARK)]
    out = set()
    while len(out) < n:
        out.add(starts[int(rng.integers(len(starts)))] + "".join(conts[int(rng.integers(len(conts)))] for _ in range(int(rng.integers(0, 3)))))
    return sorted(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--tmp", default=os.environ.get("PK_BENCH_TMP", "/tmp/pk_bench"))
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("ctc_beam_bench.py needs a CUDA device")
    os.makedirs(args.tmp, exist_ok=True)
    pkg = ge.load_package()
    O = ge.load_oracle()
    from parakeet_cpp_b200 import synth
    cfg = pkg.make_110m_config(max_batch=ROWS)
    wp = os.path.join(args.tmp, "pk110m_seed0.safetensors")
    if not os.path.exists(wp):
        synth.save_safetensors(wp + ".tmp", synth.make_weights(O.make_110m_config(), seed=0))
        os.replace(wp + ".tmp", wp)
    pieces = synth.make_vocab(cfg.vocab - 1, seed=0)
    vp = os.path.join(args.tmp, "pk110m_vocab.txt")
    synth.save_vocab(vp, pieces)
    arpa = os.path.join(args.tmp, "pk110m_3gram.arpa")
    grams = CB.make_arpa(arpa, lm_words(pieces, 5000, 1), 3, seed=1, per_order=47500)
    lm = pkg.LanguageModel(arpa)
    tok = pkg.engine.Tokenizer(vp)

    eng = pkg.Engine(cfg, wp, 0)
    buf = torch.empty(ROWS * CLIP, dtype=torch.float32).pin_memory().numpy()
    for i in range(ROWS):
        buf[i * CLIP:(i + 1) * CLIP] = synth.make_audio(CLIP, 5000 + i)
    off = np.arange(ROWS + 1, dtype=np.int64) * CLIP
    eng.job_stage(buf, off)
    eng.job_select(0, ROWS)
    stream = torch.cuda.ExternalStream(eng.stream(), device=0)
    arms = ["greedy"] + [f"beam{w}" for w in WIDTHS] + [f"beam{w}+lm" for w in WIDTHS]

    def arm_on(a):
        if a == "greedy":
            return pkg.Decoder.CTC
        w = int(a[4:].split("+")[0])
        eng.set_ctc_beam(w, lm if a.endswith("+lm") else None, tok, 0.5, 1.0)
        return pkg.Decoder.CTC_BEAM

    def steps(dec, k):
        for _ in range(k):
            eng.run_staged(dec)

    times = {a: [] for a in arms}
    ntok = {}
    for a in arms:                                     # warm-up: a graph per arm
        dec = arm_on(a)
        steps(dec, 3)
        ntok[a] = int(sum(len(u) for u in eng.fetch(ROWS)))
    for _ in range(args.rounds):
        for a in arms:
            dec = arm_on(a)
            steps(dec, 2)
            eng.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            steps(dec, args.steps)
            e1.record(stream)
            eng.sync()
            times[a].append(round(e0.elapsed_time(e1) / args.steps, 3))
    ctc_ms = {}
    for a in arms:
        dec = arm_on(a)
        steps(dec, 2)
        eng.profile_begin()
        steps(dec, 3)
        ctc_ms[a] = round(eng.profile_end()["ctc"][0] / 3, 3)
    eng.close()
    name, limit = card()
    line = dict(tool="ctc_beam_bench", workload=f"tdt-ctc-110m CTC decode, {ROWS} x {CLIP // 16000} s synthetic clips per step, device-resident PCM",
                lm=f"3-gram, {len(grams)} n-grams, alpha 0.5, beta 1.0", gpu=name, power_limit=limit, rounds=args.rounds, steps=args.steps,
                ms_per_step_device=times, ctc_class_ms=ctc_ms, tokens_per_step=ntok)
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "a") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
