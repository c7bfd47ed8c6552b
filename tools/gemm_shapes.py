#!/usr/bin/env python
"""gemm_shapes.py -- times the encoder's GEMM shapes one by one on the wgmma kernel (gemm_tc.cu).

    python tools/gemm_shapes.py [--models 110m,600m] [--math bf16x3,bf16x1] [--json OUT]

Every shape goes through pk_selftest_gemm with PK_SELFTEST_TIME=1: one launch checked against the fp32 CUDA-core GEMM,
then warm back-to-back launches over a window of >= 50 ms timed with CUDA events.  The table gives the time per launch,
the algorithmic rate, the rate the tensor pipe issues (three MMAs per product for bf16x3) and that rate as a share of
what the card can issue at the SM clock sampled during the run (SMs x 4096 dense bf16 FLOP per clock).  The environment
selects the kernel form as in the engine (PK_GEMM_CLUSTER=2|4: the wide GEMMs as clusters with the A tile multicast).
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
from bench import ClockSampler  # noqa: E402

EPI = dict(SILU_ACT=3, RESID=4, GLU=5, QKV=7)
MATH = dict(bf16x3=0, bf16x1=1)
# (name, M, N, K, epilogue): M = the packed rows of one batch (110m: 64 x 10 s clips = 64 x 126 frames; 600m: 16 x 30 s
# clips = 16 x 376 frames); per layer fc1 and fc2 run twice (two macaron feed-forward modules)
SHAPES = {
    "110m": [("fc1", 8064, 2048, 512, "SILU_ACT"), ("qkv", 8064, 1536, 512, "QKV"), ("pw1", 8064, 1024, 512, "GLU"),
             ("out/pw2", 8064, 512, 512, "RESID"), ("fc2", 8064, 512, 2048, "RESID")],
    "600m": [("fc1", 6016, 4096, 1024, "SILU_ACT"), ("qkv", 6016, 3072, 1024, "QKV"), ("pw1", 6016, 2048, 1024, "GLU"),
             ("out/pw2", 6016, 1024, 1024, "RESID"), ("fc2", 6016, 1024, 4096, "RESID")],
}
LINE = re.compile(r"gemm_tc M=(\d+) N=(\d+) K=(\d+) .*: ([0-9.]+) us")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def timed(selftest, M, N, K, epi, math):
    """-> (us per launch, max_err / max_ref): the library prints its timing on the process's stderr."""
    with tempfile.TemporaryFile(mode="w+") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            err, ref = selftest(M, N, K, epi, math)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        m = [LINE.search(x) for x in f.read().splitlines()]
    us = [float(x.group(4)) for x in m if x]
    if not us:
        raise RuntimeError(f"no timing line for M={M} N={N} K={K}")
    return us[-1], err / max(ref, 1e-30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="110m,600m")
    ap.add_argument("--math", default="bf16x3,bf16x1")
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    a = ap.parse_args()
    os.environ["PK_SELFTEST_TIME"] = "1"
    pkg = ge.load_package()
    from parakeet_cpp_b200.engine import selftest_gemm
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    info = card()
    print(f"card: {info}  ({sms} SMs)  PK_GEMM_CLUSTER={os.environ.get('PK_GEMM_CLUSTER', '-')}  lib={pkg.engine.lib_path()}")
    print(f"{'model':5} {'gemm':8} {'M':>5} {'N':>5} {'K':>5} {'epi':8} {'math':6} {'us':>9} {'alg TF/s':>9} "
          f"{'issued':>7} {'sm MHz':>6} {'of peak':>7} {'rel err':>8}")
    rows = []
    for model in a.models.split(","):
        for math in a.math.split(","):
            for name, M, N, K, epi in SHAPES[model]:
                cs = ClockSampler(0)
                cs.start()
                for _ in range(100):        # nvidia-smi is sampling before the timed window starts
                    if cs.rows:
                        break
                    time.sleep(0.05)
                us, rel = timed(selftest_gemm, M, N, K, EPI[epi], MATH[math])
                clk = cs.stop()
                alg = 2.0 * M * N * K / (us * 1e-6) / 1e12
                issued = alg * (3 if math == "bf16x3" else 1)
                mhz = clk["sm_mhz"] or clk["sm_max_mhz"]
                peak = sms * 4096 * mhz * 1e6 / 1e12 if mhz else float("nan")
                rows.append(dict(model=model, gemm=name, M=M, N=N, K=K, epi=epi, math=math, us=us, alg_tflops=alg,
                                 issued_tflops=issued, sm_mhz=mhz, frac_of_issue_peak=issued / peak, rel_err=rel))
                print(f"{model:5} {name:8} {M:5d} {N:5d} {K:5d} {epi:8} {math:6} {us:9.2f} {alg:9.1f} {issued:7.1f} "
                      f"{mhz:6.0f} {100 * issued / peak:6.1f}% {rel:8.1e}", flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=info, sms=sms, cluster=os.environ.get("PK_GEMM_CLUSTER"), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
