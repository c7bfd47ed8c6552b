"""The ping-pong GEMM's staged epilogue (shared-memory chunks written by TMA stores) against the register epilogue, byte for
byte, through pk_kernel_gemm.

The register epilogue stays in the cooperative cluster forms (cluster 2 and 4), which run the same MMA sequence per
element as the ping-pong kernel (cluster 1), and in the ping-pong kernel for launches TMA cannot store (N or ldo not a
multiple of 4, such as the CTC head).  So:
  * SILU_ACT, GLU_F32 and QKV_ACT on the ping-pong kernel write the same bytes as on the cluster forms;
  * BIAS_F32 writes the same bytes as the q columns of a cluster-form QKV_ACT whose first qcols weight and bias rows are
    its own;
  * every other kind equals its element-wise function of BIAS_F32 on the same operands: RELU_F32 = max(v, 0), the act
    planes = the bf16 split (hi = rn(v), lo = rn(v - hi)) of v or of max(v, 0), RESID_F32 = float32(r + alpha v) with
    alpha a power of two (the product is exact, so FMA contraction cannot change the sum).
Every launch also has to leave the guard bands around its outputs alone.
"""
from __future__ import annotations

import numpy as np
import pytest

from test_kernels_fp64 import EPI, MATH_X1, MATH_X3, bf16_rn, gemm_inputs, run_gemm

gpu = pytest.mark.gpu

ROWS = (1, 65, 129, 8063, 8064)


def same_bytes(a, b):
    return a is None and b is None or (a is not None and b is not None and np.array_equal(a.view(np.uint32), b.view(np.uint32)))


def launch(pkg, mth, cl, M, N, K, kind, ldo, inputs, alpha=1.0, in_place=False, q=0, lo=True):
    o = run_gemm(pkg, 1, mth, cl, M, N, K, EPI[kind], ldo, alpha, in_place, q, lo, inputs=inputs)
    assert o["guard_bad"] == 0
    return o


def rng_for(M, N, K):
    return np.random.default_rng(M * 131 + N * 17 + K)


# (kind, N, K, qcols): the 110m and 600m widths of the GEMMs that also run as clusters
CLUSTER_SHAPES = [("SILU_ACT", 2048, 512, 0), ("GLU_F32", 1024, 512, 0), ("QKV_ACT", 1536, 512, 512),
                  ("SILU_ACT", 4096, 1024, 0), ("GLU_F32", 2048, 1024, 0), ("QKV_ACT", 3072, 1024, 1024)]


@gpu
@pytest.mark.parametrize("M", ROWS)
@pytest.mark.parametrize("kind,N,K,q", CLUSTER_SHAPES, ids=lambda v: str(v))
def test_pingpong_matches_cluster_forms(pkg, kind, N, K, q, M):
    ldo = N // 2 if kind == "GLU_F32" else N - q
    inputs = gemm_inputs(rng_for(M, N, K), M, N, K, EPI[kind], ldo)
    ref = launch(pkg, MATH_X3, 1, M, N, K, kind, ldo, inputs, q=q)
    for cl in (2, 4):
        o = launch(pkg, MATH_X3, cl, M, N, K, kind, ldo, inputs, q=q)
        for k in ("of", "oh", "ol"):
            assert same_bytes(ref[k], o[k]), f"{k} differs from cluster {cl}"


@gpu
@pytest.mark.parametrize("M", ROWS)
@pytest.mark.parametrize("q,K", [(512, 512), (1024, 1024)])
def test_bias_f32_matches_cluster_qkv_q_columns(pkg, q, K, M):
    N = 3 * q
    A, W, b, _ = gemm_inputs(rng_for(M, N, K), M, N, K, EPI["QKV_ACT"], N - q)
    o = launch(pkg, MATH_X3, 1, M, q, K, "BIAS_F32", q, (A, W[:q].copy(), b[:q].copy(), None))
    for cl in (2, 4):
        r = launch(pkg, MATH_X3, cl, M, N, K, "QKV_ACT", N - q, (A, W, b, None), q=q)
        assert same_bytes(o["of"], r["of"]), f"q columns differ from cluster {cl}"


# (M, N, K, ldo): the 110m / 600m residual and projection widths, the CTC head widths (ldo padded to 4), and staged
# launches whose last column tile is partial: N % 128 of 4 (1028), 32 (96), 64 (1088) and 100 % 128, and the 64-column
# tile (N <= 64: 40, 64, 36).  At 1028, 100 and 36 the bf16 planes take the register epilogue (a row is not a multiple of
# 16 B) while the fp32 outputs are staged.
F32_SHAPES = [(M, 512, 512, 512) for M in ROWS] + [(M, 512, 2048, 512) for M in (65, 8064)] + \
             [(M, 1024, 1024, 1024) for M in (1, 129, 8063)] + [(65, 1025, 512, 1028), (8064, 1025, 512, 1028), (65, 33, 128, 36)] + \
             [(129, 1028, 512, 1028), (65, 1088, 512, 1088), (129, 96, 256, 96), (65, 100, 128, 100), (129, 40, 128, 40),
              (65, 64, 256, 64), (8063, 36, 128, 36)]


def split_planes(v, N, ldo, want_lo):
    hi = np.full(v.shape[:1] + (ldo,), np.nan, np.float32)
    lo = hi.copy() if want_lo else None
    hi[:, :N] = bf16_rn(v[:, :N])
    if want_lo:
        lo[:, :N] = bf16_rn((v[:, :N] - hi[:, :N]).astype(np.float32))
    return hi, lo


@gpu
@pytest.mark.parametrize("mth", [MATH_X3, MATH_X1], ids=["x3", "x1"])
@pytest.mark.parametrize("M,N,K,ldo", F32_SHAPES, ids=lambda v: str(v))
def test_epilogue_kinds_match_bias_f32(pkg, M, N, K, ldo, mth):
    inputs = gemm_inputs(rng_for(M, N, K), M, N, K, EPI["RESID_F32"], ldo)
    A, W, b, r = inputs
    v = launch(pkg, mth, 1, M, N, K, "BIAS_F32", ldo, inputs)["of"]
    assert np.all(np.isfinite(v[:, :N])) and np.all(np.isnan(v[:, N:]))
    relu = np.where(np.isnan(v), v, np.maximum(v, np.float32(0)))

    o = launch(pkg, mth, 1, M, N, K, "RELU_F32", ldo, inputs)["of"]
    assert np.array_equal(o, relu, equal_nan=True)

    for kind, val in (("BIAS_ACT", v), ("RELU_ACT", relu)):
        for want_lo in (True, False):
            o = launch(pkg, mth, 1, M, N, K, kind, ldo, inputs, lo=want_lo)
            hi, lo = split_planes(val, N, ldo, want_lo)
            assert np.array_equal(o["oh"], hi, equal_nan=True), f"{kind} hi"
            if want_lo:
                assert np.array_equal(o["ol"], lo, equal_nan=True), f"{kind} lo"
            else:
                assert o["ol"] is None

    for alpha in (0.5, 1.0):
        want = r[:, :N] + np.float32(alpha) * v[:, :N]
        for in_place in (False, True):
            o = launch(pkg, mth, 1, M, N, K, "RESID_F32", ldo, inputs, alpha=alpha, in_place=in_place)["of"]
            assert np.array_equal(o[:, :N], want), f"RESID alpha {alpha} in_place {in_place}"
            assert np.all(np.isnan(o[:, N:]))
