"""Sortformer's new kernels against float64 references, through their test hooks (pk_kernel_mha, pk_kernel_speaker_head) and
the LayerNorm at d 192 (pk_kernel_layernorm), with per-element bounds and the 0xFF guard bands checked.

Attention bound.  PK_MATH_FP32 runs the CUDA-core kernel: s_ij = fl(q_i . k_j) * scale with fp32 FMAs (hd = 24 terms), an
online softmax with fp32 exps, o_i = sum_j p_ij v_j / l_i.  The bf16 modes run the mma.sync kernel on operands split into
bf16 hi (+ lo).  hi + lo represents an operand to 2^-17 relative, and hi*hi + hi*lo + lo*hi drops lo*lo (2^-18), so one
product errs by at most u_op |x y| with u_op = 3 * 2^-17 <= 2^-15 (hi alone: 2 * 2^-9 + 2^-18 <= 2^-7).  With u = 2^-24,
the score errs by at most ((hd + 1) u + u_op) scale |q_i| |k_j| = e_s (fp32 accumulation plus the split, Cauchy-Schwarz);
a score error moves every normalised weight by a factor within exp(+-2 e_s); P and V enter P V split (u_op); so
    |do_ic| <= (2 e_s + (T + 8) u + u_op) sum_j p_ij |v_jc|
(T + 8: the fp32 sums over keys, the rescales and the final division, each a relative u).  Bound = 4x that (margin for
expf's few-ulp error), plus, for bf16 planes, the storage rounding of the output: 2^-8 |o| for hi alone, 2^-16 |o| for
hi + lo.

Mutated references (must exceed the bound somewhere): scale 1/sqrt(32), one key past the utterance's end, keys from the
neighbouring utterance, and bf16-hi-only q / k / v operands (against the bf16x3 and fp32 kernels)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

U = 2.0 ** -24
HD, D, H = 24, 192, 8


def _bf16(x):
    a = np.ascontiguousarray(x, np.float32).view(np.uint32)
    r = ((a + 0x7FFF + ((a >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return r.view(np.float32)


U_OP = {0: 2.0 ** -15, 1: 2.0 ** -7, 2: 0.0}      # split error of one product per math mode (pk_math), see above


def _attn64(qkv, off, scale=1 / np.sqrt(24.0), extra_key=False, neighbour=False, math=2):
    uo = U_OP[math]
    q, k, v = (qkv[:, i * D:(i + 1) * D].astype(np.float64) for i in range(3))
    out = np.full((qkv.shape[0], D), np.nan)
    bound_terms = np.zeros((qkv.shape[0], D))
    for b in range(len(off) - 1):
        r0, r1 = off[b], off[b + 1]
        k0, k1 = r0, r1
        if extra_key:
            k1 = r1 + 1
        if neighbour and b + 1 < len(off) - 1:
            k1 = off[b + 2]
        for h in range(H):
            sl = slice(h * HD, (h + 1) * HD)
            s = q[r0:r1, sl] @ k[k0:k1, sl].T * scale
            p = np.exp(s - s.max(axis=1, keepdims=True))
            p /= p.sum(axis=1, keepdims=True)
            out[r0:r1, sl] = p @ v[k0:k1, sl]
            T = r1 - r0
            es = ((HD + 1) * U + uo) * scale * np.linalg.norm(q[r0:r1, sl], axis=1)[:, None] * np.linalg.norm(k[k0:k1, sl], axis=1)[None, :]
            bound_terms[r0:r1, sl] = 4 * ((2 * es.max(axis=1, keepdims=True) + (T + 8) * U + uo) * (p @ np.abs(v[k0:k1, sl])))
    return out, bound_terms


def _run(pkg, qkv, off, math):
    L = pkg.load_library()
    rows = qkv.shape[0]
    off32 = np.asarray(off, np.int32)
    f32 = np.zeros((rows, D), np.float32) if math == 2 else None
    hi = np.zeros((rows, D), np.float32) if math != 2 else None
    lo = np.zeros((rows, D), np.float32) if math == 0 else None
    gb = np.zeros(1, np.int64)
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None  # noqa: E731
    st = L.pk_kernel_mha(0, math, len(off) - 1, off32.ctypes.data_as(C.POINTER(C.c_int32)), rows, D, H, p(qkv), p(f32), p(hi), p(lo),
                         gb.ctypes.data_as(C.POINTER(C.c_int64)))
    assert st == 0
    assert gb[0] == 0
    return f32 if math == 2 else (hi + lo if math == 0 else hi)


CASES = {
    "one_frame": [1, 1, 3],
    "tile_edges": [63, 64, 65, 1, 128, 129],
    "long": [300, 17],
}


def _inputs(lens, seed):
    """Utterance b = rows [starts[b], starts[b] + lens[b]), each followed by one NaN row."""
    rng = np.random.default_rng(seed)
    qkv = (rng.standard_normal((sum(lens) + len(lens), 3 * D)) * 1.5).astype(np.float32)
    starts = np.concatenate([[0], np.cumsum(np.asarray(lens) + 1)[:-1]]).tolist()
    for a, n in zip(starts, lens):
        qkv[a + n] = np.nan
    return qkv, [(a, a + n) for a, n in zip(starts, lens)]


@pytest.mark.gpu
@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("case", sorted(CASES))
def test_mha_against_fp64(pkg, math, case):
    lens = CASES[case]
    qkv, pairs = _inputs(lens, 11)
    # prefix offsets: each NaN row is a one-row utterance of its own (a key leaking across utterances would make NaNs), and
    # the last one lies outside every utterance
    row_off = [0]
    for a, b in pairs:
        row_off += [b, b + 1]
    row_off = row_off[:-1]
    got = _run(pkg, qkv, row_off, math)
    ref, bnd = _attn64(np.nan_to_num(qkv, nan=0.0), row_off, math=math)
    real = np.zeros(qkv.shape[0], bool)
    for a, b in pairs:
        real[a:b] = True
    store = {0: 2.0 ** -16, 1: 2.0 ** -8, 2: 0.0}[math]
    bound = bnd + store * np.abs(ref) + 1e-30
    err = np.abs(got[real] - ref[real])
    ratio = float((err / bound[real]).max())
    print(f"mha {case} math {math}: max error/bound {ratio:.3g}")
    assert ratio <= 1.0
    if math != 1:
        # mutated references must be rejected
        mutants = {
            "scale_1/sqrt(32)": _attn64(qkv, row_off, scale=1 / np.sqrt(32.0))[0],
            "bf16_hi_operands": _attn64(_bf16(qkv), row_off)[0],
        }
        for name, mref in mutants.items():
            assert float((np.abs(got[real] - mref[real]) / bound[real]).max()) > 1.0, name


@pytest.mark.gpu
@pytest.mark.parametrize("math", [0, 2])
def test_mha_keys_stay_in_the_utterance(pkg, math):
    rng = np.random.default_rng(5)
    lens = [40, 70, 33]
    off = np.concatenate([[0], np.cumsum(lens)]).tolist()
    qkv = rng.standard_normal((off[-1] + 1, 3 * D)).astype(np.float32)
    got = _run(pkg, qkv, off, math)
    ref, bnd = _attn64(qkv, off, math=math)
    bound = bnd + {0: 2.0 ** -16, 2: 0.0}[math] * np.abs(ref) + 1e-30
    n = off[-1]
    assert float((np.abs(got[:n] - ref[:n]) / bound[:n]).max()) <= 1.0
    assert np.isnan(got[n]).all()                         # the row outside every utterance is not written
    extra = _attn64(qkv, off, extra_key=True)[0]
    neigh = _attn64(qkv, off, neighbour=True)[0]
    assert float((np.abs(got[:off[1]] - extra[:off[1]]) / bound[:off[1]]).max()) > 1.0
    assert float((np.abs(got[:off[1]] - neigh[:off[1]]) / bound[:off[1]]).max()) > 1.0


@pytest.mark.gpu
def test_mha_rejects_other_head_dims(pkg):
    L = pkg.load_library()
    qkv = np.zeros((8, 3 * 256), np.float32)
    out = np.zeros((8, 256), np.float32)
    off = np.array([0, 8], np.int32)
    gb = np.zeros(1, np.int64)
    st = L.pk_kernel_mha(0, 2, 1, off.ctypes.data_as(C.POINTER(C.c_int32)), 8, 256, 4, qkv.ctypes.data_as(C.POINTER(C.c_float)),
                         out.ctypes.data_as(C.POINTER(C.c_float)), None, None, gb.ctypes.data_as(C.POINTER(C.c_int64)))
    assert st == 1


@pytest.mark.gpu
def test_speaker_head_against_fp64(pkg):
    L = pkg.load_library()
    rng = np.random.default_rng(3)
    M, Dh, S = 37, 192, 4
    x = rng.standard_normal((M, Dh)).astype(np.float32)
    w1 = (rng.standard_normal((Dh, Dh)) / np.sqrt(Dh)).astype(np.float32)
    b1 = (0.1 * rng.standard_normal(Dh)).astype(np.float32)
    w2 = (rng.standard_normal((S, Dh)) / np.sqrt(Dh)).astype(np.float32)
    b2 = (0.1 * rng.standard_normal(S)).astype(np.float32)
    probs = np.zeros((M, S), np.float32)
    gb = np.zeros(1, np.int64)
    f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
    assert L.pk_kernel_speaker_head(0, M, Dh, S, f(x), f(w1), f(b1), f(w2), f(b2), f(probs), gb.ctypes.data_as(C.POINTER(C.c_int64))) == 0
    assert gb[0] == 0
    x64 = np.maximum(x.astype(np.float64), 0)
    h = np.maximum(x64 @ w1.T.astype(np.float64) + b1, 0)
    lg = h @ w2.T.astype(np.float64) + b2
    ref = 1 / (1 + np.exp(-lg))
    # |d logit| <= 2 (D + 1) u (|W2| |h| + |W2| |W1| |x| ...): bounded by 4 D u sum of absolute products
    habs = np.abs(x64) @ np.abs(w1.T.astype(np.float64)) + np.abs(b1)
    dl = 4 * (Dh + 2) * U * (np.abs(h) @ np.abs(w2.T.astype(np.float64)) + habs @ np.abs(w2.T.astype(np.float64)) + np.abs(b2))
    bound = 0.25 * dl + 8 * U
    ratio = float((np.abs(probs - ref) / bound).max())
    print(f"speaker head: max error/bound {ratio:.3g}")
    assert ratio <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("d", [192, 64, 320])
def test_layernorm_at_widths_below_a_multiple_of_128(pkg, d):
    L = pkg.load_library()
    rng = np.random.default_rng(d)
    M = 21
    x = (rng.standard_normal((M, d)) * 3 + 1).astype(np.float32)
    w = (1 + 0.1 * rng.standard_normal(d)).astype(np.float32)
    b = (0.1 * rng.standard_normal(d)).astype(np.float32)
    y = np.zeros((M, d), np.float32)
    act = np.zeros((M, d), np.float32)
    gb = np.zeros(1, np.int64)
    f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
    st = L.pk_kernel_layernorm(0, M, d, f(x), f(w), f(b), None, None, 1, 3, f(y), f(act), None, None, gb.ctypes.data_as(C.POINTER(C.c_int64)))
    assert st == 0 and gb[0] == 0
    x64 = x.astype(np.float64)
    mu = x64.mean(1, keepdims=True)
    var = ((x64 - mu) ** 2).mean(1, keepdims=True)
    ref = (x64 - mu) / np.sqrt(var + 1e-5) * w + b
    bound = 8 * (d + 4) * U * (np.abs((x64 - mu) / np.sqrt(var + 1e-5) * w) + np.abs(b)) + 1e-30
    assert float((np.abs(y - ref) / bound).max()) <= 1.0
    assert np.array_equal(y, act)
    # the bf16 hi / lo planes (the next GEMM's operand in bf16x3), every element including each lane's partial last float4
    hi, lo = np.zeros((M, d), np.float32), np.zeros((M, d), np.float32)
    y2 = np.zeros((M, d), np.float32)
    st = L.pk_kernel_layernorm(0, M, d, f(x), f(w), f(b), None, None, 1, 2, f(y2), None, f(hi), f(lo), gb.ctypes.data_as(C.POINTER(C.c_int64)))
    assert st == 0 and gb[0] == 0
    assert np.array_equal(y2, y)
    assert np.array_equal(hi, _bf16(y))
    assert np.array_equal(lo, _bf16(y - hi))


@pytest.mark.gpu
@pytest.mark.parametrize("math", [0, 1])
def test_qkv_projection_at_d192(pkg, math):
    """The wgmma GEMM with EPI_QKV_ACT as the transformer runs it (N = 576, K = 192, qcols 192: q columns end inside a
    128-column tile) equals the fp32 CUDA-core GEMM within the split error."""
    L = pkg.load_library()
    rng = np.random.default_rng(9)
    M, N, K = 300, 3 * D, D
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(N)).astype(np.float32)
    f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None  # noqa: E731
    gb = np.zeros(1, np.int64)
    q = np.zeros((M, D), np.float32)
    hi, lo = np.zeros((M, 2 * D), np.float32), (np.zeros((M, 2 * D), np.float32) if math == 0 else None)
    st = L.pk_kernel_gemm(0, 1, math, 1, M, N, K, 7, D, 2 * D, 1.0, 0, f(A), f(W), f(bias), None, f(q), f(hi), f(lo),
                          gb.ctypes.data_as(C.POINTER(C.c_int64)))
    assert st == 0 and gb[0] == 0
    ref = A.astype(np.float64) @ W.T.astype(np.float64) + bias
    mag = np.abs(A).astype(np.float64) @ np.abs(W.T).astype(np.float64) + np.abs(bias)
    tol = (4 * K * U + 4 * U_OP[math]) * mag + U_OP[math] * np.abs(ref)
    kv = hi + lo if math == 0 else hi
    assert (np.abs(q - ref[:, :D]) <= tol[:, :D]).all()
    assert (np.abs(kv - ref[:, D:]) <= tol[:, D:] + (2.0 ** -16 if math == 0 else 2.0 ** -8) * np.abs(ref[:, D:])).all()
