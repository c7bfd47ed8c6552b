"""Each hot-path kernel against float64 math, element by element, through the pk_kernel_* hooks.

A hook runs one launcher exactly as the engine calls it and returns every output buffer whole.  Outputs sit between guard
bands and start as 0xFF bytes (NaN), so a test sees (1) whether any byte outside the buffers changed (guard_bad), (2) the
exact set of elements the kernel wrote (finite) and left alone (NaN), and (3) each written element's error against a float64
reference of the same operation on the exact fp32 inputs, divided by a per-element bound derived below.  Every case prints
its largest error / bound ratio.

Bounds (u = 2^-24, the fp32 unit roundoff; P = |A| . |W|^T in float64):
  bf16x3 GEMM  x = hi + lo + r with |r| <= 2^-16 |x|.  hi.hi + hi.lo + lo.hi drops lo.lo and the residuals: each is <= 2^-16
               |a||w|, so |err| <= 3 * 2^-16 P, plus fp32 accumulation that, summed in tiles, stays far below that.  C_X3 = 8.
  bf16x1 GEMM  hi only: |hi - x| <= 2^-8 |x|, so |err| <= (2 * 2^-8 + 2^-16) P.  C_X1 = 4.
  fp32 SIMT    sequential fma over K: |err| <= K u P (Higham, gamma_K).  C_F32 = 2.
  epilogues    + fp32 rounding of the bias add and the result (4 u (|acc| + |bias|)); ReLU is 1-Lipschitz, SiLU 1.1; GLU a *
               sigmoid(b): e_a + 0.25 |a| e_b; RESID resid + alpha v: |alpha| e + 4 u (|resid| + |alpha v|).  The tensor-core
               epilogues use fast_sigmoid (ex2.approx + rcp.approx): relative error <= 2^-20 + |x| 2^-22 (the ex2 argument is
               rounded, which costs |x| log2(e) u), added to every sigmoid.
  act planes   hi + lo stands for the fp32 value y within 2^-16 |y| (hi alone: 2^-8 |y|, half an ulp, so a correct kernel
               can come close to the bound there); |y| <= |ref| + bound.
Inputs span magnitudes (A rows scaled by 10^U(-3,3), W rows by 10^U(-2,2)), so a fault confined to small rows is not hidden
under the large ones: the bound of every element is its own.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest

gpu = pytest.mark.gpu

U = 2.0 ** -24
C_X3, C_X1, C_F32 = 8.0, 4.0, 2.0
EPI = dict(BIAS_F32=0, RELU_F32=1, RELU_ACT=2, SILU_ACT=3, RESID_F32=4, GLU_F32=5, BIAS_ACT=6, QKV_ACT=7)
MATH_X3, MATH_X1, MATH_F32 = 0, 1, 2
SEEDS = (1, 2, 3)
SAMPLE_ROWS = 256          # float64 references of the larger shapes on this many sampled rows (every row is sentinel-checked)


# ----------------------------------------------------------------------------------------------------------- helpers
def bf16_rn(x):
    """fp32 -> bf16 (round to nearest even), returned as fp32."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def split(x):
    x = np.asarray(x, np.float32)
    hi = bf16_rn(x)
    return hi, bf16_rn((x - hi).astype(np.float32))


def f32p(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def i32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def nan(shape):
    return np.full(shape, np.nan, np.float32)


def ratio(got, ref, bound):
    """max |got - ref| / bound over the elements (NaN-propagating: a NaN output counts as infinite)."""
    e = np.abs(got.astype(np.float64) - ref)
    r = e / np.maximum(bound, 1e-300)
    r = np.where(np.isnan(r), np.inf, r)
    return float(r.max()) if r.size else 0.0


def check_planes(hi, lo, ref, bound, mask=None):
    """hi is the bf16 rounding of hi + lo (|lo| <= half an ulp of hi, a tie only when lo sits exactly on it) and hi + lo is
    within the bound; without a lo plane hi itself is.  -> error / bound ratio."""
    if mask is not None:
        hi, ref, bound = hi[mask], ref[mask], bound[mask]
        lo = None if lo is None else lo[mask]
    assert np.all(bf16_rn(hi) == hi)
    if lo is None:
        return ratio(hi, ref, bound + 2.0 ** -8 * (np.abs(ref) + bound))
    assert np.all(bf16_rn(lo) == lo)
    nz = hi != 0
    ulp = np.zeros_like(hi, dtype=np.float64)
    ulp[nz] = 2.0 ** (np.floor(np.log2(np.abs(hi[nz].astype(np.float64)))) - 7)
    assert np.all(np.abs(lo[nz].astype(np.float64)) <= 0.5 * ulp[nz]), "lo is not the residual of hi"
    assert np.all(lo[~nz] == 0)
    s = hi.astype(np.float64) + lo.astype(np.float64)
    tie = np.abs(lo.astype(np.float64)) == 0.5 * ulp
    assert np.all((bf16_rn(s.astype(np.float32)) == hi) | tie)
    return ratio(s, ref, bound + 2.0 ** -16 * (np.abs(ref) + bound))


def report(name, r):
    print(f"[fp64] {name}: max err/bound = {r:.3g}")


def fast_sig_rel(x):
    return 2.0 ** -20 + np.abs(x) * 2.0 ** -22


def sig64(x):
    with np.errstate(over="ignore"):          # exp(-x) = inf for very negative x: sigmoid 0, as wanted
        return 1.0 / (1.0 + np.exp(-x))


# ----------------------------------------------------------------------------------------------------------- references
def ref_gemm(A, W, bias, resid, kind, alpha, math_mode, qcols=0, Ahi_only=False, e_in=None):
    """float64 linear + epilogue -> (value [M, N'], bound [M, N']), for the q part and the rest when kind is QKV.
    e_in: a per-element bound on the error of A (a chain of kernels): it adds e_in . |W|^T, and the kernel's own term is
    taken on |A| + e_in."""
    A64, W64 = A.astype(np.float64), W.astype(np.float64)
    if Ahi_only:                             # mutation: operands rounded to bf16 (hi only)
        A64, W64 = bf16_rn(A).astype(np.float64), bf16_rn(W).astype(np.float64)
    acc = A64 @ W64.T
    P = (np.abs(A64) if e_in is None else np.abs(A64) + e_in) @ np.abs(W64).T
    K = A.shape[1]
    eps = {MATH_X3: C_X3 * 2.0 ** -16, MATH_X1: C_X1 * 2.0 ** -8, MATH_F32: C_F32 * K * U}[math_mode] * P
    b = np.zeros(W.shape[0]) if bias is None else bias.astype(np.float64)
    v = acc + b
    e = eps + 4 * U * (np.abs(acc) + np.abs(b))
    if e_in is not None:
        e = e + e_in @ np.abs(W64).T
    if kind in (EPI["RELU_F32"], EPI["RELU_ACT"]):
        return np.maximum(v, 0), e
    if kind == EPI["SILU_ACT"]:
        y = v * sig64(v)
        return y, 1.1 * e + np.abs(y) * fast_sig_rel(v) + 4 * U * np.abs(y)
    if kind == EPI["RESID_F32"]:
        r = resid[:, :W.shape[0]].astype(np.float64)
        y = r + alpha * v
        return y, abs(alpha) * e + 4 * U * (np.abs(r) + np.abs(alpha * v))
    if kind == EPI["GLU_F32"]:
        a, g, ea, eg = v[:, 0::2], v[:, 1::2], e[:, 0::2], e[:, 1::2]
        y = a * sig64(g)
        return y, ea + 0.25 * np.abs(a) * eg + np.abs(y) * fast_sig_rel(g) + 4 * U * np.abs(y)
    return v, e


def gemm_inputs(rng, M, N, K, kind, ldo, bias=True):
    A = (rng.uniform(-1, 1, (M, K)) * 10.0 ** rng.uniform(-3, 3, (M, 1))).astype(np.float32)
    W = (rng.uniform(-1, 1, (N, K)) * 10.0 ** rng.uniform(-2, 2, (N, 1)) / math.sqrt(K)).astype(np.float32)
    b = (1e-3 * rng.uniform(-1, 1, N)).astype(np.float32) if bias else None
    r = None
    if kind == EPI["RESID_F32"]:
        r = nan((M, ldo))                         # the ldo padding columns stay NaN: the kernel must neither read nor write them
        r[:, :N] = rng.uniform(-1, 1, (M, N)) * 10.0 ** rng.uniform(-3, 3, (M, 1))
    return A, W, b, r


def run_gemm(pkg, path, math_mode, cluster, M, N, K, kind, ldo, alpha=1.0, in_place=False, qcols=0, want_lo=True, seed=1, inputs=None):
    L = pkg.load_library()
    rng = np.random.default_rng(seed * 7919 + M * 31 + N * 7 + K)
    A, W, b, r = inputs or gemm_inputs(rng, M, N, K, kind, ldo)
    qkv, glu = kind == EPI["QKV_ACT"], kind == EPI["GLU_F32"]
    act = kind in (EPI["RELU_ACT"], EPI["SILU_ACT"], EPI["BIAS_ACT"]) or qkv
    planes = act and path != 0
    of = nan((M, qcols) if qkv else (M, ldo)) if (not planes or qkv) else None
    oh = nan((M, ldo)) if planes else None
    ol = nan((M, ldo)) if planes and want_lo else None
    gb = C.c_int64(-1)
    st = L.pk_kernel_gemm(0, path, math_mode, cluster, M, N, K, kind, qcols, ldo, alpha, int(in_place), f32p(A), f32p(W), f32p(b),
                          f32p(r), f32p(of), f32p(oh), f32p(ol), C.byref(gb))
    assert st == 0, f"pk_kernel_gemm -> {st}"
    return dict(A=A, W=W, b=b, r=r, of=of, oh=oh, ol=ol, guard_bad=gb.value)


def sample_rows(M, seed):
    if M <= SAMPLE_ROWS:
        return np.arange(M)
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([[0, M - 1], np.arange(M - 64, M), rng.choice(M, SAMPLE_ROWS, replace=False)]))


def check_gemm(o, path, math_mode, M, N, K, kind, ldo, alpha, qcols, seed, mutate=False):
    """Asserts the written set and returns the largest error / bound ratio over the sampled rows."""
    assert o["guard_bad"] == 0
    qkv, glu = kind == EPI["QKV_ACT"], kind == EPI["GLU_F32"]
    n_out = N // 2 if glu else N - qcols if qkv else N
    main = o["oh"] if o["oh"] is not None else o["of"]
    assert np.all(np.isfinite(main[:, :n_out])), "an output element was not written"
    assert np.all(np.isnan(main[:, n_out:])), "the kernel wrote into the ldo padding"
    if o["ol"] is not None:
        assert np.all(np.isfinite(o["ol"][:, :n_out])) and np.all(np.isnan(o["ol"][:, n_out:]))
    if qkv:
        assert np.all(np.isfinite(o["of"]))
    rows = sample_rows(M, seed)
    A, r = o["A"][rows], None if o["r"] is None else o["r"][rows]
    ref_kind = EPI["BIAS_F32"] if qkv else kind
    y, bd = ref_gemm(A, o["W"], o["b"], r, ref_kind, alpha, math_mode, Ahi_only=mutate)
    if qkv:
        rq = ratio(o["of"][rows], y[:, :qcols], bd[:, :qcols])
        yk, bk = y[:, qcols:], bd[:, qcols:]
        return max(rq, check_planes(o["oh"][rows, :n_out], None if o["ol"] is None else o["ol"][rows, :n_out], yk, bk))
    if o["oh"] is not None:
        return check_planes(o["oh"][rows, :n_out], None if o["ol"] is None else o["ol"][rows, :n_out], y, bd)
    return ratio(main[rows, :n_out], y, bd)


# (path, math, cluster, M, N, K, kind, ldo, alpha, in_place, qcols, want_lo): the engine's calls for tiny / 110m / 600m
# (CTC head with ldo = (vocab + 3) & ~3, RESID in place, QKV with qcols = d) and the tile edges of M, N and K.
def _g(path, mth, cl, M, N, K, kind, ldo=None, alpha=1.0, inp=False, q=0, lo=True):
    k = EPI[kind]
    if ldo is None:
        ldo = N // 2 if kind == "GLU_F32" else N - q
    return (path, mth, cl, M, N, K, k, ldo, alpha, inp, q, lo)


GEMM_CASES = [
    # wgmma, bf16x3
    _g(1, MATH_X3, 1, 65, 33, 128, "BIAS_F32", ldo=36),                 # tiny CTC head
    _g(1, MATH_X3, 1, 376, 1025, 512, "BIAS_F32", ldo=1028),            # 110m CTC head
    _g(1, MATH_X3, 1, 129, 1025, 1024, "BIAS_F32", ldo=1028),           # 600m-width CTC head
    _g(1, MATH_X3, 1, 8064, 2048, 512, "SILU_ACT"),                     # 110m fc1, 64 x 10 s
    _g(1, MATH_X3, 1, 376, 512, 2048, "RESID_F32", alpha=0.5, inp=True),  # 110m fc2 (+ residual, in place)
    _g(1, MATH_X3, 1, 127, 1024, 1024, "RESID_F32", alpha=1.0, inp=True),  # 600m out_proj
    _g(1, MATH_X3, 1, 64, 384, 640, "RESID_F32", alpha=0.5),
    _g(1, MATH_X3, 1, 376, 1536, 512, "QKV_ACT", q=512),                # 110m q | k | v
    _g(1, MATH_X3, 1, 65, 3072, 1024, "QKV_ACT", q=1024),               # 600m q | k | v
    _g(1, MATH_X3, 1, 129, 1024, 512, "GLU_F32"),                       # 110m pw1
    _g(1, MATH_X3, 1, 6016, 2048, 1024, "GLU_F32"),                     # 600m pw1
    _g(1, MATH_X3, 1, 17, 640, 640, "RELU_F32"),
    _g(1, MATH_X3, 1, 63, 384, 4096, "RELU_ACT"),
    _g(1, MATH_X3, 1, 128, 4096, 1024, "BIAS_ACT"),                     # 600m fc1 width
    _g(1, MATH_X3, 1, 1, 640, 2560, "BIAS_F32"),
    _g(1, MATH_X3, 1, 8064, 640, 64, "BIAS_F32"),
    # wgmma, bf16x1 (with and without a lo plane)
    _g(1, MATH_X1, 1, 376, 2048, 512, "SILU_ACT"),
    _g(1, MATH_X1, 1, 376, 2048, 512, "SILU_ACT", lo=False),
    _g(1, MATH_X1, 1, 129, 512, 2048, "RESID_F32", alpha=0.5, inp=True),
    _g(1, MATH_X1, 1, 65, 1025, 512, "BIAS_F32", ldo=1028),
    _g(1, MATH_X1, 1, 129, 1536, 512, "QKV_ACT", q=512, lo=False),
    # cluster (TMA multicast of the A tile) forms
    _g(1, MATH_X3, 2, 376, 2048, 512, "SILU_ACT"),
    _g(1, MATH_X3, 4, 129, 1024, 512, "GLU_F32"),
    _g(1, MATH_X3, 4, 65, 1536, 512, "QKV_ACT", q=512),
    _g(1, MATH_X3, 2, 127, 3072, 1024, "QKV_ACT", q=1024),
    # the few-row kernel
    _g(2, MATH_X3, 1, 1, 2048, 512, "SILU_ACT"),
    _g(2, MATH_X3, 1, 17, 512, 2048, "RESID_F32", alpha=0.5, inp=True),
    _g(2, MATH_X3, 1, 128, 1025, 512, "BIAS_F32", ldo=1028),
    _g(2, MATH_X3, 1, 64, 1536, 512, "QKV_ACT", q=512),
    _g(2, MATH_X3, 1, 127, 1024, 512, "GLU_F32"),
    _g(2, MATH_X3, 1, 63, 33, 128, "BIAS_F32", ldo=36),
    _g(2, MATH_X1, 1, 65, 2048, 512, "SILU_ACT"),
    _g(2, MATH_X3, 1, 128, 384, 4096, "RELU_ACT"),
    # fp32 CUDA-core kernel (the checker of the others)
    _g(0, MATH_F32, 1, 63, 33, 64, "BIAS_F32", ldo=36),
    _g(0, MATH_F32, 1, 376, 1025, 512, "BIAS_F32", ldo=1028),
    _g(0, MATH_F32, 1, 129, 512, 2048, "RESID_F32", alpha=0.5, inp=True),
    _g(0, MATH_F32, 1, 65, 1024, 512, "RESID_F32", alpha=1.0, inp=True),
    _g(0, MATH_F32, 1, 65, 1024, 512, "SILU_ACT"),
    _g(0, MATH_F32, 1, 376, 1024, 512, "GLU_F32"),
    _g(0, MATH_F32, 1, 1, 640, 128, "RELU_F32"),
    _g(0, MATH_F32, 1, 127, 384, 640, "RELU_ACT"),
    _g(0, MATH_F32, 1, 8064, 384, 128, "BIAS_ACT"),
]


def _gid(c):
    path, mth, cl, M, N, K, k, ldo, alpha, inp, q, lo = c
    kn = [n for n, v in EPI.items() if v == k][0]
    return (f"{['simt', 'wgmma', 'skinny'][path]}-{['x3', 'x1', 'f32'][mth]}-cl{cl}-{kn}-M{M}-N{N}-K{K}-ldo{ldo}"
            + (f"-a{alpha}" + ("-inplace" if inp else "") if k == EPI["RESID_F32"] else "") + ("" if lo else "-nolo"))


@gpu
@pytest.mark.parametrize("case", GEMM_CASES, ids=_gid)
def test_gemm_against_fp64(pkg, case):
    path, mth, cl, M, N, K, kind, ldo, alpha, inp, q, lo = case
    worst = 0.0
    for seed in SEEDS:
        o = run_gemm(pkg, path, mth, cl, M, N, K, kind, ldo, alpha, inp, q, lo, seed)
        worst = max(worst, check_gemm(o, path, mth, M, N, K, kind, ldo, alpha, q, seed))
    report("gemm " + _gid(case), worst)
    assert worst <= 1.0


@gpu
@pytest.mark.parametrize("path", [1, 2])
def test_gemm_bound_rejects_bf16_hi_only_operands(pkg, path):
    """The bf16x3 bound is tight enough to tell the three-product split from operands rounded to bf16 (hi only)."""
    M, N, K, kind = 64, 512, 512, EPI["BIAS_F32"]
    o = run_gemm(pkg, path, MATH_X3, 1, M, N, K, kind, N, seed=5)
    assert check_gemm(o, path, MATH_X3, M, N, K, kind, N, 1.0, 0, 5) <= 1.0
    r = check_gemm(o, path, MATH_X3, M, N, K, kind, N, 1.0, 0, 5, mutate=True)
    report(f"gemm mutation hi-only path {path}", r)
    assert r > 1.0


# ----------------------------------------------------------------------------------------------------------- attention
def ref_attention(qkv, pp, u, v, row_off, n_utt, d, H, tmax, math_mode, kernel, shift=0, drop_u=False, extra_key=False,
                  e_qkv=None, e_pp=None):
    """float64 relative-position attention per utterance and head:
        S[i,j] = ((q_i + u).k_j + (q_i + v).PP[i - j + tmax - 1]) / sqrt(hd) over keys j < T of the same utterance,
        ctx_i = softmax(S[i]) V.
    Bound of ctx[i, c] (per head): the score error of the products is <= eps_s * max_j (|Qu_i|.|k_j| + |Qv_i|.|PP_ij|) / sqrt(hd)
    = D_i (eps_s = 3 * 2^-16 per bf16x3 product on the tensor cores, hd u for the fp32 dot products); a score error D_i
    moves each softmax weight by at most a factor (1 +- 2 D_i), so ctx moves by <= 2 D_i max_j |V_jc|; P.V adds eps_pv
    max_j |V_jc| (bf16x3 P and V: 3 * 2^-16, fp32 sums: T u) and ex2.approx 2^-21.  Times C_ATT = 4.
    Mutations (the bound must reject them): `shift` relative positions, `drop_u`, `extra_key` (key T included).
    e_qkv [rows, 3 d] / e_pp [2 tmax - 1, d]: bounds on the errors of the inputs (a chain of kernels).  They move score i, j
    by <= (|e_q|.|k_j| + |qu|.e_k + |e_q|.|PP_ij| + |qv|.e_PP) / sqrt(hd); with D_i the row's largest such move, ctx moves by
    <= 2 D_i sum_j p_ij |V_jc| + sum_j p_ij e_V,jc, added to the bound as it stands (first order)."""
    hd = d // H
    out = np.zeros((qkv.shape[0], d))
    bound = np.zeros((qkv.shape[0], d))
    q64 = qkv.astype(np.float64)
    for b in range(n_utt):
        r0, r1 = int(row_off[b]), int(row_off[b + 1])
        T = r1 - r0
        if T == 0:
            continue
        Tk = T + 1 if extra_key else T
        i = np.arange(T)[:, None]
        j = np.arange(Tk)[None, :]
        prow = np.clip(i - j + shift + tmax - 1, 0, 2 * tmax - 2)
        for h in range(H):
            cs = slice(h * hd, (h + 1) * hd)
            q = q64[r0:r1, cs]
            k = q64[r0:r0 + Tk, d + h * hd:d + (h + 1) * hd]
            V = q64[r0:r0 + Tk, 2 * d + h * hd:2 * d + (h + 1) * hd]
            qu = q + (0.0 if drop_u else u[cs].astype(np.float64))
            qv = q + v[cs].astype(np.float64)
            PPh = pp[:, cs].astype(np.float64)                       # [2 tmax - 1, hd]; position scores gathered at i - j
            G, Ga = qv @ PPh.T, np.abs(qv) @ np.abs(PPh).T
            s = (qu @ k.T + np.take_along_axis(G, prow, axis=1)) / math.sqrt(hd)
            sa = (np.abs(qu) @ np.abs(k).T + np.take_along_axis(Ga, prow, axis=1)) / math.sqrt(hd)
            m = s.max(axis=1, keepdims=True)
            p = np.exp(s - m)
            p /= p.sum(axis=1, keepdims=True)
            out[r0:r1, cs] = p @ V
            if kernel == 0:
                eps_s, eps_pv = hd * U * 2, T * U * 2
            else:
                eps_s, eps_pv = 3 * 2.0 ** -16 + hd * U, 3 * 2.0 ** -16 + T * U + 2.0 ** -21
            D = eps_s * sa.max(axis=1, keepdims=True)
            vmax = np.abs(V[:T]).max(axis=0, keepdims=True)
            bound[r0:r1, cs] = 4.0 * (2 * D + eps_pv) * vmax
            if e_qkv is not None:
                eq = e_qkv[r0:r1, cs]
                ek = e_qkv[r0:r0 + Tk, d + h * hd:d + (h + 1) * hd]
                ev = e_qkv[r0:r0 + Tk, 2 * d + h * hd:2 * d + (h + 1) * hd]
                gq = eq @ np.abs(PPh).T
                if e_pp is not None:
                    gq = gq + np.abs(qv) @ e_pp[:, cs].T
                Din = (eq @ np.abs(k).T + np.abs(qu) @ ek.T + np.take_along_axis(gq, prow, axis=1)).max(axis=1, keepdims=True)
                bound[r0:r1, cs] += 2 * Din / math.sqrt(hd) * (p @ np.abs(V)) + p @ ev
    return out, bound


def attn_inputs(rng, rows_total, d, tmax, regime="plain", sentinel_rows=()):
    qkv = rng.uniform(-1, 1, (rows_total, 3 * d)).astype(np.float32)
    pp = rng.uniform(-1, 1, (2 * tmax - 1, d)).astype(np.float32)
    u = (0.3 * rng.uniform(-1, 1, d)).astype(np.float32)
    v = (0.3 * rng.uniform(-1, 1, d)).astype(np.float32)
    if regime == "peaky":
        qkv[:, :d] *= 3
    elif regime == "flat":
        qkv[:, d:2 * d] = qkv[0, d:2 * d]
    elif regime == "content":
        pp[:] = 0
    elif regime == "position":
        qkv[:, d:2 * d] = 0
    qkv[list(sentinel_rows)] = np.nan                     # rows outside every utterance: must never be read
    return qkv, pp, u, v


def run_attention(pkg, kernel, math_mode, row_off, rows_total, d, H, tmax, qkv, pp, u, v):
    L = pkg.load_library()
    ro = np.ascontiguousarray(row_off, np.int32)
    f32 = math_mode == MATH_F32
    of = nan((rows_total, d)) if f32 else None
    oh = None if f32 else nan((rows_total, d))
    ol = nan((rows_total, d)) if math_mode == MATH_X3 else None
    gb = C.c_int64(-1)
    st = L.pk_kernel_attention(0, kernel, math_mode, len(ro) - 1, i32p(ro), rows_total, d, H, tmax, f32p(qkv), f32p(pp), f32p(u), f32p(v),
                               f32p(of), f32p(oh), f32p(ol), C.byref(gb))
    assert st == 0, f"pk_kernel_attention -> {st}"
    assert gb.value == 0
    return of, oh, ol


def check_attention(out, row_off, rows_total, ref, bd):
    of, oh, ol = out
    inside = np.zeros(rows_total, bool)
    for b in range(len(row_off) - 1):
        inside[row_off[b]:row_off[b + 1]] = True
    main = of if of is not None else oh
    assert np.all(np.isfinite(main[inside])), "a ctx element was not written"
    assert np.all(np.isnan(main[~inside])), "a row outside the batch was written"
    if ol is not None:
        assert np.all(np.isfinite(ol[inside])) and np.all(np.isnan(ol[~inside]))
    if of is not None:
        return ratio(of[inside], ref[inside], bd[inside])
    return check_planes(oh[inside], None if ol is None else ol[inside], ref[inside], bd[inside])


ATTN_CFGS = {  # (d, heads): T values
    (128, 2): [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 192, 193, 376],
    (512, 8): [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 192, 193, 376],
    (1024, 8): [1, 63, 64, 65, 113, 128, 129, 376],
}
ATTN_KERNELS = [(0, MATH_F32), (1, MATH_X3), (1, MATH_X1)]


@gpu
@pytest.mark.parametrize("kernel,math_mode", ATTN_KERNELS, ids=["fp32", "mma-x3", "mma-x1"])
@pytest.mark.parametrize("cfg", list(ATTN_CFGS), ids=lambda c: f"d{c[0]}h{c[1]}")
def test_attention_against_fp64(pkg, kernel, math_mode, cfg):
    """Ragged batches of every length (tmax = the longest, and larger), then each length alone at a non-zero row offset
    inside NaN sentinel rows, then the score regimes on a ragged batch."""
    d, H = cfg
    lens = ATTN_CFGS[cfg]
    worst = 0.0
    for seed in SEEDS:
        rng = np.random.default_rng(seed * 101 + d + kernel)
        order = list(rng.permutation(lens))
        off = np.concatenate([[0], np.cumsum(order)]).astype(np.int32)
        M = int(off[-1])
        for tmax in (max(lens), max(lens) + 37):
            qkv, pp, u, v = attn_inputs(rng, M, d, tmax)
            ref, bd = ref_attention(qkv, pp, u, v, off, len(order), d, H, tmax, math_mode, kernel)
            worst = max(worst, check_attention(run_attention(pkg, kernel, math_mode, off, M, d, H, tmax, qkv, pp, u, v), off, M, ref, bd))
    rng = np.random.default_rng(7 + kernel)
    for T in lens:                                                    # alone, at row 5 of T + 11 rows
        off = np.array([5, 5 + T], np.int32)
        rows = T + 11
        tmax = max(lens)
        qkv, pp, u, v = attn_inputs(rng, rows, d, tmax, sentinel_rows=[*range(5), *range(5 + T, rows)])
        ref, bd = ref_attention(qkv, pp, u, v, off, 1, d, H, tmax, math_mode, kernel)
        worst = max(worst, check_attention(run_attention(pkg, kernel, math_mode, off, rows, d, H, tmax, qkv, pp, u, v), off, rows, ref, bd))
    for regime in ("peaky", "flat", "content", "position"):
        sub = lens[-4:]
        off = np.concatenate([[0], np.cumsum(sub)]).astype(np.int32)
        M = int(off[-1])
        qkv, pp, u, v = attn_inputs(rng, M, d, max(sub), regime)
        ref, bd = ref_attention(qkv, pp, u, v, off, len(sub), d, H, max(sub), math_mode, kernel)
        worst = max(worst, check_attention(run_attention(pkg, kernel, math_mode, off, M, d, H, max(sub), qkv, pp, u, v), off, M, ref, bd))
    report(f"attention kernel {kernel} math {math_mode} d {d} heads {H}", worst)
    assert worst <= 1.0


@gpu
@pytest.mark.parametrize("kernel,math_mode", [(0, MATH_F32), (1, MATH_X3)], ids=["fp32", "mma-x3"])
def test_attention_bound_rejects_mutations(pkg, kernel, math_mode):
    d, H = 512, 8
    lens = [65, 17, 128, 40]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    M, tmax = int(off[-1]), 128
    rng = np.random.default_rng(11)
    qkv, pp, u, v = attn_inputs(rng, M, d, tmax)
    out = run_attention(pkg, kernel, math_mode, off, M, d, H, tmax, qkv, pp, u, v)
    ref, bd = ref_attention(qkv, pp, u, v, off, len(lens), d, H, tmax, math_mode, kernel)
    assert check_attention(out, off, M, ref, bd) <= 1.0
    for name, kw, n in (("position off by one", dict(shift=1), len(lens)), ("pos_bias_u dropped", dict(drop_u=True), len(lens)),
                        ("one key past T", dict(extra_key=True), len(lens) - 1)):
        mref, _ = ref_attention(qkv, pp, u, v, off, n, d, H, tmax, math_mode, kernel, **kw)
        rows = slice(0, int(off[n]))
        r = check_attention(tuple(None if a is None else a[rows] for a in out), off[:n + 1], int(off[n]), mref[rows], bd[rows])
        report(f"attention kernel {kernel} mutation {name}", r)
        assert r > 1.0, name


def test_attention_hook_rejects_unknown_kernel(pkg):
    """kernel is 0 (fp32) or 1 (mma.sync); any other value is refused with PK_ERR_INVALID before the device is touched."""
    L = pkg.load_library()
    d, H, tmax = 512, 8, 4
    ro = np.array([0, tmax], np.int32)
    qkv, pp, u, v = np.zeros((tmax, 3 * d), np.float32), np.zeros((2 * tmax - 1, d), np.float32), np.zeros(d, np.float32), np.zeros(d, np.float32)
    oh, ol = np.zeros((tmax, d), np.float32), np.zeros((tmax, d), np.float32)
    for kernel in (2, -1):
        st = L.pk_kernel_attention(0, kernel, MATH_X3, 1, i32p(ro), tmax, d, H, tmax, f32p(qkv), f32p(pp), f32p(u), f32p(v),
                                   f32p(None), f32p(oh), f32p(ol), C.byref(C.c_int64(-1)))
        assert st == 1, (kernel, st)


# ----------------------------------------------------------------------------------------------------------- LayerNorm
def ref_layernorm(x, w, b, e_in=None, unbiased=False):
    """float64 LayerNorm (biased variance, eps = 1e-5 inside the sqrt) -> (y, bound).
    The kernel: one warp per row, lane sums of 4 d/128 elements then a 5-level butterfly, for the mean and then for the
    centred second moment; n = 4 d/128 + 5 rounded adds.  |mean error| <= dm = n u mean|x| (+ the input error), so every
    centred value is off by <= E = dm + max e_in; the variance by <= 2 E mean|c| + E^2 + n u var (relative to var:
    r_v), rsqrt by r_v / 2 + 2 u.  |y error| <= |w| (E / s + |c| / s (r_v / 2 + 2 u)) + 4 u (|y| + |b|), times C_LN = 2."""
    x64 = x.astype(np.float64)
    d = x.shape[1]
    mu = x64.mean(axis=1, keepdims=True)
    c = x64 - mu
    var = (c * c).sum(axis=1, keepdims=True) / (d - 1 if unbiased else d)
    s = np.sqrt(var + 1e-5)
    y = c / s * w.astype(np.float64) + b.astype(np.float64)
    n = 4 * d // 128 + 5
    ein = np.zeros_like(x64) if e_in is None else e_in
    E = n * U * np.abs(x64).mean(axis=1, keepdims=True) + ein.max(axis=1, keepdims=True)
    rv = (2 * E * np.abs(c).mean(axis=1, keepdims=True) + E * E + n * U * var) / (var + 1e-5)
    bound = np.abs(w) * (E / s + np.abs(c) / s * (rv / 2 + 2 * U)) + 4 * U * (np.abs(y) + np.abs(b))
    return y, 2.0 * bound


def ln_rows(rng, M, d, kind):
    x = rng.normal(0, 1, (M, d)) * 10.0 ** rng.uniform(-2, 2, (M, 1))
    if kind == "offset":            # large common offset: mean 1e3, std 1e-2
        x[::2] = 1e3 + 1e-2 * rng.normal(0, 1, (len(x[::2]), d))
    elif kind == "constant":        # variance 0
        x[::2] = rng.uniform(-3, 3, (len(x[::2]), 1))
    return x.astype(np.float32)


def run_layernorm(pkg, x, w1, b1, w2, b2, want_f32, planes):
    L = pkg.load_library()
    M, d = x.shape
    y1 = nan((M, d)) if want_f32 else None
    af = nan((M, d)) if planes == 3 else None
    hi = nan((M, d)) if planes in (1, 2) else None
    lo = nan((M, d)) if planes == 2 else None
    gb = C.c_int64(-1)
    st = L.pk_kernel_layernorm(0, M, d, f32p(x), f32p(w1), f32p(b1), f32p(w2), f32p(b2), int(want_f32), planes, f32p(y1), f32p(af),
                               f32p(hi), f32p(lo), C.byref(gb))
    assert st == 0, f"pk_kernel_layernorm -> {st}"
    assert gb.value == 0
    for a in (y1, af, hi, lo):
        assert a is None or np.all(np.isfinite(a)), "a LayerNorm output element was not written"
    return y1, af, hi, lo


@gpu
@pytest.mark.parametrize("d", [128, 512, 1024])
@pytest.mark.parametrize("M", [1, 7, 8, 9, 8064])
@pytest.mark.parametrize("kind", ["plain", "offset", "constant"])
def test_layernorm_against_fp64(pkg, d, M, kind):
    worst = 0.0
    for seed in SEEDS:
        rng = np.random.default_rng(seed * 13 + d + M)
        x = ln_rows(rng, M, d, kind)
        w1, b1, w2, b2 = (rng.uniform(0.5, 1.5, d).astype(np.float32), rng.uniform(-0.3, 0.3, d).astype(np.float32),
                          rng.uniform(0.5, 1.5, d).astype(np.float32), rng.uniform(-0.3, 0.3, d).astype(np.float32))
        rows = sample_rows(M, seed)
        y1r, b1r = ref_layernorm(x[rows], w1, b1)
        # single LayerNorm: hi | lo operand planes (bf16x3), hi only (bf16x1), fp32 operand (fp32 math)
        for planes in (1, 2, 3):
            _, af, hi, lo = run_layernorm(pkg, x, w1, b1, None, None, False, planes)
            worst = max(worst, ratio(af[rows], y1r, b1r) if planes == 3 else check_planes(hi[rows], None if lo is None else lo[rows], y1r, b1r))
        # LN1 in place over x and its planes (the block's attention / conv norms)
        y1, _, hi, lo = run_layernorm(pkg, x, w1, b1, None, None, True, 2)
        worst = max(worst, ratio(y1[rows], y1r, b1r), check_planes(hi[rows], lo[rows], y1r, b1r))
        # chained: y1 = LN1(x) in place, planes = LN2(y1) (final_norm_ + the next block's ffn1_.norm_)
        y1, _, hi, lo = run_layernorm(pkg, x, w1, b1, w2, b2, True, 2)
        y2r, b2r = ref_layernorm(y1r, w2, b2, e_in=b1r)
        worst = max(worst, ratio(y1[rows], y1r, b1r), check_planes(hi[rows], lo[rows], y2r, b2r))
    report(f"layernorm d {d} M {M} {kind}", worst)
    assert worst <= 1.0


@gpu
def test_layernorm_bound_rejects_unbiased_variance(pkg):
    rng = np.random.default_rng(3)
    d, M = 128, 64
    x = ln_rows(rng, M, d, "plain")
    w, b = rng.uniform(0.5, 1.5, d).astype(np.float32), rng.uniform(-0.3, 0.3, d).astype(np.float32)
    _, af, _, _ = run_layernorm(pkg, x, w, b, None, None, False, 3)
    y, bd = ref_layernorm(x, w, b)
    assert ratio(af, y, bd) <= 1.0
    ym, _ = ref_layernorm(x, w, b, unbiased=True)
    r = ratio(af, ym, bd)
    report("layernorm mutation unbiased variance", r)
    assert r > 1.0


# ----------------------------------------------------------------------------------------------------------- dwconv
def ref_dwconv(g, w_tap, bias, row_off, neighbour_pad=False, e_in=None, w_rel=0.0):
    """float64 depthwise conv (k taps, zero padding inside each utterance) + folded bias, then SiLU -> (y, bound).
    The kernel: fma chain over the k taps from the bias: |err| <= (k + 1) u (sum |w g| + |b|); SiLU with expf is
    1.1-Lipschitz plus 8 u |y| (expf, the division, the product).  Times C_DW = 2.  neighbour_pad (mutation): taps outside the utterance read the
    neighbouring rows instead of zeros.  A chain of kernels adds 1.1 sum_taps |w| e_in (input error bound e_in) and
    1.1 w_rel (sum |w g| + |b|) (weights and bias off by w_rel relative, e.g. a rounded BatchNorm fold)."""
    ks, d = w_tap.shape
    half = ks // 2
    g64 = g.astype(np.float64)
    y = np.zeros_like(g64)
    bd = np.zeros_like(g64)
    for b in range(len(row_off) - 1):
        r0, r1 = int(row_off[b]), int(row_off[b + 1])
        T = r1 - r0
        acc = np.tile(bias.astype(np.float64), (T, 1))
        aab = np.tile(np.abs(bias.astype(np.float64)), (T, 1))
        prop = np.zeros((T, d))
        for j in range(ks):
            src = np.arange(T) + j - half
            ok = (src >= 0) & (src < T)
            if neighbour_pad:
                ok = (r0 + src >= 0) & (r0 + src < g.shape[0])
            tap = np.zeros((T, d))
            tap[ok] = g64[r0 + src[ok]]
            acc += w_tap[j].astype(np.float64) * tap
            aab += np.abs(w_tap[j].astype(np.float64) * tap)
            if e_in is not None:
                etap = np.zeros((T, d))
                etap[ok] = e_in[r0 + src[ok]]
                prop += np.abs(w_tap[j].astype(np.float64)) * etap
        yy = acc * sig64(acc)
        y[r0:r1] = yy
        bd[r0:r1] = 2.0 * (1.1 * (ks + 1) * U * aab + 8 * U * np.abs(yy)) + 1.1 * (prop + w_rel * aab)
    return y, bd


def run_dwconv(pkg, math_mode, row_off, rows_total, g, w_tap, bias):
    L = pkg.load_library()
    ro = np.ascontiguousarray(row_off, np.int32)
    d = g.shape[1]
    f32 = math_mode == MATH_F32
    of = nan((rows_total, d)) if f32 else None
    hi = None if f32 else nan((rows_total, d))
    lo = nan((rows_total, d)) if math_mode == MATH_X3 else None
    gb = C.c_int64(-1)
    st = L.pk_kernel_dwconv(0, math_mode, len(ro) - 1, i32p(ro), rows_total, d, w_tap.shape[0], f32p(g), f32p(w_tap), f32p(bias), f32p(of),
                            f32p(hi), f32p(lo), C.byref(gb))
    assert st == 0, f"pk_kernel_dwconv -> {st}"
    assert gb.value == 0
    return of, hi, lo


def check_dwconv(out, row_off, rows_total, y, bd):
    of, hi, lo = out
    inside = np.zeros(rows_total, bool)
    for b in range(len(row_off) - 1):
        inside[row_off[b]:row_off[b + 1]] = True
    main = of if of is not None else hi
    assert np.all(np.isfinite(main[inside])) and np.all(np.isnan(main[~inside]))
    if lo is not None:
        assert np.all(np.isfinite(lo[inside])) and np.all(np.isnan(lo[~inside]))
    if of is not None:
        return ratio(of[inside], y[inside], bd[inside])
    return check_planes(hi[inside], None if lo is None else lo[inside], y[inside], bd[inside])


DW_T = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 63, 64, 65, 376]


@gpu
@pytest.mark.parametrize("d", [128, 512, 1024])
@pytest.mark.parametrize("math_mode", [MATH_X3, MATH_X1, MATH_F32], ids=["x3", "x1", "f32"])
def test_dwconv_against_fp64(pkg, d, math_mode):
    worst = 0.0
    for seed in SEEDS:
        rng = np.random.default_rng(seed * 17 + d + math_mode)
        w = rng.uniform(-0.5, 0.5, (9, d)).astype(np.float32)
        b = rng.uniform(-0.5, 0.5, d).astype(np.float32)
        order = list(rng.permutation(DW_T))                 # ragged batch: every tap at every utterance edge
        off = np.concatenate([[0], np.cumsum(order)]).astype(np.int32)
        M = int(off[-1])
        g = (rng.normal(0, 1, (M, d)) * 10.0 ** rng.uniform(-2, 2, (M, 1))).astype(np.float32)
        y, bd = ref_dwconv(g, w, b, off)
        worst = max(worst, check_dwconv(run_dwconv(pkg, math_mode, off, M, g, w, b), off, M, y, bd))
    rng = np.random.default_rng(99 + d)
    for T in DW_T:                                          # alone at row 3 of T + 8 rows; the rest are NaN and must not be read
        rows = T + 8
        off = np.array([3, 3 + T], np.int32)
        g = nan((rows, d))
        g[3:3 + T] = rng.normal(0, 1, (T, d))
        y, bd = ref_dwconv(g, w, b, off)
        worst = max(worst, check_dwconv(run_dwconv(pkg, math_mode, off, rows, g, w, b), off, rows, y, bd))
    report(f"dwconv d {d} math {math_mode}", worst)
    assert worst <= 1.0


@gpu
def test_dwconv_bound_rejects_neighbour_padding(pkg):
    rng = np.random.default_rng(4)
    d = 128
    w = rng.uniform(-0.5, 0.5, (9, d)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, d).astype(np.float32)
    off = np.array([0, 10, 75, 80], np.int32)
    g = rng.normal(0, 1, (80, d)).astype(np.float32)
    out = run_dwconv(pkg, MATH_F32, off, 80, g, w, b)
    y, bd = ref_dwconv(g, w, b, off)
    assert check_dwconv(out, off, 80, y, bd) <= 1.0
    ym, _ = ref_dwconv(g, w, b, off, neighbour_pad=True)
    r = check_dwconv(out, off, 80, ym, bd)
    report("dwconv mutation neighbour padding", r)
    assert r > 1.0


# ----------------------------------------------------------------------------------------------------------- CTC argmax
def ref_ctc(logits):
    """first maximum (the reference's strict '>' scan from index 0), exp(max log-prob), log-softmax, in float64 ->
    (best, conf, logprobs, conf bound, logprobs bound).  The kernel sums V expf terms per row (32 lanes + butterfly):
    relative error of the sum <= (V / 32 + 5 + 2 V) u; |logprob error| <= u |l - max| + that + u |lse|.  Times C_CTC = 4."""
    l64 = logits.astype(np.float64)
    V = logits.shape[1]
    best = np.array([first_argmax64(r) for r in l64])
    mx = l64.max(axis=1, keepdims=True)
    s = np.exp(l64 - mx).sum(axis=1, keepdims=True)
    lse = np.log(s)
    lp = l64 - mx - lse
    rel = (V / 32 + 5 + 2 * V) * U + 4 * U
    conf = 1.0 / s[:, 0]
    return best, conf, lp, 4.0 * rel * conf, 4.0 * (U * np.abs(l64 - mx) + rel + U * np.abs(lse))


def first_argmax64(row):
    best, bv = 0, row[0]
    for i in range(1, len(row)):
        if row[i] > bv:
            best, bv = i, row[i]
    return best


def run_ctc(pkg, logits_padded, V, want_lp=True):
    L = pkg.load_library()
    M, ld = logits_padded.shape
    best = np.full(M, -7, np.int32)
    conf = nan(M)
    lp = nan((M, V)) if want_lp else None
    gb = C.c_int64(-1)
    st = L.pk_kernel_ctc_argmax(0, M, V, ld, f32p(logits_padded), i32p(best), f32p(conf), f32p(lp), C.byref(gb))
    assert st == 0, f"pk_kernel_ctc_argmax -> {st}"
    assert gb.value == 0
    return best, conf, lp


@gpu
@pytest.mark.parametrize("V", [33, 1025])
def test_ctc_argmax_against_fp64(pkg, V):
    ld = (V + 3) & ~3
    worst = 0.0
    for seed in SEEDS:
        rng = np.random.default_rng(seed * 5 + V)
        M = 300
        x = rng.normal(0, 3, (M, V)).astype(np.float32)
        # exact ties spread across lanes (the first index must win), the maximum at the last column, large dynamic range
        for r in range(0, 40):
            cols = np.sort(rng.choice(V, size=min(V, 2 + r % 5), replace=False))
            x[r, cols] = x[r].max() + 1.0
        x[40:60, V - 1] = x[40:60].max(axis=1) + 0.5
        x[60:80] = (rng.normal(0, 1, (20, V)) * 10.0 ** rng.uniform(0, 4, (20, 1))).astype(np.float32)
        x[80, :] = 2.5                                        # every column tied
        xp = nan((M, ld))                                     # the padding columns are NaN: they must never be read
        xp[:, :V] = x
        best, conf, lp = run_ctc(pkg, xp, V)
        rb, rc, rlp, bc, blp = ref_ctc(x)
        assert np.array_equal(best, rb)
        worst = max(worst, ratio(conf, rc, bc), ratio(lp, rlp, blp))
    report(f"ctc argmax V {V}", worst)
    assert worst <= 1.0


@gpu
def test_ctc_argmax_row_without_a_finite_maximum(pkg, O):
    """A row of -inf: the reference's scan (and the oracle's first_argmax) keep index 0; the kernel must not return an
    out-of-vocabulary index for it."""
    V, ld = 33, 36
    x = np.random.default_rng(0).normal(0, 1, (4, ld)).astype(np.float32)
    x[1, :] = -np.inf
    best, _, _ = run_ctc(pkg, x, V, want_lp=False)
    assert best[1] == O.first_argmax(x[1, :V]) == 0
    assert np.array_equal(best[[0, 2, 3]], [first_argmax64(x[r, :V]) for r in (0, 2, 3)])


# ----------------------------------------------------------------------------------------------------------- the references, pinned (CPU)
def test_ref_gemm_matches_oracle_linear(O):
    rng = np.random.default_rng(0)
    A, W, b = (rng.normal(0, 1, s).astype(np.float32) for s in ((9, 24), (13, 24), (13,)))
    y, bd = ref_gemm(A, W, b, None, EPI["BIAS_F32"], 1.0, MATH_F32)
    assert np.allclose(O.linear(A, W, b), y, rtol=1e-5, atol=1e-5)
    y, _ = ref_gemm(A, W, b, None, EPI["SILU_ACT"], 1.0, MATH_F32)
    assert np.allclose(O.silu(O.linear(A, W, b)), y, rtol=1e-5, atol=1e-5)
    Wg = np.empty_like(W[:12])                                  # interleaved GLU columns (a0, b0, a1, b1, ...)
    Wg[0::2], Wg[1::2] = W[:6], W[6:12]
    y, _ = ref_gemm(A, Wg, None, None, EPI["GLU_F32"], 1.0, MATH_F32)
    h = O.linear(A, W[:12])
    assert np.allclose(h[:, :6] * O.sigmoid(h[:, 6:]), y, rtol=1e-5, atol=1e-5)
    r = rng.normal(0, 1, (9, 13)).astype(np.float32)
    y, _ = ref_gemm(A, W, b, r, EPI["RESID_F32"], 0.5, MATH_F32)
    assert np.allclose(r + 0.5 * O.linear(A, W, b), y, rtol=1e-5, atol=1e-5)


def test_ref_layernorm_matches_oracle(O):
    rng = np.random.default_rng(1)
    x = rng.normal(0, 2, (6, 128)).astype(np.float32)
    w, b = rng.uniform(0.5, 1.5, 128).astype(np.float32), rng.normal(0, 0.1, 128).astype(np.float32)
    y, _ = ref_layernorm(x, w, b)
    assert np.allclose(O.layer_norm(x, w, b), y, rtol=1e-5, atol=1e-5)
    y2, _ = ref_layernorm(y, w, b)
    assert np.allclose(O.layer_norm(O.layer_norm(x, w, b), w, b), y2, rtol=1e-4, atol=1e-4)


def test_ref_attention_matches_oracle_rel_shift(O):
    """The i - j indexing of the position table equals the oracle's rel_shift of (q + v) P^T, with the oracle's table
    (row r <-> relative position T - 1 - r) cut from ours (row p + tmax - 1 <-> position p)."""
    rng = np.random.default_rng(2)
    d, H, T, tmax = 32, 2, 7, 9
    hd = d // H
    qkv, pp, u, v = attn_inputs(rng, T, d, tmax)
    ours, _ = ref_attention(qkv, pp, u, v, np.array([0, T]), 1, d, H, tmax, MATH_F32, 0)
    q = qkv[:, :d].reshape(T, H, hd).transpose(1, 0, 2)
    k = qkv[:, d:2 * d].reshape(T, H, hd).transpose(1, 0, 2)
    vv = qkv[:, 2 * d:].reshape(T, H, hd).transpose(1, 0, 2)
    opp = pp[[T - 1 - r + tmax - 1 for r in range(2 * T - 1)]].reshape(2 * T - 1, H, hd).transpose(1, 0, 2)
    ac = (q + u.reshape(H, 1, hd)) @ k.transpose(0, 2, 1)
    bd = O.rel_shift((q + v.reshape(H, 1, hd)) @ opp.transpose(0, 2, 1))
    a = O.softmax(((ac + bd) * np.float32(1 / math.sqrt(hd))).astype(np.float32), axis=-1)
    want = (a @ vv).transpose(1, 0, 2).reshape(T, d)
    assert np.allclose(want, ours, rtol=1e-4, atol=1e-5)


def test_ref_dwconv_matches_oracle(O):
    rng = np.random.default_rng(3)
    d, T = 8, 12
    g = rng.normal(0, 1, (T, d)).astype(np.float32)
    w = rng.normal(0, 0.5, (9, d)).astype(np.float32)
    b = rng.normal(0, 0.5, d).astype(np.float32)
    y, _ = ref_dwconv(g, w, b, np.array([0, T]))
    want = O.silu(O.depthwise_conv1d(g.T, w.T[:, None, :], b, 4)).T
    assert np.allclose(want, y, rtol=1e-5, atol=1e-6)


def test_ref_ctc_matches_oracle(O):
    rng = np.random.default_rng(4)
    x = rng.normal(0, 3, (20, 33)).astype(np.float32)
    x[3, [4, 9, 31]] = 50.0
    x[5, :] = 1.0
    x[6, :] = -np.inf
    best, conf, lp, _, _ = ref_ctc(x[:6])
    assert [O.first_argmax(r) for r in x[:6]] == list(best)
    assert best[3] == 4 and best[5] == 0
    assert O.first_argmax(x[6]) == first_argmax64(x[6]) == 0        # no finite maximum: index 0
    assert np.allclose(O.log_softmax(x[:6]), lp, atol=1e-5)
    assert np.allclose(np.exp(O.log_softmax(x[:6]).max(axis=1)), conf, rtol=1e-5)


def test_bf16_split_helpers():
    x = np.array([1.0, 1.00390625, 1.005859375, -3.14159, 1e-30, 65504.0], np.float32)
    hi, lo = split(x)
    assert np.all(bf16_rn(hi) == hi) and np.all(bf16_rn(lo) == lo)
    assert hi[1] == 1.0 and hi[2] == np.float32(1.0078125)          # ties to even, then up
    assert np.all(np.abs(hi.astype(np.float64) + lo - x) <= 2.0 ** -16 * np.abs(x))
