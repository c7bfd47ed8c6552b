"""The streaming encoder kernels (csrc/stream.cu) against float64 math, element by element, through pk_kernel_stream_attention
and pk_kernel_stream_dwconv.  Each hook runs the launcher as pk_stream_step does for one layer, on host fp32 inputs (rings,
cache lengths, ring starts, active-stream list, row offsets, position table) and returns the outputs and the updated state
between 0xFF guard bands (NaN in fp32 and bf16), plus the count of changed guard bytes.

Bounds (u = 2^-24; both kernels are fp32 CUDA-core code; sums are sequential fma chains):
  attention  keys = [cl ring rows, oldest first | the C chunk rows], kv = cl + C.  A score is two hd-term dot products over
             sqrt(hd): |err| <= 2 hd u S_a, S_a = (|q + u| . |k| + |q + v| . |pp|) / sqrt(hd).  A score error e moves
             every softmax weight by at most 2 e relative (both the exponent and the normaliser), expf adds 2 u, the
             sequential normaliser kv u, and P.V another kv u relative to max |V| (weights sum to 1):
             |err| <= 4 (2 * 2 hd u max_j S_a + (2 kv + 4) u) max |V|  -- the factor 4 covers the second-order terms.
  ring       the chunk's K / V rows are copied: the updated rings must be bit-exact.
  dwconv     ks-term fma chain plus the bias: |err_pre| <= (ks + 2) u (sum_j |w_j x_j| + |b|); SiLU is 1.1-Lipschitz and
             its expf / division add 4 u |y|: |err| <= 4 (1.1 err_pre + 4 u |y|).  The conv cache is bit-exact.
  planes     bf16 hi + lo stands for the fp32 value within 2^-16 |y| (added to the bound).
The position table is the launcher's: pp holds the projected table of 2 tmax - 1 rows with relative position p at row
p + tmax - 1, and key j of kv keys has p = kv - L - C - j (the reference's un-shifted right-most columns); the engine-level
tests (tests/test_nemotron.py, test_gpu_parity.py) pin that convention against the compiled reference end to end.
Sensitivity: references mutated the way a plausible bug would (an off-by-one position row, the ring read without
ring_start, pos_bias_v dropped, the conv cache ignored) must be rejected by the same checks.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest

gpu = pytest.mark.gpu
U = 2.0 ** -24
MATH_X3, MATH_F32 = 0, 2


def _f(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def _i(a):
    return np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int32))


def report(what, r):
    print(f"{what}: max error / bound = {r:.3g}")


def ratio(got, ref, bound):
    e = np.abs(got.astype(np.float64) - ref) / np.maximum(bound, 1e-300)
    e = np.where(np.isnan(e), np.inf, e)
    return float(e.max()) if e.size else 0.0


# ------------------------------------------------------------------------------------------------------------ references
def ref_stream_attention(qkv, pp, pu, pv, kc, vc, act, row_off, cache_len, ring_start, L, d, H, tmax,
                         pos_shift=0, ignore_ring_start=False, drop_v=False):
    """-> (ctx [rows][d], bound [rows][d], kc_new, vc_new) in float64 / exact fp32 for the rings."""
    hd = d // H
    rows = qkv.shape[0]
    out, bound = np.full((rows, d), np.nan), np.zeros((rows, d))
    kc_new, vc_new = kc.copy(), vc.copy()
    q64 = qkv.astype(np.float64)
    for a, s in enumerate(act):
        r0, r1 = int(row_off[a]), int(row_off[a + 1])
        Cn, cl, rs = r1 - r0, int(cache_len[s]), int(ring_start[s])
        slots = [(j if ignore_ring_start else (rs + j) % L) for j in range(cl)]
        K = np.concatenate([kc[s, slots].astype(np.float64), q64[r0:r1, d:2 * d]])
        V = np.concatenate([vc[s, slots].astype(np.float64), q64[r0:r1, 2 * d:]])
        kv = cl + Cn
        prow = np.clip(kv - L - Cn - np.arange(kv) + tmax - 1 + pos_shift, 0, 2 * tmax - 2)
        for h in range(H):
            cs = slice(h * hd, (h + 1) * hd)
            q = q64[r0:r1, cs]
            qu, qv = q + pu[cs], q + (0.0 if drop_v else pv[cs].astype(np.float64))
            Pp = pp[prow][:, cs].astype(np.float64)
            sc = (qu @ K[:, cs].T + qv @ Pp.T) / math.sqrt(hd)
            sa = (np.abs(qu) @ np.abs(K[:, cs]).T + np.abs(qv) @ np.abs(Pp).T) / math.sqrt(hd)
            p = np.exp(sc - sc.max(axis=1, keepdims=True))
            p /= p.sum(axis=1, keepdims=True)
            out[r0:r1, cs] = p @ V[:, cs]
            bd = 4.0 * (2 * 2 * hd * U * sa.max(axis=1, keepdims=True) + (2 * kv + 4) * U) * np.abs(V[:, cs]).max()
            bound[r0:r1, cs] = bd
        first = max(Cn - L, 0)
        for r in range(first, Cn):
            slot = (rs + cl + r) % L
            kc_new[s, slot] = qkv[r0 + r, d:2 * d]
            vc_new[s, slot] = qkv[r0 + r, 2 * d:]
    return out, bound, kc_new, vc_new


def ref_stream_dwconv(glu, w, b, cache, act, row_off, ks, ignore_cache=False):
    rows, d = glu.shape
    out, bound = np.full((rows, d), np.nan), np.zeros((rows, d))
    cache_new = cache.copy()
    for a, s in enumerate(act):
        r0, r1 = int(row_off[a]), int(row_off[a + 1])
        left = np.zeros((ks - 1, d)) if ignore_cache else cache[s].astype(np.float64)
        seq = np.concatenate([left, glu[r0:r1].astype(np.float64)])
        for t in range(r1 - r0):
            terms = w.T.astype(np.float64) * seq[t:t + ks]          # [ks][d]
            pre = terms.sum(axis=0) + b
            y = pre / (1.0 + np.exp(-pre))
            out[r0 + t] = y
            bound[r0 + t] = 4.0 * (1.1 * (ks + 2) * U * (np.abs(terms).sum(axis=0) + np.abs(b)) + 4 * U * np.abs(y))
        cache_new[s] = seq[seq.shape[0] - (ks - 1):].astype(np.float32)
    return out, bound, cache_new


# ------------------------------------------------------------------------------------------------------------ hooks
def _outs(math_mode, rows, d):
    f32 = math_mode == MATH_F32
    return (np.full((rows, d), np.nan, np.float32) if f32 else None, None if f32 else np.full((rows, d), np.nan, np.float32),
            np.full((rows, d), np.nan, np.float32) if math_mode == MATH_X3 else None)


def run_stream_attention(pkg, math_mode, case):
    L_ = pkg.load_library()
    c = case
    rows, d = c["qkv"].shape[0], c["d"]
    of, oh, ol = _outs(math_mode, rows, d)
    kco, vco = np.full_like(c["kc"], np.nan), np.full_like(c["vc"], np.nan)
    gb = C.c_int64(-1)
    st = L_.pk_kernel_stream_attention(0, math_mode, c["kc"].shape[0], len(c["act"]), _i(c["act"]), _i(c["off"]), rows, _i(c["cl"]),
                                       _i(c["rs"]), c["L"], d, c["H"], c["tmax"], _f(c["qkv"]), _f(c["pp"]), _f(c["u"]), _f(c["v"]),
                                       _f(c["kc"]), _f(c["vc"]), _f(of), _f(oh), _f(ol), _f(kco), _f(vco), C.byref(gb))
    assert st == 0, f"pk_kernel_stream_attention -> {st}"
    return dict(f32=of, hi=oh, lo=ol, kc=kco, vc=vco, guard_bad=gb.value)


def run_stream_dwconv(pkg, math_mode, case):
    L_ = pkg.load_library()
    c = case
    rows, d = c["glu"].shape
    of, oh, ol = _outs(math_mode, rows, d)
    co = np.full_like(c["cache"], np.nan)
    gb = C.c_int64(-1)
    st = L_.pk_kernel_stream_dwconv(0, math_mode, c["cache"].shape[0], len(c["act"]), _i(c["act"]), _i(c["off"]), rows, d, c["ks"],
                                    _f(c["glu"]), _f(c["w"]), _f(c["b"]), _f(c["cache"]), _f(of), _f(oh), _f(ol), _f(co), C.byref(gb))
    assert st == 0, f"pk_kernel_stream_dwconv -> {st}"
    return dict(f32=of, hi=oh, lo=ol, cache=co, guard_bad=gb.value)


def check_out(got, ref, bound, inside):
    """Written set exact (rows of active streams finite, the rest still NaN) -> error / bound ratio."""
    main = got["f32"] if got["f32"] is not None else got["hi"]
    assert np.all(np.isfinite(main[inside])), "an output element of an active stream was not written"
    assert np.all(np.isnan(main[~inside])), "a row outside the active streams was written"
    if got["f32"] is not None:
        return ratio(main[inside], ref[inside], bound[inside])
    lo = got["lo"]
    assert np.all(np.isfinite(lo[inside])) and np.all(np.isnan(lo[~inside]))
    y = main[inside].astype(np.float64) + lo[inside]
    return ratio(y, ref[inside], bound[inside] + 2.0 ** -16 * np.abs(ref[inside]) + 1e-30)


# ------------------------------------------------------------------------------------------------------------ cases
def attention_case(seed, d, H, L, S, act, Cs, cache_len, ring_start, extra_rows=3):
    """Streams `act` (in that order) take Cs[a] rows each; the packed rows end with NaN sentinel rows no stream owns."""
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(Cs)]).astype(np.int32)
    rows = int(off[-1]) + extra_rows
    tmax = L + max(Cs) + 5
    qkv = rng.uniform(-1, 1, (rows, 3 * d)).astype(np.float32)
    qkv[int(off[-1]):] = np.nan
    kc = rng.uniform(-1, 1, (S, L, d)).astype(np.float32)
    vc = rng.uniform(-1, 1, (S, L, d)).astype(np.float32)
    return dict(d=d, H=H, L=L, tmax=tmax, act=np.array(act, np.int32), off=off, cl=np.array(cache_len, np.int32),
                rs=np.array(ring_start, np.int32), qkv=qkv, pp=rng.uniform(-1, 1, (2 * tmax - 1, d)).astype(np.float32),
                u=(0.3 * rng.uniform(-1, 1, d)).astype(np.float32), v=(0.3 * rng.uniform(-1, 1, d)).astype(np.float32), kc=kc, vc=vc)


def attention_cases(d, H):
    """Empty ring, partly filled ring, full wrapped ring, C > L, several active streams with gaps."""
    return {
        "empty": attention_case(1, d, H, 12, 1, [0], [2], [0], [0]),
        "partial": attention_case(2, d, H, 12, 1, [0], [2], [5], [0]),
        "wrapped": attention_case(3, d, H, 12, 1, [0], [1], [12], [7]),
        "c_gt_l": attention_case(4, d, H, 4, 1, [0], [6], [3], [2]),
        "gaps": attention_case(5, d, H, 70, 6, [4, 0, 2], [2, 1, 2], [70, 0, 33, 9, 65, 1], [13, 0, 0, 5, 69, 0]),
    }


def run_attention_case(pkg, math_mode, c):
    got = run_stream_attention(pkg, math_mode, c)
    ref, bd, kcn, vcn = ref_stream_attention(c["qkv"], c["pp"], c["u"], c["v"], c["kc"], c["vc"], c["act"], c["off"], c["cl"], c["rs"],
                                             c["L"], c["d"], c["H"], c["tmax"])
    inside = np.zeros(c["qkv"].shape[0], bool)
    inside[:int(c["off"][-1])] = True
    return got, ref, bd, kcn, vcn, inside


@gpu
@pytest.mark.parametrize("math_mode", [MATH_F32, MATH_X3], ids=["fp32", "bf16x3"])
@pytest.mark.parametrize("d,H", [(128, 2), (256, 2), (1024, 8)], ids=["hd64", "hd128", "hd128-d1024"])
def test_stream_attention_against_fp64(pkg, d, H, math_mode):
    worst = 0.0
    for name, c in attention_cases(d, H).items():
        got, ref, bd, kcn, vcn, inside = run_attention_case(pkg, math_mode, c)
        assert got["guard_bad"] == 0, name
        r = check_out(got, ref, bd, inside)
        assert r <= 1.0, (name, r)
        worst = max(worst, r)
        assert np.array_equal(got["kc"], kcn) and np.array_equal(got["vc"], vcn), f"{name}: ring update"
    report(f"stream attention d {d} heads {H} math {math_mode}", worst)


@gpu
def test_stream_attention_bound_rejects_mutations(pkg):
    """An off-by-one position row, the ring read without ring_start and a dropped pos_bias_v each exceed the bound."""
    c = attention_cases(256, 2)["gaps"]
    got, ref, bd, _, _, inside = run_attention_case(pkg, MATH_F32, c)
    assert check_out(got, ref, bd, inside) <= 1.0
    args = (c["qkv"], c["pp"], c["u"], c["v"], c["kc"], c["vc"], c["act"], c["off"], c["cl"], c["rs"], c["L"], c["d"], c["H"], c["tmax"])
    for kw in (dict(pos_shift=1), dict(ignore_ring_start=True), dict(drop_v=True)):
        mref, mbd, _, _ = ref_stream_attention(*args, **kw)
        r = ratio(got["f32"][inside], mref[inside], mbd[inside])
        report(f"stream attention mutation {kw}", r)
        assert r > 1.0, kw


def dwconv_case(seed, d, S, act, Cs, zero_cache=False, ks=9, extra_rows=2):
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(Cs)]).astype(np.int32)
    rows = int(off[-1]) + extra_rows
    glu = rng.uniform(-2, 2, (rows, d)).astype(np.float32)
    glu[int(off[-1]):] = np.nan
    cache = np.zeros((S, ks - 1, d), np.float32) if zero_cache else rng.uniform(-2, 2, (S, ks - 1, d)).astype(np.float32)
    return dict(ks=ks, act=np.array(act, np.int32), off=off, glu=glu, cache=cache,
                w=(rng.uniform(-1, 1, (d, ks)) / 3).astype(np.float32), b=rng.uniform(-0.5, 0.5, d).astype(np.float32))


DWCONV_CASES = {
    "zero_cache": lambda d: dwconv_case(11, d, 2, [1], [2], zero_cache=True),
    "carried": lambda d: dwconv_case(12, d, 5, [3, 0, 4], [2, 1, 2]),
    "c1": lambda d: dwconv_case(13, d, 3, [2], [1]),
}


@gpu
@pytest.mark.parametrize("math_mode", [MATH_F32, MATH_X3], ids=["fp32", "bf16x3"])
@pytest.mark.parametrize("d", [128, 1024])
def test_stream_dwconv_against_fp64(pkg, d, math_mode):
    worst = 0.0
    for name, mk in DWCONV_CASES.items():
        c = mk(d)
        got = run_stream_dwconv(pkg, math_mode, c)
        assert got["guard_bad"] == 0, name
        ref, bd, cn = ref_stream_dwconv(c["glu"], c["w"], c["b"], c["cache"], c["act"], c["off"], c["ks"])
        inside = np.zeros(c["glu"].shape[0], bool)
        inside[:int(c["off"][-1])] = True
        r = check_out(got, ref, bd, inside)
        assert r <= 1.0, (name, r)
        worst = max(worst, r)
        assert np.array_equal(got["cache"], cn), f"{name}: conv cache"
    report(f"stream dwconv d {d} math {math_mode}", worst)


@gpu
def test_stream_dwconv_bound_rejects_ignored_cache(pkg):
    c = DWCONV_CASES["carried"](128)
    got = run_stream_dwconv(pkg, MATH_F32, c)
    inside = np.zeros(c["glu"].shape[0], bool)
    inside[:int(c["off"][-1])] = True
    mref, mbd, _ = ref_stream_dwconv(c["glu"], c["w"], c["b"], c["cache"], c["act"], c["off"], c["ks"], ignore_cache=True)
    r = ratio(got["f32"][inside], mref[inside], mbd[inside])
    report("stream dwconv mutation: cache ignored", r)
    assert r > 1.0


# ------------------------------------------------------------------------------------------------------------ CPU
def test_ref_stream_dwconv_matches_oracle_conv_cached(O):
    """The float64 dwconv reference against oracle.depthwise_conv1d on [cache | chunk] (no padding)."""
    c = dwconv_case(22, 16, 1, [0], [3], extra_rows=0)
    ref, _, cn = ref_stream_dwconv(c["glu"], c["w"], c["b"], c["cache"], c["act"], c["off"], c["ks"])
    seq = np.concatenate([c["cache"][0], c["glu"]]).T                # (d, ks - 1 + C)
    pre = O.depthwise_conv1d(seq, c["w"][:, None, :], c["b"], 0).T.astype(np.float64)
    want = pre / (1 + np.exp(-pre))
    assert np.abs(ref - want).max() < 1e-5 * max(1.0, np.abs(want).max())
    assert np.array_equal(cn[0], np.concatenate([c["cache"][0], c["glu"]])[-(c["ks"] - 1):])


def test_mutated_references_differ(O):
    """The mutations the GPU test must reject change the float64 reference well beyond the bound (CPU-side check of the
    sensitivity cases, so that a weak case shows up without a device)."""
    c = attention_cases(256, 2)["gaps"]
    args = (c["qkv"], c["pp"], c["u"], c["v"], c["kc"], c["vc"], c["act"], c["off"], c["cl"], c["rs"], c["L"], c["d"], c["H"], c["tmax"])
    ref, bd, _, _ = ref_stream_attention(*args)
    inside = np.zeros(c["qkv"].shape[0], bool)
    inside[:int(c["off"][-1])] = True
    for kw in (dict(pos_shift=1), dict(ignore_ring_start=True), dict(drop_v=True)):
        m, _, _, _ = ref_stream_attention(*args, **kw)
        assert ratio(m[inside], ref[inside], bd[inside]) > 10.0, kw
    d = DWCONV_CASES["carried"](128)
    ref, bd, _ = ref_stream_dwconv(d["glu"], d["w"], d["b"], d["cache"], d["act"], d["off"], d["ks"])
    m, _, _ = ref_stream_dwconv(d["glu"], d["w"], d["b"], d["cache"], d["act"], d["off"], d["ks"], ignore_cache=True)
    ins = np.zeros(d["glu"].shape[0], bool)
    ins[:int(d["off"][-1])] = True
    assert ratio(m[ins], ref[ins], bd[ins]) > 10.0
