"""The front of the pipeline against float64 math, element by element: the log-mel (mel.cu K1, offline and streaming), the
per-utterance normalisation (K2) and the convolutional subsampling front (subsample.cu K3 conv1 + ReLU + dw1, K4 dw2),
through pk_kernel_mel, pk_kernel_mel_stream, pk_kernel_subsample_conv1 and pk_kernel_subsample_dw.  As in
test_kernels_fp64.py, outputs sit between 0xFF guard bands (NaN), so each case checks that no guard byte changed, the exact
set of elements written, and every element's error against a float64 reference divided by its own bound.

The references work on the exact fp32 inputs and the fp32 constants the kernels use: the fp32 symmetric Hann window, the
fp32 Slaney filterbank (the oracle's mel_filterbank, built in double as the engine builds it), 0.97f, 5.96046448e-8f, 1e-5f.

Bounds (u = 2^-24):
  K1 input    y_i = x_i - 0.97 x_{i-1} (one fma or two roundings), then v = y w: |e_v| <= 3 u |w| (|x_i| + 0.97 |x_{i-1}|).
  K1 FFT      the 512 real samples are a 256-point complex FFT in 8 radix-2 levels (three in the 8-point DFT, five across the
              lanes), each with at most one twiddle product (W8, the four-step twiddle, W_{2h}); twiddles are fp32 roundings.
              Higham (Accuracy and Stability, Thm 24.2): ||dZ||_2 <= 8 eta ||Z||_2 with eta = mu + gamma_4 (sqrt 2 + mu) <= 7.1 u
              and ||Z||_2 = 16 ||v||_2, so ||dZ||_2 <= 909 u ||v||_2.  The untangling X_k = E_k + W_k O_k reads Z_k and Z_{256-k}
              and rounds a few times: |dX_k| <= 2 * 909 u ||v|| + 8 u * 16 ||v|| <= 1946 u ||v||.  Written as
              C_FFT log2(512) sqrt(512) u ||v||_2 with C_FFT = 10 (9.6 needed).  The bound is norm-wise: the kernel's summation
              order differs from rfft's, so one bin's error is not bounded by its own terms.  D_k = sum |e_v| + that.
  K1 power    P = |X|^2 in fp32: |dP| <= 2 |X| D + D^2 plus 3 u of the result.
  K1 mel      sparse fma chain of len_m filter weights: |dmel| <= fb . |dP| + (len_m + 1) u fb . (P + |dP|); + 5.96e-8f rounds
              once more (u a, a = mel + 5.96e-8).  log: |dlog| <= -log(1 - da / a) (infinite when da >= a: such a bin is not
              constrained) plus logf's 1 ulp (2 u |log a|).  Times C_K1 = 2.  Weak bins next to strong ones get a large bound,
              strong bins a tight one.
  K1 stream   the signal is already pre-emphasised: |e_v| <= u |v|; the rest as above.
  K2          on the kernel's own log-mel x (F frames of an utterance, one bin), shifted: z = x - x0 (x0 = frame 0), one
              rounding, |dz| <= u |z|.  16 chunks of n_c in {floor(F/16), ceil(F/16)} frames; G = 640 / n_mels thread groups
              each add ceil(n_c / G) frames, then the G partials are added: depth k_c = ceil(n_c / G) + G.  Chunk mean of z:
              |dm_c| <= (k_c + 1) u mean_c |z| + u |m_c|.  Chunk M2 (fma of the rounded differences d = z - m_c, each off by
              u |z| + dm_c; the dm_c terms cancel to first order): |dM2_c| <= (k_c + 3) u M2_c + 2 u sqrt(M2_c S_c) +
              2 u^2 S_c + 2 n_c dm_c^2 (S_c = sum z^2).  Chan's combination: mean = (16-term fma chain of n_c m_c) / F:
              |dmu| <= (17 u sum n_c |m_c| + sum n_c dm_c) / F + u |mu|; between-chunk term
              B = sum n_c d_c^2 (d_c = m_c - mu) with |dd_c| <= e_c = dm_c + dmu + u |d_c|: |dB| <= sum n_c (2 |d_c| e_c + e_c^2)
              + 4 u B; the 32 partial sums: 18 u (sum M2_c + B).  var = M2 / (F - 1) (+ u var); sigma: |ds| <=
              min(dvar / (2 s), sqrt(dvar)) + u s; 1 / (s + 1e-5) (two roundings): relative r = (ds + u den) / (den - ds - u den) + u;
              y = (z - mu) inv: |dy| <= (dmu + u |z|) inv + |z - mu| inv r + 2 u |y|.  Times C_K2 = 2.  A constant bin (digital
              silence) has z = 0 exactly: its features are exactly 0.  A single two-pass sum would give
              F u instead of the depth k_c: the bound follows the chunked form the kernel runs.
  K3          conv1: 9-term fma chain from the bias: |e1| <= 10 u (|b1| + sum |w1 x|); ReLU is 1-Lipschitz; dw1 the same chain
              on conv1's values: |err| <= sum |wd| e1 + 10 u (|bd| + sum |wd h|).  Padding is exact zeros.  Times C_SUB = 2.
  K4          one such chain: |err| <= 10 u (|bd| + sum |wd x|), times C_SUB.
  planes      bf16 hi + lo stands for the fp32 value within 2^-16 |y| (check_planes adds it).
Sensitivity: references mutated the way a plausible bug would (periodic Hann, one reflection, reflection before
pre-emphasis, biased variance, eps inside the root, equal chunk weights, conv1 values in dw1's padding, neighbour rows
instead of zero padding) are compared with the same kernel output and must be rejected.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math

import numpy as np
import pytest
from test_kernels_fp64 import check_planes, nan, ratio, report

gpu = pytest.mark.gpu

U = 2.0 ** -24
C_FFT, C_K1, C_K2, C_SUB = 10.0, 2.0, 2.0, 2.0
PRE = float(np.float32(0.97))
EPS_LOG = float(np.float32(5.96046448e-8))
EPS_STD = float(np.float32(1e-5))
MATH_X3, MATH_X1, MATH_F32 = 0, 1, 2
MATHS = (MATH_X3, MATH_X1, MATH_F32)
MEL_CH = 16


def _f(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def _i32(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _i64(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def cl(n):
    """output length of a 3-tap, stride-2, padding-1 convolution"""
    return (n - 1) // 2 + 1


# ----------------------------------------------------------------------------------------------------------- K1 reference
def hann(periodic=False):
    i = np.arange(400, dtype=np.float64)
    return (0.5 - 0.5 * np.cos(2.0 * np.pi * i / (400.0 if periodic else 399.0))).astype(np.float32).astype(np.float64)


def reflect(i, n, once=False):
    """axiom's reflect padding, repeated until the index lands in [0, n) (once: one reflection, then clamped)."""
    i = i.copy()
    while True:
        i = np.where(i < 0, -i, i)
        i = np.where(i >= n, 2 * n - 2 - i, i)
        if once:
            return np.clip(i, 0, n - 1)
        if not ((i < 0) | (i >= n)).any():
            return i


def offline_frames(x, mutate=None):
    """Windowed samples of every centred frame (taps 56..455 of the 512-point frame) -> (v [F][400], input error bound [F][400]).
    mutate: "periodic" Hann, "once" (one reflection), "reflect_raw" (reflect the raw signal, pre-emphasise after)."""
    n = len(x)
    F = 1 + n // 160
    x64 = x.astype(np.float64)
    idx = np.arange(F)[:, None] * 160 - 256 + 56 + np.arange(400)[None, :]
    if mutate == "reflect_raw":
        cur, prev = x64[reflect(idx, n)], x64[reflect(idx - 1, n)]
    else:
        r = reflect(idx, n, once=mutate == "once")
        cur, prev = x64[r], np.where(r > 0, x64[np.maximum(r - 1, 0)], 0.0)
    w = hann(periodic=mutate == "periodic")
    return (cur - PRE * prev) * w, 3 * U * (np.abs(cur) + PRE * np.abs(prev)) * w


def spectrum(v, ev):
    """-> (|X| [F][257] of the 512-point frames, norm-wise bin error D [F])."""
    X = np.fft.rfft(np.pad(v, ((0, 0), (56, 56))), axis=1)
    D = ev.sum(axis=1) + C_FFT * 9 * math.sqrt(512) * U * np.linalg.norm(v, axis=1)
    return np.abs(X), D


def logmel_from_spectrum(absX, D, fb):
    """-> (float64 log-mel [F][n_mels], bound)."""
    P = absX ** 2
    dP = 2 * absX * D[:, None] + D[:, None] ** 2
    dP += 3 * U * (P + dP)
    ln = (fb != 0).sum(axis=0)
    mel = P @ fb
    dmel = dP @ fb + (ln + 1) * U * ((P + dP) @ fb)
    a = mel + EPS_LOG
    da = dmel + U * (a + dmel)
    r = da / a
    dlog = np.where(r < 1, -np.log1p(-np.minimum(r, 1 - 1e-16)), np.inf)
    return np.log(a), C_K1 * (dlog + 2 * U * np.abs(np.log(a)))


def ref_logmel(x, fb, mutate=None):
    return logmel_from_spectrum(*spectrum(*offline_frames(x, mutate)), fb)


# ----------------------------------------------------------------------------------------------------------- K2 reference
def chunks(F):
    return [(c * F // MEL_CH, (c + 1) * F // MEL_CH) for c in range(MEL_CH)]


def ref_normalize(lm, n_mels, mutate=None):
    """float64 normalisation of one utterance's log-mel x [F][n_mels] -> (features, bound).
    mutate: "biased" variance, "eps_inside" the root, "equal_weights" in Chan's combination."""
    x = lm.astype(np.float64)
    x = x - x[0]                          # the kernel's shift; exact here, one rounding in the kernel (in the bound)
    F = x.shape[0]
    G = 640 // n_mels
    n_c = np.array([b - a for a, b in chunks(F)], np.float64)
    m_c = np.array([x[a:b].mean(axis=0) if b > a else np.zeros(x.shape[1]) for a, b in chunks(F)])
    A_c = np.array([np.abs(x[a:b]).sum(axis=0) for a, b in chunks(F)])
    M2_c = np.array([((x[a:b] - m) ** 2).sum(axis=0) for (a, b), m in zip(chunks(F), m_c)])
    S_c = np.array([(x[a:b] ** 2).sum(axis=0) for a, b in chunks(F)])
    if mutate == "equal_weights":
        w = np.full(MEL_CH, F / MEL_CH)
        mu = (w[:, None] * m_c).sum(axis=0) / F
        M2 = M2_c.sum(axis=0) + (w[:, None] * (m_c - mu) ** 2).sum(axis=0)
    else:
        mu = x.mean(axis=0)
        M2 = ((x - mu) ** 2).sum(axis=0)
    var = M2 / (F if mutate == "biased" else F - 1)
    sd = np.sqrt(var)
    den = np.sqrt(var + EPS_STD) if mutate == "eps_inside" else sd + EPS_STD
    c = x - mu
    y = c / den
    # bound
    k_c = np.ceil(n_c / G) + G
    safe = np.maximum(n_c, 1)[:, None]
    dm_c = np.where(n_c[:, None] > 0, (k_c[:, None] + 1) * U * A_c / safe + U * np.abs(m_c), 0.0)
    dM2_c = (k_c[:, None] + 3) * U * M2_c + 2 * U * np.sqrt(M2_c * S_c) + 2 * U * U * S_c + 2 * n_c[:, None] * dm_c ** 2
    dmu = (17 * U * (n_c[:, None] * np.abs(m_c)).sum(axis=0) + (n_c[:, None] * dm_c).sum(axis=0)) / F + U * np.abs(mu)
    d_c = m_c - mu
    e_c = dm_c + dmu + U * np.abs(d_c)
    B = (n_c[:, None] * d_c ** 2).sum(axis=0)
    dB = (n_c[:, None] * (2 * np.abs(d_c) * e_c + e_c ** 2)).sum(axis=0) + 4 * U * B
    dm2 = dM2_c.sum(axis=0) + dB + 18 * U * (M2_c.sum(axis=0) + B)
    dvar = dm2 / (F - 1) + U * var
    with np.errstate(divide="ignore", invalid="ignore"):
        dsd = np.minimum(np.where(sd > 0, dvar / (2 * sd), np.inf), np.sqrt(dvar)) + U * sd
    dd = dsd + U * (sd + EPS_STD)
    r_inv = np.where(dd < sd + EPS_STD, dd / np.maximum(sd + EPS_STD - dd, 1e-300), np.inf) + U
    inv = 1.0 / (sd + EPS_STD)
    bound = (dmu + U * np.abs(x)) * inv + np.abs(c) * inv * r_inv + 2 * U * np.abs(y)
    return y, C_K2 * bound


# ----------------------------------------------------------------------------------------------------------- K3 / K4 references
def ref_conv1_dw1(xu, w1, b1, wd, bd, ctx=None, conv1_pad=False):
    """float64 conv1 (1 -> C, 3x3, s2, p1) + ReLU + depthwise dw1 (3x3, s2, p1) of one utterance's features xu [F][mel]
    -> (y [(t2, f2)][C], bound).  Mutations: ctx [F + 6][mel] = the packed rows -3 .. F + 2 around the utterance (conv1
    reads neighbour rows instead of zeros); conv1_pad: dw1's padding rows t1 = -1 and t1n hold conv1 evaluated there
    (ReLU(b1 + ...)) instead of zeros."""
    F, mel = xu.shape
    Cn = w1.shape[0]
    t1n, f1n = cl(F), cl(mel)
    t2n, f2n = cl(t1n), cl(f1n)
    X = np.zeros((F + 6, mel + 6))
    X[3:3 + F, 3:3 + mel] = xu
    if ctx is not None:
        X[:, 3:3 + mel] = ctx
    y = np.zeros((Cn, t2n, f2n))
    bd_ = np.zeros((Cn, t2n, f2n))
    for c0 in range(0, Cn, 128):
        cs = slice(c0, min(Cn, c0 + 128))
        W1, B1, WD, BD = (a[cs].astype(np.float64) for a in (w1, b1, wd, bd))
        # conv1 on the grid t1 = -1 .. t1n, f1 = -1 .. f1n (index + 1): reads feature rows 2 t1 - 1 + p
        h = np.broadcast_to(B1[:, None, None], (len(B1), t1n + 2, f1n + 2)).copy()
        A1 = np.abs(h)
        for p in range(3):
            for q in range(3):
                patch = X[p:p + 2 * (t1n + 2):2, q:q + 2 * (f1n + 2):2][None]
                h += W1[:, 3 * p + q, None, None] * patch
                A1 += np.abs(W1[:, 3 * p + q, None, None] * patch)
        r = np.maximum(h, 0)
        e1 = 10 * U * A1
        keep = np.zeros((t1n + 2, f1n + 2), bool)
        keep[1:t1n + 1, 1:f1n + 1] = True
        if conv1_pad:
            keep[:, 1:f1n + 1] = True
        r, e1 = np.where(keep, r, 0.0), np.where(keep, e1, 0.0)
        acc = np.broadcast_to(BD[:, None, None], (len(BD), t2n, f2n)).copy()
        A2, E = np.abs(acc), np.zeros_like(acc)
        for i in range(3):
            for j in range(3):
                wk = WD[:, 3 * i + j, None, None]
                tap = r[:, i:i + 2 * t2n:2, j:j + 2 * f2n:2]
                acc += wk * tap
                A2 += np.abs(wk * tap)
                E += np.abs(wk) * e1[:, i:i + 2 * t2n:2, j:j + 2 * f2n:2]
        y[cs], bd_[cs] = acc, C_SUB * (E + 10 * U * A2)
    return y.transpose(1, 2, 0).reshape(-1, Cn), bd_.transpose(1, 2, 0).reshape(-1, Cn)


def ref_dw(xu, wd_tap, bd, prev_row=None, next_row=None, e_in=None):
    """float64 depthwise 3x3 s2 p1 of one utterance xu [tin][fin][C] -> (y [(t', f')][C], bound).  Mutation: prev_row /
    next_row [fin][C] = the neighbouring utterances' rows read instead of zeros at t = -1 / tin.  e_in [tin][fin][C]: a
    bound on the input's error (a chain of kernels), which adds sum |wd| e_in."""
    tin, fin, Cn = xu.shape
    tout, fout = cl(tin), cl(fin)
    X = np.zeros((tin + 2, fin + 2, Cn))
    X[1:tin + 1, 1:fin + 1] = xu
    E = np.zeros((tin + 2, fin + 2, Cn))
    if e_in is not None:
        E[1:tin + 1, 1:fin + 1] = e_in
    if prev_row is not None:
        X[0, 1:fin + 1] = prev_row
    if next_row is not None:
        X[tin + 1, 1:fin + 1] = next_row
    acc = np.broadcast_to(bd.astype(np.float64), (tout, fout, Cn)).copy()
    A, P = np.abs(acc), np.zeros_like(acc)
    for i in range(3):
        for j in range(3):
            t = wd_tap[3 * i + j].astype(np.float64) * X[i:i + 2 * tout:2, j:j + 2 * fout:2]
            acc += t
            A += np.abs(t)
            P += np.abs(wd_tap[3 * i + j].astype(np.float64)) * E[i:i + 2 * tout:2, j:j + 2 * fout:2]
    return acc.reshape(-1, Cn), (C_SUB * 10 * U * A + P).reshape(-1, Cn)


# ----------------------------------------------------------------------------------------------------------- hook runners
def run_mel(pkg, pcms, n_mels, normalize, lead=0):
    """-> (log-mel per utterance, features per utterance or None); `lead` NaN samples before the first utterance."""
    L = pkg.load_library()
    lens = np.array([len(p) for p in pcms], np.int64)
    off = np.concatenate([[lead], lead + np.cumsum(lens)]).astype(np.int64)
    buf = np.ascontiguousarray(np.concatenate([nan(lead)] + [np.asarray(p, np.float32) for p in pcms]))
    F = 1 + lens // 160
    fo = np.concatenate([[0], np.cumsum(F)])
    lm = nan((int(fo[-1]), n_mels))
    ft = nan((int(fo[-1]), n_mels)) if normalize else None
    gb = C.c_int64(-1)
    st = L.pk_kernel_mel(0, len(pcms), _i64(off), _f(buf), n_mels, int(normalize), _f(lm), _f(ft), C.byref(gb))
    assert st == 0, f"pk_kernel_mel -> {st}"
    assert gb.value == 0
    assert np.all(np.isfinite(lm)), "a log-mel element was not written"
    if ft is not None:
        assert np.all(np.isfinite(ft)), "a feature element was not written"
    cut = lambda a: None if a is None else [a[fo[b]:fo[b + 1]] for b in range(len(pcms))]   # noqa: E731
    return cut(lm), cut(ft)


def run_mel_stream(pkg, sigs, n_frames, out_row, rows_total, n_mels, lead=0):
    L = pkg.load_library()
    off = np.concatenate([[lead], lead + np.cumsum([len(s) for s in sigs])]).astype(np.int64)
    buf = np.ascontiguousarray(np.concatenate([nan(lead)] + [np.asarray(s, np.float32) for s in sigs]))
    nf, orow = np.array(n_frames, np.int32), np.array(out_row, np.int32)
    lm = nan((rows_total, n_mels))
    gb = C.c_int64(-1)
    st = L.pk_kernel_mel_stream(0, len(sigs), _i64(off), _f(buf), _i32(nf), _i32(orow), rows_total, n_mels, _f(lm), C.byref(gb))
    assert st == 0, f"pk_kernel_mel_stream -> {st}"
    assert gb.value == 0
    return lm


def act_arrays(math_mode, shape):
    f32 = math_mode == MATH_F32
    return (nan(shape) if f32 else None, None if f32 else nan(shape), nan(shape) if math_mode == MATH_X3 else None)


def run_conv1(pkg, math_mode, frame_off, feats, w1, b1, wd, bd):
    L = pkg.load_library()
    fo = np.ascontiguousarray(frame_off, np.int32)
    rows, mel = feats.shape
    Cn = w1.shape[0]
    n_out = sum(cl(cl(int(fo[b + 1] - fo[b]))) for b in range(len(fo) - 1)) * cl(cl(mel))
    of, hi, lo = act_arrays(math_mode, (n_out, Cn))
    gb = C.c_int64(-1)
    st = L.pk_kernel_subsample_conv1(0, math_mode, len(fo) - 1, _i32(fo), rows, _f(feats), mel, Cn, _f(w1), _f(b1), _f(wd), _f(bd),
                                     _f(of), _f(hi), _f(lo), C.byref(gb))
    assert st == 0, f"pk_kernel_subsample_conv1 -> {st}"
    assert gb.value == 0
    return of, hi, lo


def run_dw(pkg, math_mode, in_rows, x, wd_tap, bd):
    L = pkg.load_library()
    ir = np.ascontiguousarray(in_rows, np.int32)
    _, fin, Cn = x.shape
    n_out = sum(cl(int(t)) for t in ir) * cl(fin)
    of, hi, lo = act_arrays(math_mode, (n_out, Cn))
    gb = C.c_int64(-1)
    st = L.pk_kernel_subsample_dw(0, math_mode, len(ir), _i32(ir), fin, Cn, _f(np.ascontiguousarray(x)), _f(wd_tap), _f(bd), _f(of), _f(hi),
                                  _f(lo), C.byref(gb))
    assert st == 0, f"pk_kernel_subsample_dw -> {st}"
    assert gb.value == 0
    return of, hi, lo


def check_act(out, y, bd, rows=None):
    """the written set (every row of `rows`, default all, finite) and err / bound of the output in its math mode's form."""
    of, hi, lo = out
    sel = (lambda a: a) if rows is None else (lambda a: a[rows])   # noqa: E731
    for a in (of, hi, lo):
        assert a is None or np.all(np.isfinite(sel(a))), "an output element was not written (or read NaN padding)"
    if of is not None:
        return ratio(sel(of), y, bd)
    return check_planes(sel(hi), None if lo is None else sel(lo), y, bd)


# ----------------------------------------------------------------------------------------------------------- signals
MEL_LENS = [400, 401, 559, 560, 561, 2399, 2560, 16000, 16159, 960000]       # 2399: F = 15, 2560: F = 17, 960000: 60 s
SHORT_LENS = [2, 3, 17, 100, 199, 200, 201, 255, 256, 257, 399]
SIGNALS = ["speech", "near_silence", "clipped_noise", "impulse", "tone", "dc", "zeros"]


def signal(kind, n, seed, synth):
    rng = np.random.default_rng(seed)
    if kind == "speech":
        return synth.make_audio(n, seed)
    if kind == "near_silence":
        return (1e-4 * rng.standard_normal(n)).astype(np.float32)
    if kind == "clipped_noise":
        return np.clip(1.5 * rng.standard_normal(n), -1, 1).astype(np.float32)
    if kind == "impulse":
        x = np.zeros(n, np.float32)
        x[[0, n // 2, n - 1]] = 1.0
        return x
    if kind == "tone":                     # on the centre of FFT bin 40 (1250 Hz)
        return (0.5 * np.sin(2 * np.pi * 40 / 512 * np.arange(n))).astype(np.float32)
    if kind == "dc":
        return np.full(n, 0.25, np.float32)
    return np.zeros(n, np.float32)


def fbank(O, n_mels):
    return O.mel_filterbank(257, n_mels).astype(np.float64)


# ----------------------------------------------------------------------------------------------------------- K1 + K2, offline
@gpu
@pytest.mark.parametrize("n_mels", [80, 128, 24])
def test_mel_against_fp64(pkg, O, synth, n_mels):
    """Every signal kind as a permuted ragged batch of every length (the interior / edge switch at n = 160 k and 160 k + 159,
    F = 15 and 17 for the chunked normalisation, a 60 s clip of 6001 frames), with NaN samples before the first utterance."""
    fb = fbank(O, n_mels)
    w1 = w2 = 0.0
    for si, kind in enumerate(SIGNALS):
        rng = np.random.default_rng(si + n_mels)
        lens = [int(v) for v in rng.permutation(MEL_LENS)]
        pcms = [signal(kind, n, 1000 * si + n % 997, synth) for n in lens]
        lm, ft = run_mel(pkg, pcms, n_mels, True, lead=13)
        for x, g_lm, g_ft in zip(pcms, lm, ft):
            ref, bd = ref_logmel(x, fb)
            w1 = max(w1, ratio(g_lm, ref, bd))
            y, bd2 = ref_normalize(g_lm, n_mels)
            w2 = max(w2, ratio(g_ft, y, bd2))
            if kind == "zeros":            # digital silence: log(5.96e-8f) in every bin and features of exactly 0
                assert np.all(g_lm == g_lm[0, 0]) and abs(float(g_lm[0, 0]) - math.log(EPS_LOG)) <= 2 * U * abs(math.log(EPS_LOG))
                assert np.all(g_ft == 0)
    report(f"mel K1 n_mels {n_mels}", w1)
    report(f"mel K2 n_mels {n_mels}", w2)
    assert w1 <= 1.0 and w2 <= 1.0


@gpu
@pytest.mark.parametrize("n_mels", [128, 80])
def test_mel_unnormalised_short_signals_against_fp64(pkg, O, synth, n_mels):
    """normalize = 0 (the Sortformer path) on 2..399-sample signals: repeated reflection; every output row is checked."""
    fb = fbank(O, n_mels)
    worst = 0.0
    for seed, kind in enumerate(("speech", "clipped_noise", "impulse")):
        rng = np.random.default_rng(seed)
        lens = [int(v) for v in rng.permutation(SHORT_LENS)]
        pcms = [signal(kind, n, 50 + seed * 7 + n, synth) for n in lens]
        lm, _ = run_mel(pkg, pcms, n_mels, False, lead=5)
        for x, g in zip(pcms, lm):
            ref, bd = ref_logmel(x, fb)
            assert g.shape == ref.shape
            worst = max(worst, ratio(g, ref, bd))
    report(f"mel K1 normalize=0 n_mels {n_mels}", worst)
    assert worst <= 1.0


@gpu
@pytest.mark.parametrize("n_mels", [128, 80])
def test_mel_stream_against_fp64(pkg, O, n_mels):
    """The streaming frames (no centring, no reflection) of streams with 0, 1, 2 and 7 frames into rows with gaps between
    streams; the rows not named by out_row / n_frames must stay unwritten."""
    fb = fbank(O, n_mels)
    rng = np.random.default_rng(n_mels)
    nfs = [7, 0, 1, 2, 7, 1, 0, 2]
    sigs, rows, r = [], [], 3
    for i, nf in enumerate(nfs):
        n = (nf - 1) * 160 + 512 + int(rng.integers(0, 159)) if nf else int(rng.integers(0, 300))
        s = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 0)).astype(np.float32)
        sigs.append(s)
        rows.append(r)
        r += nf + int(rng.integers(0, 3))
    rows_total = r + 4
    lm = run_mel_stream(pkg, sigs, nfs, rows, rows_total, n_mels, lead=9)
    named = np.zeros(rows_total, bool)
    worst = 0.0
    w = hann()
    for s, nf, r0 in zip(sigs, nfs, rows):
        named[r0:r0 + nf] = True
        if nf == 0:
            continue
        idx = np.arange(nf)[:, None] * 160 + 56 + np.arange(400)[None, :]
        v = s.astype(np.float64)[idx] * w
        ref, bd = logmel_from_spectrum(*spectrum(v, U * np.abs(v)), fb)
        worst = max(worst, ratio(lm[r0:r0 + nf], ref, bd))
    assert np.all(np.isfinite(lm[named])), "a named row was not written"
    assert np.all(np.isnan(lm[~named])), "a row outside the streams' frames was written"
    report(f"mel stream n_mels {n_mels}", worst)
    assert worst <= 1.0


@gpu
def test_mel_bounds_reject_mutations(pkg, O, synth):
    """Each mutated reference is compared with the kernel's real output and must exceed the bound."""
    n_mels = 128
    fb = fbank(O, n_mels)
    rng = np.random.default_rng(77)
    pcms = [synth.make_audio(n, 300 + n) for n in (16000, 2399, 2560, 561, 4000)]
    pcms.append((0.3 * np.sin(2 * np.pi * 23 / 512 * np.arange(8000)) + 1e-3 * rng.standard_normal(8000)).astype(np.float32))
    lm, ft = run_mel(pkg, pcms, n_mels, True)
    short = [synth.make_audio(n, 400 + n) for n in (17, 100, 150, 199, 200)]
    lm_s, _ = run_mel(pkg, short, n_mels, False)

    def worst_k1(xs, got, mutate):
        w = 0.0
        for x, g in zip(xs, got):
            ref, bd = ref_logmel(x, fb)
            assert ratio(g, ref, bd) <= 1.0
            if mutate:
                mref, _ = ref_logmel(x, fb, mutate)
                w = max(w, ratio(g, mref, bd))
        return w

    worst_k1(pcms + short, lm + lm_s, None)
    for name, xs, got in (("periodic", pcms, lm), ("reflect_raw", pcms, lm), ("once", short, lm_s)):
        r = worst_k1(xs, got, name)
        report(f"mel mutation {name}", r)
        assert r > 1.0, name
    for name in ("biased", "eps_inside", "equal_weights"):
        r = 0.0
        for g_lm, g_ft in zip(lm, ft):
            y, bd = ref_normalize(g_lm, n_mels)
            assert ratio(g_ft, y, bd) <= 1.0
            if name == "equal_weights" and g_lm.shape[0] % MEL_CH == 0:
                continue
            r = max(r, ratio(g_ft, ref_normalize(g_lm, n_mels, name)[0], bd))
        report(f"mel normalisation mutation {name}", r)
        assert r > 1.0, name


# ----------------------------------------------------------------------------------------------------------- same code as the engine
@gpu
@pytest.mark.parametrize("n_mels", [80, 128])
def test_mel_hook_runs_the_engine_code(pkg, O, synth, tiny, tmp_path, n_mels):
    """pk_kernel_mel's features equal Engine.mel of the same batch bit for bit: the hook runs the engine's tables and launches."""
    if n_mels == tiny.ocfg.mel_bins:
        cfg, wpath = tiny.cfg, tiny.weights_path
    else:
        ocfg = dataclasses.replace(O.make_tiny_config(), mel_bins=n_mels)
        wpath = str(tmp_path / f"tiny_mel{n_mels}.safetensors")
        synth.save_safetensors(wpath, synth.make_weights(ocfg, seed=4))
        cfg = pkg.make_tiny_config(mel_bins=n_mels)
    pcms = [synth.make_audio(n, 60 + n % 89) for n in (16000, 401, 2399, 33333, 560)]
    e = pkg.Engine(cfg, wpath, 0)
    try:
        want = np.concatenate(e.mel(pcms))
    finally:
        e.close()
    _, ft = run_mel(pkg, pcms, n_mels, True)
    assert np.array_equal(np.concatenate(ft), want)


@gpu
@pytest.mark.parametrize("mel_bins", [648, 1024, 0])
def test_engine_rejects_mel_bins_beyond_the_normalisation(pkg, mel_bins):
    """The normalisation runs 640 / mel_bins frame groups per block: configs outside 8..640 are refused at creation, with a
    message, instead of failing at the first pk_mel."""
    with pytest.raises(RuntimeError, match="mel_bins"):
        pkg.Engine(pkg.make_tiny_config(mel_bins=mel_bins), "/nonexistent/weights.safetensors", 0)
    with pytest.raises(RuntimeError, match="mel_bins"):
        pkg.Engine(pkg.engine.make_tiny_sortformer_config(mel_bins=mel_bins), "/nonexistent/weights.safetensors", 0)


# ----------------------------------------------------------------------------------------------------------- K3
CONV1_F = [1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 63, 64, 65, 1001]
CONV1_CFGS = [(80, 64), (80, 256), (80, 260), (80, 1024), (128, 64), (128, 256), (128, 260), (128, 1024), (82, 64)]   # 82: f1n odd


def conv1_weights(rng, Cn):
    return (rng.normal(0, 0.4, (Cn, 9)).astype(np.float32), rng.normal(0, 0.2, Cn).astype(np.float32),
            rng.normal(0, 0.4, (Cn, 9)).astype(np.float32), rng.normal(0, 0.1, Cn).astype(np.float32))


def feat_rows(rng, rows, mel):
    return (rng.standard_normal((rows, mel)) * 10.0 ** rng.uniform(-1, 1, (rows, 1))).astype(np.float32)


@gpu
@pytest.mark.parametrize("mel,Cn", CONV1_CFGS, ids=[f"mel{m}-C{c}" for m, c in CONV1_CFGS])
def test_subsample_conv1_against_fp64(pkg, mel, Cn):
    """A permuted ragged batch of every F (every residue of F mod 4, neighbour utterances on both sides), then each F alone
    inside NaN feature rows (a read outside the utterance makes NaN); all three math modes."""
    rng = np.random.default_rng(mel * 7 + Cn)
    w = conv1_weights(rng, Cn)
    worst = dict.fromkeys(MATHS, 0.0)
    order = [int(v) for v in rng.permutation(CONV1_F)]
    fo = np.concatenate([[0], np.cumsum(order)]).astype(np.int32)
    feats = feat_rows(rng, int(fo[-1]), mel)
    refs = [ref_conv1_dw1(feats[fo[b]:fo[b + 1]], *w) for b in range(len(order))]
    y, bd = np.concatenate([r[0] for r in refs]), np.concatenate([r[1] for r in refs])
    for m in MATHS:
        worst[m] = max(worst[m], check_act(run_conv1(pkg, m, fo, feats, *w), y, bd))
    for F in CONV1_F:
        lead, tail = 5, 6
        x = nan((lead + F + tail, mel))
        x[lead:lead + F] = feat_rows(rng, F, mel)
        y, bd = ref_conv1_dw1(x[lead:lead + F], *w)
        for m in MATHS:
            worst[m] = max(worst[m], check_act(run_conv1(pkg, m, np.array([lead, lead + F]), x, *w), y, bd))
    for m in MATHS:
        report(f"subsample conv1+dw1 mel {mel} C {Cn} math {m}", worst[m])
    assert max(worst.values()) <= 1.0


@gpu
def test_subsample_conv1_bound_rejects_mutations(pkg):
    mel, Cn = 80, 64
    rng = np.random.default_rng(21)
    w = conv1_weights(rng, Cn)
    lens = [9, 16, 5, 17, 64]
    fo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    feats = feat_rows(rng, int(fo[-1]), mel)
    out = run_conv1(pkg, MATH_F32, fo, feats, *w)
    padded = np.zeros((int(fo[-1]) + 6, mel), np.float32)
    padded[3:3 + int(fo[-1])] = feats
    refs, muts = [], {"conv1 values in dw1's padding": [], "neighbour rows": []}
    for b in range(len(lens)):
        xu = feats[fo[b]:fo[b + 1]]
        refs.append(ref_conv1_dw1(xu, *w))
        muts["conv1 values in dw1's padding"].append(ref_conv1_dw1(xu, *w, conv1_pad=True)[0])
        muts["neighbour rows"].append(ref_conv1_dw1(xu, *w, ctx=padded[fo[b]:fo[b + 1] + 6])[0])
    y, bd = np.concatenate([r[0] for r in refs]), np.concatenate([r[1] for r in refs])
    assert check_act(out, y, bd) <= 1.0
    for name, ys in muts.items():
        r = check_act(out, np.concatenate(ys), bd)
        report(f"subsample conv1 mutation {name}", r)
        assert r > 1.0, name


# ----------------------------------------------------------------------------------------------------------- K4
DW_ROWS = [1, 2, 3, 4, 5, 8, 9, 16, 17, 63, 64, 65, 251]


def dw_weights(rng, Cn):
    return rng.normal(0, 0.4, (9, Cn)).astype(np.float32), rng.normal(0, 0.1, Cn).astype(np.float32)


@gpu
@pytest.mark.parametrize("fin", [20, 32], ids=["mel80", "mel128"])
@pytest.mark.parametrize("Cn", [64, 256, 260, 1024])
def test_subsample_dw_against_fp64(pkg, fin, Cn):
    """dw2 on a permuted ragged batch (the out_off binary search and every utterance edge), then each length between two
    NaN utterances (their rows must read as zero padding); all three math modes."""
    rng = np.random.default_rng(fin * 11 + Cn)
    wd, bd = dw_weights(rng, Cn)
    worst = dict.fromkeys(MATHS, 0.0)
    rows = [int(v) for v in rng.permutation(DW_ROWS)]
    x = (rng.standard_normal((sum(rows), fin, Cn)) * 10.0 ** rng.uniform(-1, 1, (sum(rows), 1, 1))).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(rows)])
    refs = [ref_dw(x[off[b]:off[b + 1]], wd, bd) for b in range(len(rows))]
    y, bnd = np.concatenate([r[0] for r in refs]), np.concatenate([r[1] for r in refs])
    for m in MATHS:
        worst[m] = max(worst[m], check_act(run_dw(pkg, m, rows, x, wd, bd), y, bnd))
    for t in DW_ROWS:
        xs = np.full((3 + t + 2, fin, Cn), np.nan, np.float32)
        xs[3:3 + t] = rng.standard_normal((t, fin, Cn))
        y, bnd = ref_dw(xs[3:3 + t], wd, bd)
        first = cl(3) * cl(fin)
        sel = np.arange(first, first + y.shape[0])
        for m in MATHS:
            worst[m] = max(worst[m], check_act(run_dw(pkg, m, [3, t, 2], xs, wd, bd), y, bnd, rows=sel))
    for m in MATHS:
        report(f"subsample dw2 fin {fin} C {Cn} math {m}", worst[m])
    assert max(worst.values()) <= 1.0


@gpu
def test_subsample_dw_bound_rejects_neighbour_rows(pkg):
    fin, Cn = 20, 64
    rng = np.random.default_rng(8)
    wd, bd = dw_weights(rng, Cn)
    rows = [5, 8, 3, 16]
    x = rng.standard_normal((sum(rows), fin, Cn)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(rows)])
    out = run_dw(pkg, MATH_F32, rows, x, wd, bd)
    refs, muts = [], []
    for b in range(len(rows)):
        xu = x[off[b]:off[b + 1]]
        refs.append(ref_dw(xu, wd, bd))
        muts.append(ref_dw(xu, wd, bd, prev_row=x[off[b] - 1] if b else None, next_row=x[off[b + 1]] if b + 1 < len(rows) else None)[0])
    y, bnd = np.concatenate([r[0] for r in refs]), np.concatenate([r[1] for r in refs])
    assert check_act(out, y, bnd) <= 1.0
    r = check_act(out, np.concatenate(muts), bnd)
    report("subsample dw2 mutation neighbour rows", r)
    assert r > 1.0


# ----------------------------------------------------------------------------------------------------------- the references, pinned (CPU)
def test_ref_logmel_matches_oracle(O, synth):
    """The float64 log-mel equals the oracle's fp32 log_mel_unnormalised within the kernel's bound (which covers fp32
    noise), at 80 and 128 bins, for centred frames at both edges and for 2..200-sample signals (repeated reflection)."""
    for n_mels in (80, 128):
        fb = fbank(O, n_mels)
        for n in (2, 17, 100, 199, 200, 201, 400, 561, 2399, 16000):
            x = synth.make_audio(n, 7 + n)
            ref, bd = ref_logmel(x, fb)
            assert ratio(O.log_mel_unnormalised(x, n_mels).T, ref, bd) <= 1.0, n


def test_ref_normalize_matches_oracle(O, synth):
    for n_mels in (80, 128):
        for n in (400, 2399, 2560, 16000):
            x = synth.make_audio(n, 11 + n)
            lm = O.log_mel_unnormalised(x, n_mels).T
            y, bd = ref_normalize(lm, n_mels)
            assert ratio(O.preprocess_audio(x, n_mels), y, bd) <= 1.0, n


def test_ref_subsampling_matches_oracle(O, tiny):
    """conv1 + ReLU + dw1 and the depthwise stage equal the oracle's conv2d / depthwise_conv2d path of the subsampling
    (conv_subsampling's stages, with the checkpoint's [C, 1, 3, 3] weights read as [C][9])."""
    p = "encoder_.subsampling_."
    W = tiny.W
    Cn = W[p + "conv1_.weight"].shape[0]
    rng = np.random.default_rng(5)
    for F in (1, 2, 5, 16, 17, 64):
        feats = feat_rows(rng, F, tiny.ocfg.mel_bins)
        _, st = O.conv_subsampling(W, feats, tiny.ocfg, return_stages=True)
        w = (W[p + "conv1_.weight"].reshape(Cn, 9), W[p + "conv1_.bias"], W[p + "dw1_.weight"].reshape(Cn, 9), W[p + "dw1_.bias"])
        y, bd = ref_conv1_dw1(feats, *w)
        want = st["dw1"].transpose(1, 2, 0).reshape(-1, Cn)
        assert ratio(want, y, bd + 1e-6 * np.abs(y)) <= 1.0, F
        d2 = O.depthwise_conv2d(st["dw1"], W[p + "dw2_.weight"], W[p + "dw2_.bias"], 2, 1)
        yd, bdd = ref_dw(st["dw1"].transpose(1, 2, 0), W[p + "dw2_.weight"].reshape(Cn, 9).T.copy(), W[p + "dw2_.bias"])
        assert ratio(d2.transpose(1, 2, 0).reshape(-1, Cn), yd, bdd + 1e-6 * np.abs(yd)) <= 1.0, F


def test_frontend_helpers():
    assert [cl(n) for n in (1, 2, 3, 4, 5, 1001)] == [1, 1, 2, 2, 3, 501]
    assert list(reflect(np.array([-5, -1, 0, 3, 4, 9]), 4)) == [1, 1, 0, 3, 2, 3]
    assert hann()[0] == 0 and hann()[199] == hann()[200] and hann(periodic=True)[200] == 1
    assert sum(b - a for a, b in chunks(15)) == 15 and min(b - a for a, b in chunks(15)) == 0
