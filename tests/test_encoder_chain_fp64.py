"""The offline encoder (pk_engine::run_subsample_tail and run_encoder) against float64, one residual sub-block at a time.

The kernel files (test_kernels_fp64.py, test_frontend_fp64.py) check each kernel alone.  This file checks how the engine
wires them: which buffer and which planes each GEMM reads, each epilogue's ldo, alpha and residual, which LayerNorm weights
go with which GEMM, the position table and the Tmax it is indexed with, the BatchNorm fold, the GLU interleave and the
choice between the few-row, wgmma and cluster GEMMs.

Taps: x_0 is the subsampling output (Engine.encode(taps=True)); x_n is the fp32 residual stream after n residual
sub-blocks (PK_DEBUG_SUBBLOCKS=n), four per layer: ffn1, attention, conv, ffn2 + final_norm_.  Sub-block n is computed in
float64 from the device's own x_{n-1} and the raw safetensors weights (not the engine's folded, interleaved or split
copies), so errors do not compound and each bound stays that of one sub-block.  Sub-block 0 starts from the features;
the CTC head starts from the device's encoder output.

Bounds compose the kernel bounds of the kernel files, with their constants.  Every intermediate is a pair (float64 value,
per-element bound e):
  operands     a GEMM operand stored as bf16 hi + lo planes adds 2^-16 (|y| + e) (hi only: 2^-8; fp32: 0).
  LayerNorm    ref_layernorm(x, w, b, e_in) with e_in = 0 on the device's own x (for final_norm_: the residual's bound).
  GEMM         ref_gemm(A, ..., e_in = e_A): e_A . |W|^T plus the kernel's own term on |A| + e_A; the epilogue carries e
               through (SiLU 1.1-Lipschitz + fast_sigmoid, GLU e_a + 0.25 |a| e_g, ReLU 1-Lipschitz, RESID |alpha| e).
  attention    ref_attention(..., e_qkv, e_pp): the score of query row i moves by <= D_i = max_j (|e_q|.|k_j| + |qu|.e_k +
               |e_q|.|PP_ij| + |qv|.e_PP) / sqrt(hd); ctx by <= 2 D_i sum_j p_ij |V_jc| + sum_j p_ij e_V,jc, plus the
               kernel's term.  The kernel term already covers the bf16 split of k, v and PP (the kernel test feeds fp32
               values and splits them as the QKV epilogue and the load-time split do), so it is not added twice.
  position     PP = emb . Wpos^T, built at load by launch_gemm_simt over Tmax (row p + Tmax - 1 <-> position p): ref_gemm
               in fp32 mode (2 d u |emb|.|Wpos|^T), with emb computed on the host in fp32 as the engine does; a libm that
               rounds sinf / cosf / expf one ulp differently moves emb by <= 2 u (1 + |angle|), carried as e_in.
  dwconv       ref_dwconv(g, folded w, folded b, e_in = e_g, w_rel = 2 u): 1.1 sum_taps |w| e_g plus the fold's rounding
               (the engine folds BatchNorm in double and rounds each weight and bias once to fp32: <= u; 2 u is kept).
  subsampling  ref_conv1_dw1 -> planes -> conv2 (RELU_F32) -> ref_dw(e_in) -> planes -> conv3 (RELU_ACT) -> planes -> proj
               (BIAS_F32, K = C f3n in the reference's channel-major order).
  CTC head     log_softmax(enc W^T + b) with enc stored as planes: |d log p| <= 2 max_v |d logit_v| + ref_ctc's term.
C_CHAIN: every propagated term above is first order.  What it drops are products of two bounds (e.g. the e_a e_g term of
GLU, e^(2D) - 1 against 2D in the softmax, the LayerNorm's 1/s taken at the reference), each a relative correction no larger
than the largest relative bound in the chain: below 2^-6 even in bf16x1 and far below in the other modes.  A factor 2 on
each sub-block's composed bound covers them with room to spare, as the kernel files' constants of 2 do; it is not fitted.

Coverage (synthetic weights from synth.make_weights; Tmax = 188, above every batch's longest utterance):
  width                 shape                              (a) one utterance, M <= 128   (b) ragged, M > 128
  tiny                  d 128, 2 heads, hd 64              T = 100 (few-row GEMM)         T = 1, 63, 65, 127, 129
  110m-width, 3 layers  d 512, 8 heads, ff 2048, mel 80    as tiny                        as tiny
  600m-width, 2 layers  d 1024, hd 128, ff 4096, mel 128   as tiny                        as tiny (staged-Q attention)
Each batch in bf16x3, bf16x1 and fp32; for tiny and 110m-width also PK_GEMM_CLUSTER=2 and 4 on (b)
and PK_ATTN_TC=0 (fp32 attention with a BIAS_F32 QKV) on (b), in bf16x3.  Bitwise engine checks: a stop run twice gives
the same bytes, the layers tap of layer i equals stop 4 (i + 1), every row of the batch is finite.

Norm-wise check (bf16x3).  The element-wise bound is a worst case: it adds |e_A|.|W| over K terms where rounding errors add
like a random walk, and in the attention the score bound sums hd such terms before the softmax.  A GEMM run with hi-only
operands moves a sub-block output by about 2^-9 sqrt(K) per element, far inside that bound: measured on the CPU (110m-width),
hi-only fc1 / fc2 / pw1 / pw2 reach 0.02 - 0.04 of it and qkv / out 0.001, and the position table indexed with the
wrong Tmax 0.14.  So each bf16x3 sub-block is also held to C_LO rms(x_n - ref) <= the smallest rms move of its output when one
of its GEMMs runs hi only (ref computed with that GEMM's operands rounded to bf16).  bf16x3 keeps 3 * 2^-16 of each
product where hi only keeps 2^-8, and every other term (planes 2^-16, fast_sigmoid 2^-20, fp32 sums) is smaller still,
so a correct engine sits one to two orders of magnitude below that move; C_LO = 4 leaves that margin wide and rejects a
GEMM whose A or W operand lost its lo plane (half the hi-only move or more).
Mutations (110m-width, bf16x3; each must fail the element-wise or the norm-wise check against the device output): fc1 /
fc2 / qkv / out / pw1 / pw2 with hi-only operands and the position table indexed with the batch's longest T instead of
Tmax (norm-wise); FFN alpha 1, the neighbouring layer's LayerNorm weights, ffn2 without final_norm_, the BatchNorm left
unfolded, the residual taken from LN(x) (both).
"""
from __future__ import annotations

import dataclasses
import math
import os

import numpy as np
import pytest
from test_frontend_fp64 import ref_conv1_dw1, ref_dw
from test_kernels_fp64 import (EPI, MATH_F32, MATH_X1, MATH_X3, U, ratio, ref_attention, ref_ctc, ref_dwconv, ref_gemm,
                               ref_layernorm, report)

gpu = pytest.mark.gpu

C_CHAIN = 2.0
C_LO = 4.0
STORE = {MATH_X3: 2.0 ** -16, MATH_X1: 2.0 ** -8, MATH_F32: 0.0}
KINDS = ("ffn1", "attn", "conv", "ffn2")
GEMMS = {"ffn1": ("fc1", "fc2"), "attn": ("qkv", "out"), "conv": ("pw1", "pw2"), "ffn2": ("fc1", "fc2")}
MAX_SAMPLES = 240000                 # Fmax 1501, Tmax 188
LENS_A = [100]
LENS_B = [65, 1, 129, 63, 127]       # T = 1 and both sides of 64 and 128; M = 385
# the mutations the element-wise bound rejects by itself (the rest need the norm-wise check, see the module docstring)
ELEMENTWISE_REJECTS = ("alpha", "ln_neighbour", "no_final_norm", "bn_unfolded", "resid_ln")
MUTATIONS = ("fc1", "fc2", "qkv", "out", "pw1", "pw2", "alpha", "ln_neighbour", "no_final_norm", "tmax", "bn_unfolded",
             "resid_ln")


def rms(a):
    return float(np.sqrt(np.mean(np.square(a, dtype=np.float64))))


def lo_ratio(R, n, x_prev, off, got, ref, base=None):
    """bf16x3: C_LO rms(got - ref) / the smallest rms move of sub-block n's output (base: the unmutated reference, default
    ref) when one of its GEMMs runs hi only"""
    base = ref if base is None else base
    dev = min(rms(R.sub_block(n, x_prev, off, g)[0] - base) for g in GEMMS[KINDS[(n - 1) % 4]])
    return C_LO * rms(got - ref) / dev


def store(y, e, mode):
    """the bound of a value held as a GEMM operand in `mode`'s form"""
    return e + STORE[mode] * (np.abs(y) + e)


def frames_for(T):
    return 2 if T == 1 else 8 * T - 3              # ceil(F / 8) = T


# ----------------------------------------------------------------------------------------------------------- references
class Ref:
    """float64 sub-blocks of one model (raw weights W, oracle config ocfg) in one math mode."""

    def __init__(self, W, ocfg, mode, tc_attn, tmax):
        self.W, self.c, self.mode, self.tc, self.tmax = W, ocfg, mode, tc_attn, tmax
        self.d, self.H = ocfg.d_model, ocfg.n_heads
        self._pp = {}

    def p(self, i):
        return f"encoder_.layers_.{i}."

    def ln(self, x, pre, i, mut, e_in=None):
        """LayerNorm `pre` of layer i (mutation: the neighbouring layer's weights)"""
        j = (i + 1) % self.c.n_layers if mut == "ln_neighbour" else i
        return ref_layernorm(x, self.W[self.p(j) + pre + "weight"], self.W[self.p(j) + pre + "bias"], e_in)

    def ffn(self, x, i, f, mut=None):
        W, m, q = self.W, self.mode, self.p(i) + ("ffn1_." if f == 0 else "ffn2_.")
        h, eh = self.ln(x, ("ffn1_." if f == 0 else "ffn2_.") + "norm_.", i, mut)
        eh = store(h, eh, m)
        a, ea = ref_gemm(h, W[q + "fc1_.weight"], W[q + "fc1_.bias"], None, EPI["SILU_ACT"], 1.0, m, Ahi_only=mut == "fc1", e_in=eh)
        ea = store(a, ea, m)
        r = self.ln(x, ("ffn1_." if f == 0 else "ffn2_.") + "norm_.", i, None)[0] if mut == "resid_ln" else x
        y, ey = ref_gemm(a, W[q + "fc2_.weight"], W[q + "fc2_.bias"], r, EPI["RESID_F32"], 1.0 if mut == "alpha" else 0.5, m,
                         Ahi_only=mut == "fc2", e_in=ea)
        if f == 1 and mut != "no_final_norm":
            y, ey = ref_layernorm(y, W[self.p(i) + "final_norm_.weight"], W[self.p(i) + "final_norm_.bias"], ey)
        return y, ey

    def pos_table(self, i):
        """PP [2 Tmax - 1, d] as the engine builds it at load, and its bound"""
        if i not in self._pp:
            d, T = self.d, self.tmax
            pos = np.arange(2 * T - 1, dtype=np.float32) - np.float32(T - 1)
            c = np.float32(-np.float32(np.log(np.float32(10000.0)))) / np.float32(d)
            div = np.exp((np.arange(0, d, 2, dtype=np.float32) * c).astype(np.float64)).astype(np.float32)
            ang = (pos[:, None] * div[None, :]).astype(np.float32).astype(np.float64)
            emb = np.zeros((2 * T - 1, d))
            emb[:, 0::2] = np.sin(ang).astype(np.float32)
            emb[:, 1::2] = np.cos(ang).astype(np.float32)
            e_emb = np.repeat(2 * U * (1 + np.abs(ang)), 2, axis=1)
            self._pp[i] = ref_gemm(emb, self.W[self.p(i) + "attn_.pos_proj_.weight"], None, None, EPI["BIAS_F32"], 1.0, MATH_F32,
                                   e_in=e_emb)
        return self._pp[i]

    def attn(self, x, i, off, mut=None):
        W, m, d, q = self.W, self.mode, self.d, self.p(i) + "attn_."
        h, eh = self.ln(x, "attn_.norm_.", i, mut)
        eh = store(h, eh, m)
        Wqkv = np.concatenate([W[q + f"mha_.{n}_proj.weight"] for n in "qkv"])
        bqkv = np.concatenate([W[q + f"mha_.{n}_proj.bias"] for n in "qkv"])
        qkv, eq = ref_gemm(h, Wqkv, bqkv, None, EPI["BIAS_F32"], 1.0, m, Ahi_only=mut == "qkv", e_in=eh)
        pp, epp = self.pos_table(i)
        lens = np.diff(off)
        tm = int(lens.max()) if mut == "tmax" else self.tmax
        ctx, ec = ref_attention(qkv, pp, W[q + "pos_bias_u_"].reshape(d), W[q + "pos_bias_v_"].reshape(d), off, len(lens), d, self.H,
                                tm, m, 1 if self.tc else 0, e_qkv=eq, e_pp=epp)
        ec = store(ctx, ec, m)
        r = h if mut == "resid_ln" else x
        return ref_gemm(ctx, W[q + "mha_.out_proj.weight"], W[q + "mha_.out_proj.bias"], r, EPI["RESID_F32"], 1.0, m,
                        Ahi_only=mut == "out", e_in=ec)

    def conv(self, x, i, off, mut=None):
        W, m, d, q = self.W, self.mode, self.d, self.p(i) + "conv_."
        h, eh = self.ln(x, "conv_.norm_.", i, mut)
        eh = store(h, eh, m)
        w1, b1 = W[q + "pointwise_conv1_.weight"][:, :, 0], W[q + "pointwise_conv1_.bias"]
        wg, bg = np.empty_like(w1), np.empty_like(b1)           # GLU pairs channel j with j + d: adjacent columns
        wg[0::2], wg[1::2], bg[0::2], bg[1::2] = w1[:d], w1[d:], b1[:d], b1[d:]
        g, eg = ref_gemm(h, wg, bg, None, EPI["GLU_F32"], 1.0, m, Ahi_only=mut == "pw1", e_in=eh)
        w, b = W[q + "depthwise_conv_.weight"][:, 0, :].astype(np.float64), W[q + "depthwise_conv_.bias"].astype(np.float64)
        if mut != "bn_unfolded":
            sc = W[q + "batch_norm_.weight"] / np.sqrt(W[q + "batch_norm_.running_var"].astype(np.float64) + 1e-5)
            w, b = w * sc[:, None], (b - W[q + "batch_norm_.running_mean"]) * sc + W[q + "batch_norm_.bias"]
        cv, ev = ref_dwconv(g, w.T, b, off, e_in=eg, w_rel=2 * U)
        ev = store(cv, ev, m)
        r = h if mut == "resid_ln" else x
        return ref_gemm(cv, W[q + "pointwise_conv2_.weight"][:, :, 0], W[q + "pointwise_conv2_.bias"], r, EPI["RESID_F32"], 1.0, m,
                        Ahi_only=mut == "pw2", e_in=ev)

    def sub_block(self, n, x, off, mut=None):
        """sub-block n >= 1 on x_{n-1} -> (x_n, bound)"""
        i, k = divmod(n - 1, 4)
        if k == 1:
            y, e = self.attn(x, i, off, mut)
        elif k == 2:
            y, e = self.conv(x, i, off, mut)
        else:
            y, e = self.ffn(x, i, k // 3, mut)
        return y, C_CHAIN * e

    def subsampling(self, feats):
        """conv1 .. proj of each utterance -> (x_0 rows, bound)"""
        W, m, Cn = self.W, self.mode, self.c.sub_channels
        s = "encoder_.subsampling_."
        w = lambda n: W[s + n]                                          # noqa: E731
        ys, es = [], []
        for f in feats:
            y, e = ref_conv1_dw1(f, w("conv1_.weight").reshape(Cn, 9), w("conv1_.bias"), w("dw1_.weight").reshape(Cn, 9), w("dw1_.bias"))
            t2 = -(-f.shape[0] // 4)
            f2 = y.shape[0] // t2
            y, e = ref_gemm(y, w("conv2_.weight")[:, :, 0, 0], w("conv2_.bias"), None, EPI["RELU_F32"], 1.0, m, e_in=store(y, e, m))
            y, e = ref_dw(y.reshape(t2, f2, Cn), w("dw2_.weight").reshape(Cn, 9).T.copy(), w("dw2_.bias"), e_in=e.reshape(t2, f2, Cn))
            y, e = ref_gemm(y, w("conv3_.weight")[:, :, 0, 0], w("conv3_.bias"), None, EPI["RELU_ACT"], 1.0, m, e_in=store(y, e, m))
            e = store(y, e, m)
            T = -(-t2 // 2)
            flat = lambda a: a.reshape(T, -1, Cn).transpose(0, 2, 1).reshape(T, -1)      # noqa: E731  (c, f) channel-major
            y, e = ref_gemm(flat(y), w("proj_.weight"), w("proj_.bias"), None, EPI["BIAS_F32"], 1.0, m, e_in=flat(e))
            ys.append(y)
            es.append(e)
        return np.concatenate(ys), C_CHAIN * np.concatenate(es)

    def ctc(self, enc):
        """log-probs of the CTC head on a host encoder output (staged as operand planes) -> (value, bound)"""
        W, m = self.W, self.mode
        lg, el = ref_gemm(enc, W["ctc_decoder_.proj_.weight"][:, :, 0], W["ctc_decoder_.proj_.bias"], None, EPI["BIAS_F32"], 1.0, m,
                          e_in=STORE[m] * np.abs(enc.astype(np.float64)))
        _, _, lp, _, blp = ref_ctc(lg)
        return lp, C_CHAIN * (blp + 2 * el.max(axis=1, keepdims=True))


# ----------------------------------------------------------------------------------------------------------- models
WIDTHS = {   # name: (oracle config factory, engine config factory, n_layers, weight seed)
    "tiny": ("make_tiny_config", "make_tiny_config", 2, 3),
    "110m": ("make_110m_config", "make_110m_config", 3, 0),
    "600m": ("make_tdt_600m_config", "make_tdt_600m_config", 2, 0),
}


class Width:
    def __init__(self, name, tmpdir, pkg, O, synth):
        of, ef, nl, seed = WIDTHS[name]
        self.name = name
        self.ocfg = dataclasses.replace(getattr(O, of)(), n_layers=nl)
        self.ecfg = getattr(pkg, ef)(n_layers=nl, max_batch=8, max_samples=MAX_SAMPLES)
        self.W = synth.make_weights(self.ocfg, seed=seed)
        self.path = os.path.join(tmpdir, f"{name}.safetensors")
        synth.save_safetensors(self.path, self.W)


@pytest.fixture(scope="module")
def widths(tmp_path_factory, pkg, O, synth):
    d = str(tmp_path_factory.mktemp("chain"))
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = Width(name, d, pkg, O, synth)
        return cache[name]
    return get


def batch_feats(mel, lens, seed):
    rng = np.random.default_rng(seed)
    return [rng.normal(0, 1, (frames_for(T), mel)).astype(np.float32) for T in lens]


def offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


# ----------------------------------------------------------------------------------------------------------- device runs
def device_states(pkg, e, feats, n_layers, monkeypatch):
    """[x_0 .. x_{4 L}] of the batch, with the engine-level bitwise checks"""
    monkeypatch.delenv("PK_DEBUG_SUBBLOCKS", raising=False)
    encs, subs, lays = e.encode(feats, taps=True)
    xs = [np.concatenate(subs)]
    lay = np.concatenate(lays, axis=1)
    for n in range(1, 4 * n_layers + 1):
        monkeypatch.setenv("PK_DEBUG_SUBBLOCKS", str(n))
        xs.append(np.concatenate(e.encode(feats)))
        if n in (1, 4 * n_layers - 1):
            again = np.concatenate(e.encode(feats))
            assert again.tobytes() == xs[-1].tobytes(), f"stop {n} run twice differs"
    monkeypatch.delenv("PK_DEBUG_SUBBLOCKS")
    for i in range(n_layers):
        assert lay[i].tobytes() == xs[4 * (i + 1)].tobytes(), f"layers tap {i} != stop {4 * (i + 1)}"
    assert np.concatenate(encs).tobytes() == xs[-1].tobytes()
    for n, x in enumerate(xs):
        assert np.all(np.isfinite(x)), f"x_{n} has a row that was not written"
    return xs


MATH = {"x3": MATH_X3, "x1": MATH_X1, "f32": MATH_F32}
# (width, variant, math, env, batches)
RUNS = [(w, m, m, {}, ("a", "b")) for w in WIDTHS for m in MATH]
RUNS += [(w, f"cluster{c}", "x3", {"PK_GEMM_CLUSTER": str(c)}, ("b",)) for w in ("tiny", "110m") for c in (2, 4)]
RUNS += [(w, "attn_tc0", "x3", {"PK_ATTN_TC": "0"}, ("b",)) for w in ("tiny", "110m")]


def make_engine(pkg, wd, mode, env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    e = pkg.Engine(dataclasses.replace(wd.ecfg, math=int(mode)), wd.path, 0)
    for k in env:
        monkeypatch.delenv(k)
    return e


@gpu
@pytest.mark.parametrize("run", RUNS, ids=lambda r: f"{r[0]}-{r[1]}")
def test_encoder_chain_against_fp64(pkg, widths, monkeypatch, run):
    name, variant, mname, env, batches = run
    wd, mode = widths(name), MATH[mname]
    e = make_engine(pkg, wd, mode, env, monkeypatch)
    tc = env.get("PK_ATTN_TC") != "0" and mode != MATH_F32
    R = Ref(wd.W, wd.ocfg, mode, tc, e.Tmax)
    assert e.Tmax > max(LENS_B)
    worst = {}
    for b in batches:
        lens = LENS_A if b == "a" else LENS_B
        feats = batch_feats(wd.ocfg.mel_bins, lens, 17 + len(lens))
        off = offsets(lens)
        xs = device_states(pkg, e, feats, wd.ocfg.n_layers, monkeypatch)
        w = {"sub": ratio(xs[0], *R.subsampling(feats))}
        for n in range(1, len(xs)):
            k = KINDS[(n - 1) % 4]
            ref, bd = R.sub_block(n, xs[n - 1], off)
            w[k] = max(w.get(k, 0.0), ratio(xs[n], ref, bd))
            if mode == MATH_X3:
                w[k + " rms"] = max(w.get(k + " rms", 0.0), lo_ratio(R, n, xs[n - 1], off, xs[n], ref))
        if wd.ocfg.has_ctc:
            enc = xs[-1]
            for u in range(len(lens)):
                rows = slice(int(off[u]), int(off[u + 1]))
                got = e.ctc_logprobs(enc[rows])
                w["ctc"] = max(w.get("ctc", 0.0), ratio(got, *R.ctc(enc[rows])))
        for k, r in w.items():
            report(f"chain {name} {variant} ({b}) {k}", r)
            worst[(b, k)] = r
    e.close()
    bad = {k: r for k, r in worst.items() if not r <= 1.0}
    assert not bad, bad


def mutation_ratios(R, xs, off, cmp):
    """the largest err / bound of each mutated reference over the sub-blocks it changes, against cmp[n] (x_n)"""
    base = [None] + [R.sub_block(n, xs[n - 1], off) for n in range(1, len(xs))]
    out = {}
    for mut in MUTATIONS:
        kinds = {"fc1": (0, 3), "fc2": (0, 3), "alpha": (0, 3), "resid_ln": (0, 1, 2, 3), "ln_neighbour": (0, 1, 2, 3),
                 "no_final_norm": (3,), "qkv": (1,), "out": (1,), "tmax": (1,), "pw1": (2,), "pw2": (2,), "bn_unfolded": (2,)}[mut]
        r = [0.0, 0.0]
        for n in range(1, len(xs)):
            if (n - 1) % 4 in kinds:
                ym, _ = R.sub_block(n, xs[n - 1], off, mut)
                r = [max(r[0], ratio(cmp[n], ym, base[n][1])), max(r[1], lo_ratio(R, n, xs[n - 1], off, cmp[n], ym, base[n][0]))]
        out[mut] = tuple(r)
    return out


@gpu
def test_encoder_chain_bound_rejects_mutations(pkg, widths, monkeypatch):
    wd = widths("110m")
    e = make_engine(pkg, wd, MATH_X3, {}, monkeypatch)
    off = offsets(LENS_B)
    feats = batch_feats(wd.ocfg.mel_bins, LENS_B, 17 + len(LENS_B))
    xs = device_states(pkg, e, feats, wd.ocfg.n_layers, monkeypatch)
    R = Ref(wd.W, wd.ocfg, MATH_X3, True, e.Tmax)
    e.close()
    rs = mutation_ratios(R, xs, off, xs)
    for mut, (r, q) in rs.items():
        report(f"chain 110m mutation {mut}", r)
        report(f"chain 110m mutation {mut} rms", q)
    assert all(max(r) > 1.0 for r in rs.values()), rs
    assert all(rs[m][0] > 1.0 for m in ELEMENTWISE_REJECTS), rs


# ----------------------------------------------------------------------------------------------------------- CPU: the references, pinned
def oracle_states(O, W, ocfg, feats):
    """the oracle's own x_0 .. x_{4 L} of one utterance (its fp32 sub-blocks)"""
    x = O.conv_subsampling(W, feats, ocfg)
    pos = O.sinusoidal_position_embedding(x.shape[0], x.shape[1])
    xs = [x]
    for i in range(ocfg.n_layers):
        p = f"encoder_.layers_.{i}."
        xs.append(O.feed_forward(W, p + "ffn1_.", xs[-1]))
        xs.append(O.conformer_attention(W, p + "attn_.", xs[-1], pos, ocfg))
        xs.append(O.conformer_conv(W, p + "conv_.", xs[-1], ocfg))
        xs.append(O.layer_norm(O.feed_forward(W, p + "ffn2_.", xs[-1]), W[p + "final_norm_.weight"], W[p + "final_norm_.bias"]))
    return xs


@pytest.mark.parametrize("name", ["tiny", "110m"])
def test_chain_reference_matches_oracle_teacher_forced(O, widths, name):
    """Each float64 sub-block, fed the oracle's own x_{n-1}, gives the oracle's x_n within the fp32 bound (the oracle is an
    fp32 restatement of the same model); x_4i are the oracle's encoder_forward layers."""
    wd = widths(name)
    T = 50
    feats = batch_feats(wd.ocfg.mel_bins, [T], 5)
    xs = oracle_states(O, wd.W, wd.ocfg, feats[0])
    enc, sub, lay = O.encoder_forward(wd.W, feats[0], wd.ocfg, return_layers=True)
    for i in range(wd.ocfg.n_layers):
        assert np.array_equal(lay[i], xs[4 * (i + 1)])
    R = Ref(wd.W, wd.ocfg, MATH_F32, False, T + 37)        # the position table over a longer Tmax: same positions
    off = offsets([T])
    assert ratio(xs[0], *R.subsampling(feats)) <= 1.0
    for n in range(1, len(xs)):
        r = ratio(xs[n], *R.sub_block(n, xs[n - 1], off))
        assert r <= 1.0, (n, r)
    if wd.ocfg.has_ctc:
        assert ratio(O.ctc_log_probs(wd.W, enc), *R.ctc(enc)) <= 1.0


def test_chain_mutations_exceed_the_bound(O, widths):
    """On the CPU: every mutation moves the float64 reference, fed the oracle's own states, by more than the bf16x3 bound."""
    wd = widths("110m")
    lens = [65, 40]
    feats = batch_feats(wd.ocfg.mel_bins, lens, 9)
    per = [oracle_states(O, wd.W, wd.ocfg, f) for f in feats]
    xs = [np.concatenate([p[n] for p in per]) for n in range(len(per[0]))]
    R = Ref(wd.W, wd.ocfg, MATH_X3, True, 188)
    off = offsets(lens)
    refs = [None] + [R.sub_block(n, xs[n - 1], off)[0] for n in range(1, len(xs))]
    rs = mutation_ratios(R, xs, off, refs)
    for mut, (r, q) in rs.items():
        report(f"chain reference mutation {mut}", r)
        report(f"chain reference mutation {mut} rms", q)
    assert all(max(r) > 1.0 for r in rs.values()), rs
    assert all(rs[m][0] > 1.0 for m in ELEMENTWISE_REJECTS), rs


def test_chain_helpers():
    assert [-(-frames_for(T) // 8) for T in (1, 63, 64, 65, 128, 129)] == [1, 63, 64, 65, 128, 129]
    assert store(np.array([2.0]), np.array([0.0]), MATH_X1)[0] == 2.0 ** -7
    assert math.isclose(C_CHAIN, 2.0)
