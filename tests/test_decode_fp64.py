"""The TDT / RNN-T decode kernel (csrc/tdt.cu) against a float64 replay of the greedy decode, through pk_kernel_tdt_decode.

The hook takes the decode's inputs in the reference's layouts (EP = enc_proj(enc) + bias and G0 = W_ih0 . E + b_ih0 are GEMM
outputs, tested elsewhere, so they are taken as given), builds TdtParams as the engine does and returns every output between
0xFF guard bands, plus the last step's LSTM h planes, joint hidden z, arg-max keys and label log-sum-exp.  `ref_decode` replays
the same decode in float64 on the exact fp32 inputs: lock step over the batch like the kernel (every utterance is evaluated
at every step, idle ones from their committed state), LSTM cell (gate order i, f, g, o), z = relu(EP[t] + W_p h), both heads,
first-maximum arg-max (index 0 when nothing is above -inf) and the TDT / RNN-T state rules: blank reverts the state and
advances max(skip, 1); a symbol commits it and advances skip; RNN-T advances after max_sym symbols on a frame; the token
capacity stops an utterance (overflow); with `carry`, frames are numbered from frame_base and the end frame is not clamped.

Along its own path it propagates a per-element error bound (u = 2^-24):
  products    y = W x with the kernel's x given as bf16 hi + lo of its fp32 value x^ (|x^ - x| <= e_x):
              hi.hi + hi.lo + lo.hi: C_X3 2^-16 |W| (|x| + e_x) (as test_kernels_fp64.py), storing x as hi + lo:
              2^-16 |W| (|x| + e_x), fp32 accumulation (mma chains of K / 16 steps x 3, then the CL partials): (3 K / 16 + 8) u
              |W| (|x| + e_x), and the propagated error |W| e_x.
  epilogues   + G0[token] / b_ih / EP / b_out and the partial-sum adds in fp32: 4 u (|W| (|x| + e_x) + |pre|).
  cell        sigmoidf_ = 1 / (1 + expf(-x)) (expf <= 2 ulp, a true division): 8 u sigma + e_x / 4 (sigma' <= 1/4);
              tanhf (<= 2 ulp): 4 u |tanh| + e_x (tanh' <= 1);  c' = sf c + si tg: (sf + e_sf) e_c + |c| e_sf + (si + e_si)
              e_tg + |tg| e_si + 4 u (|sf c| + |si tg|);  h' = so tanh(c'): (so + e_so) e_tc + |tc| e_so + 2 u |h'|.
  joint       ReLU is 1-Lipschitz: e_z = e(EP + W_p h').
  across steps the bound vectors of h and c are carried with the state (and reverted with it), so a long decode has its own
              growing bound.
  log-sum-exp 1-Lipschitz in the max norm: max e_l over the labels, plus the fp32 online sums of each CTA (<= ceil(OPC/CL) + 2
              terms, 8 u each, relative) -- the partials are combined in double by the hook.
  confidence  exp(l_max - lse) of the kernel's logits: conf (exp(e_l[max] + max e_l + rel) - 1), rel = 8 u (ceil(OPC/CL) + 16)
              for the fp32 combination of up to 256 partials in finalize_conf.
Outputs stored as bf16 hi + lo are compared with check_planes (which adds 2^-16 of the value).  Token ids, timestamps,
overflow and the step count must be EQUAL: every decision on the reference path has a top-2 gap (labels, and durations for
TDT) larger than 4x the propagated logit bound, which the CPU tests check for every case, so a seed that would make the
comparison a coin toss fails here, without a GPU.  Exact ties are allowed only where they are exact in the kernel too (rows
with zero weights and equal biases).
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import functools
import math

import numpy as np
import pytest

import rnnt_oracle as RO
from test_kernels_fp64 import C_X3, U, bf16_rn, check_planes, first_argmax64, ratio, report, split

gpu = pytest.mark.gpu

# ----------------------------------------------------------------------------------------------------------- geometry
# Mirror of tdt_smem_bytes / tdt_geom (csrc/tdt.cu): which weights stay in shared memory for nc clusters of CL CTAs.
RG, RLD, MYMAX, BCH = 80, 68, 40, 64
BUDGET = 225 * 1024 // 4


def plan(P, J, V, D, L, Bpad, nc, CL, no_stage=False):
    cd = lambda a, b: -(-a // b)  # noqa: E731
    UPC, JPC, OPC = cd(P, nc), cd(J, nc), cd(V + D, nc)
    KSP, KSJ = P // CL, J // CL
    MU = cd(UPC, CL)
    xrows = min(BCH, Bpad)
    fixed = RG * RLD + MYMAX * BCH + xrows * (max(KSP, KSJ) + 8) + L * 2 * MU * Bpad + (8 if D == 0 else 7) * Bpad
    hh, ih = L * UPC * 4 * (KSP + 4), (L - 1) * UPC * 4 * (KSP + 4)
    wp, wo = JPC * (KSP + 4), OPC * (KSJ + 4)
    total = fixed + hh + wp
    wih = ih == 0 or total + ih <= BUDGET
    out = total + (ih if wih else 0) + wo <= BUDGET
    rows = 0
    if not out:
        r = max(BUDGET - total, 0) // (KSJ + 4)
        rows = next((x for x in (80, 64, 48, 32, 16) if r >= x), 0)
        total += rows * (KSJ + 4)
        wih = ih == 0 or total + ih <= BUDGET
    if no_stage:
        rows = 0
    nU0 = min(UPC, P)
    staged = (not wih) and L > 1 and rows >= nU0 * 4 and nU0 <= RG // 4 and KSP == KSJ
    return dict(cl=CL, upc=UPC, opc=OPC, out_in_smem=int(out), wih_in_smem=int(wih), staged_ih=int(staged), wstage_rows=rows)


def fits(P, J, CL):
    return P % (16 * CL) == 0 and J % (16 * CL) == 0


# ----------------------------------------------------------------------------------------------------------- cases
@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    P: int = 640
    J: int = 640
    V: int = 1025
    durations: tuple = (0, 1, 2, 3, 4)      # () = RNN-T
    L: int = 1
    max_sym: int = 10
    lens: tuple = (7,)
    cap: int = 0                            # 0: 3 T'max + 8 (TDT), max_sym T'max + 8 (RNN-T), as the engine sizes it
    max_steps: int = 0                      # 0: T'max + cap + 2, as run_tdt
    carry: bool = False
    cluster: int = 0
    max_ctas: int = 120                     # SMs the launch plans for: 30 clusters of 4 (what an H100 80GB HBM3 co-schedules,
                                            # the engine's geometry there) or 60 of 2, a fixed geometry
    no_stage: bool = False
    seed: int = 1
    blank_bias: float = 0.0
    force_label: int = -1                   # a label whose bias dominates (always emitted)
    force_dur: int = -1                     # a duration whose bias dominates
    expect: tuple = ()                      # (key, value) pairs of the geometry the launch must choose

    @property
    def D(self):
        return len(self.durations)

    @property
    def n(self):
        return len(self.lens)

    @property
    def bpad(self):
        return (self.n + 31) // 32 * 32

    @property
    def capacity(self):
        if self.cap:
            return self.cap
        T = max(self.lens)
        return (self.max_sym * T + 8) if self.D == 0 else 3 * T + 8

    @property
    def steps_limit(self):
        return self.max_steps or max(self.lens) + self.capacity + 2


def _lens(seed, n, lo=2, hi=8, extra=()):
    r = np.random.default_rng(seed)
    return tuple(int(x) for x in r.integers(lo, hi + 1, n - len(extra))) + tuple(extra)


M110 = dict(P=640, J=640, V=1025)
M600 = dict(P=640, J=640, V=8193, L=2)
RNNT = dict(P=640, J=640, V=1025, L=2, durations=())
CASES = [
    Case("110m-n1-cl4", **M110, lens=(9,), cluster=4, seed=3, expect=(("cl", 4), ("out_in_smem", 1))),
    Case("110m-n33-cl4", **M110, lens=_lens(5, 33, extra=(0, 1)), cluster=4, seed=5, expect=(("cl", 4), ("out_in_smem", 1))),
    Case("110m-n72-cl4", **M110, lens=_lens(6, 72, extra=(1,)), cluster=4, seed=9, expect=(("cl", 4), ("out_in_smem", 1))),
    Case("110m-n1-cl2", **M110, lens=(9,), cluster=2, seed=3, expect=(("cl", 2), ("out_in_smem", 1))),
    Case("110m-n33-cl2", **M110, lens=_lens(7, 33, extra=(0,)), cluster=2, seed=8, expect=(("cl", 2), ("out_in_smem", 1))),
    Case("110m-n72-cl2", **M110, lens=_lens(8, 72), cluster=2, seed=12, expect=(("cl", 2), ("out_in_smem", 1))),
    Case("600m-n16", **M600, lens=_lens(9, 16), seed=10, expect=(("cl", 4), ("out_in_smem", 0), ("wih_in_smem", 0), ("staged_ih", 0))),
    Case("600m-n72", **M600, lens=_lens(10, 72, hi=6), seed=18,
         expect=(("cl", 4), ("out_in_smem", 0), ("wih_in_smem", 0), ("staged_ih", 0))),
    Case("600m-n16-nostage", **M600, lens=_lens(9, 16), seed=10, no_stage=True,
         expect=(("cl", 4), ("out_in_smem", 0), ("wih_in_smem", 0), ("staged_ih", 0), ("wstage_rows", 0))),
    Case("600m-n72-nostage", **M600, lens=_lens(10, 72, hi=6), seed=18, no_stage=True,
         expect=(("out_in_smem", 0), ("wih_in_smem", 0), ("wstage_rows", 0))),
    # the 600m head with P = J = 576: 20 units per cluster, so the tile holds W_ih of layer 1 as well (P = 640 needs 32 clusters)
    Case("600m-P576-staged", P=576, J=576, V=8193, L=2, lens=_lens(25, 16), seed=25,
         expect=(("cl", 4), ("upc", 20), ("out_in_smem", 0), ("wih_in_smem", 0), ("staged_ih", 1), ("wstage_rows", 80))),
    Case("rnnt-ms1", **RNNT, max_sym=1, lens=_lens(11, 8), seed=11, blank_bias=-1.0, expect=(("cl", 4), ("wih_in_smem", 0))),
    Case("rnnt-ms10-forced", **RNNT, max_sym=10, lens=(3, 2, 4, 1), seed=12, force_label=17, expect=(("cl", 4),)),
    Case("rnnt-ms64", **RNNT, max_sym=64, lens=_lens(13, 6), seed=15, blank_bias=-1.0, expect=(("cl", 4),)),
    Case("upc64-L2", P=256, J=256, V=129, L=2, lens=_lens(14, 5), cluster=4, max_ctas=16, seed=14,
         expect=(("cl", 4), ("upc", 64), ("wih_in_smem", 0), ("staged_ih", 0))),
    Case("L3-wih-resident", P=384, J=384, V=257, L=3, lens=_lens(15, 6), cluster=4, max_ctas=80, seed=15,
         expect=(("cl", 4), ("upc", 20), ("wih_in_smem", 1))),
    Case("L4-wih-staged", P=384, J=384, V=4097, L=4, lens=_lens(16, 6), cluster=4, max_ctas=80, seed=16,
         expect=(("cl", 4), ("upc", 20), ("wih_in_smem", 0), ("staged_ih", 1), ("out_in_smem", 0))),
    Case("L4-wih-l2", P=384, J=384, V=257, L=4, lens=_lens(17, 6), cluster=4, max_ctas=80, seed=17,
         expect=(("cl", 4), ("wih_in_smem", 0), ("staged_ih", 0))),
    Case("P640-J384", P=640, J=384, V=1025, L=2, lens=_lens(18, 9), cluster=4, seed=20,
         expect=(("cl", 4), ("wih_in_smem", 0), ("staged_ih", 0))),
    Case("P640-J384-V8193", P=640, J=384, V=8193, L=2, lens=_lens(26, 16), cluster=4, seed=28,
         expect=(("cl", 4), ("wih_in_smem", 0), ("staged_ih", 0), ("out_in_smem", 0))),
    Case("P96", P=96, J=96, V=129, lens=_lens(19, 5), seed=19, expect=(("cl", 2),)),
    Case("capacity", **M110, lens=(5, 0, 3), cap=6, seed=20, force_label=5, force_dur=0, expect=(("cl", 4),)),
    Case("carry-tdt", **M110, durations=(1, 2, 4, 6, 8), lens=_lens(21, 6, extra=(0,)), carry=True, seed=21),
    Case("clamp-tdt", **M110, durations=(1, 2, 4, 6, 8), lens=_lens(21, 6, extra=(0,)), seed=21),
    Case("carry-rnnt", **RNNT, lens=_lens(22, 4), carry=True, seed=22, blank_bias=-1.0),
    Case("one-step-tdt", **M600, lens=(4, 3, 5), max_steps=1, carry=True, seed=23, force_label=9),
    Case("one-step-rnnt", **RNNT, lens=(4, 3), max_steps=1, carry=True, seed=24, force_label=9),
]
BY_NAME = {c.name: c for c in CASES}


def case_inputs(c: Case):
    return _inputs(c)


@functools.lru_cache(maxsize=4)
def _inputs(c: Case):
    """Seeded fp32 inputs.  The propagated bound is a worst case (|W| e_x), so the recurrent weights are contractive under it
    (row sums of |W_hh| 0.3, |W_ih| 1, |W_p| 0.5): the bound of a long decode grows, but slowly.  The rows of W_out have two
    entries and the biases a wide spread, so the logits carry little cancellation and the top-2 gaps stay clear of 4x the
    bound (the CPU tests check every decision)."""
    r = np.random.default_rng(c.seed * 1000 + c.P + c.V)
    P, J, V, D, L = c.P, c.J, c.V, c.D, c.L
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    Whh = [f(r.uniform(-1, 1, (4 * P, P)) * (0.6 / P)) for _ in range(L)]
    Wih = [None] + [f(r.uniform(-1, 1, (4 * P, P)) * (2.0 / P)) for _ in range(1, L)]
    bih = [None] + [f(r.normal(0, 0.5, 4 * P)) for _ in range(1, L)]
    G0 = f(r.normal(0, 1.0, (V, 4 * P)))
    Wp = f(r.uniform(-1, 1, (J, P)) * (1.0 / P))
    Wout = np.zeros((V + D, J))
    for row in range(V + D):
        Wout[row, r.choice(J, 2, replace=False)] = r.normal(0, 1.0, 2)
    Wout = f(Wout)
    bout = r.normal(0, 3.0, V + D)
    bout[V - 1] = bout[:V - 1].max() + c.blank_bias
    if c.force_label >= 0:
        bout[c.force_label] = 40.0
    if c.force_dur >= 0:
        bout[V + c.force_dur] = 40.0
    bout = f(bout)
    rows = sum(c.lens) + 3
    EP = f(r.normal(0, 1.0, (rows, J)))
    off = np.concatenate([[0], np.cumsum(c.lens)]).astype(np.int32)
    inp = dict(P=P, J=J, V=V, D=D, durations=tuple(c.durations), L=L, max_sym=c.max_sym, n=c.n, off=off, rows=rows, EP=EP, G0=G0,
               Whh=Whh, Wih=Wih, bih=bih, Wp=Wp, Wout=Wout, bout=bout, cap=c.capacity, max_steps=c.steps_limit, carry=c.carry)
    if c.carry:
        inp["h0"] = f(r.uniform(-0.7, 0.7, (L, c.n, P)))
        inp["c0"] = f(r.uniform(-2, 2, (L, c.n, P)))
        inp["tok0"] = r.integers(0, V - 1, c.n).astype(np.int32)
        inp["fbase"] = r.integers(1, 500, c.n).astype(np.int32)
    return inp


# ----------------------------------------------------------------------------------------------------------- float64 reference
MUTATIONS = ("gate_if", "no_revert", "no_relu", "h_hi_only", "zero_c", "unclamped", "ties_last")


def _argmax(row, last=False):
    if last:
        return len(row) - 1 - int(np.argmax(row[::-1]))
    return int(np.argmax(row))       # first maximum; an all -inf row gives 0, as the strict '>' scan from index 0


def _gap(row):
    """top-1 minus the largest value below it (exact ties excluded), or inf."""
    top = row.max()
    if not np.isfinite(top):
        return np.inf
    below = row[row < top]
    return float(top - below.max()) if below.size else np.inf


def ref_decode(inp, mut=frozenset()):
    P, J, V, D, L, n = inp["P"], inp["J"], inp["V"], inp["D"], inp["L"], inp["n"]
    rnnt, cap, carry = D == 0, inp["cap"], inp["carry"]
    off = inp["off"]
    T = np.diff(off)
    f64 = lambda a: a.astype(np.float64)  # noqa: E731
    Whh, Wih = [f64(w) for w in inp["Whh"]], [None if w is None else f64(w) for w in inp["Wih"]]
    bih = [None if b is None else f64(b) for b in inp["bih"]]
    aWhh, aWih = [np.abs(w) for w in Whh], [None if w is None else np.abs(w) for w in Wih]
    G0, Wp, Wout, bout, EP = f64(inp["G0"]), f64(inp["Wp"]), f64(inp["Wout"]), f64(inp["bout"]), f64(inp["EP"])
    aWp, aWout = np.abs(Wp), np.abs(Wout)

    def product(W, aW, x, ex):
        """W x for the rows of x, and its bound (module docstring)."""
        K = W.shape[1]
        if "h_hi_only" in mut:
            x = f64(bf16_rn(x.astype(np.float32)))
        A = (np.abs(x) + ex) @ aW.T
        return x @ W.T, ((C_X3 + 1) * 2.0 ** -16 + (3 * K / 16 + 8) * U) * A + ex @ aW.T, A

    # state planes as the kernel keeps them: h [L][2] (n, P) with bounds, c [L][2]; plane cur[b] is committed
    hp = [[np.zeros((n, P)), np.zeros((n, P))] for _ in range(L)]
    ehp = [[np.zeros((n, P)), np.zeros((n, P))] for _ in range(L)]
    cp = [[np.zeros((n, P)), np.zeros((n, P))] for _ in range(L)]
    ecp = [[np.zeros((n, P)), np.zeros((n, P))] for _ in range(L)]
    if carry:
        for l in range(L):
            hp[l][0] = f64(inp["h0"][l])
            if "zero_c" not in mut:
                cp[l][0] = f64(inp["c0"][l])
    cur = np.zeros(n, int)
    tok = np.array(inp["tok0"], int) if carry else np.full(n, V - 1)
    base = np.array(inp["fbase"], int) if carry else np.zeros(n, int)
    t = np.zeros(n, int)
    active = T > 0
    ntok, nsym, overflow = np.zeros(n, int), np.zeros(n, int), np.zeros(n, int)
    emis = [[] for _ in range(n)]
    margins = []
    idx = np.arange(n)
    step = 0
    while True:
        new_h, new_eh, new_c, new_ec = [], [], [], []
        x_in, ex_in = None, None
        for l in range(L):
            h, eh = np.stack([hp[l][cur[b]][b] for b in idx]), np.stack([ehp[l][cur[b]][b] for b in idx])
            c, ec = np.stack([cp[l][cur[b]][b] for b in idx]), np.stack([ecp[l][cur[b]][b] for b in idx])
            g, eg, A = product(Whh[l], aWhh[l], h, eh)
            if l == 0:
                pre = G0[tok]
            else:
                g2, eg2, A2 = product(Wih[l], aWih[l], x_in, ex_in)
                g, eg, A = g + g2, eg + eg2, A + A2
                pre = np.broadcast_to(bih[l], g.shape)
            eg = eg + 4 * U * (A + np.abs(pre))
            g = g + pre
            gi, gf, gg, go = (g[:, k * P:(k + 1) * P] for k in range(4))
            ei, ef, eG, eo = (eg[:, k * P:(k + 1) * P] for k in range(4))
            if "gate_if" in mut:
                gi, gf = gf, gi
            si, sf, so = (1 / (1 + np.exp(-x)) for x in (gi, gf, go))
            esi, esf, eso = (8 * U * s + 0.25 * e for s, e in ((si, ei), (sf, ef), (so, eo)))
            tg = np.tanh(gg)
            etg = 4 * U * np.abs(tg) + eG
            c2 = sf * c + si * tg
            ec2 = (sf + esf) * ec + np.abs(c) * esf + (si + esi) * etg + np.abs(tg) * esi + 4 * U * (np.abs(sf * c) + np.abs(si * tg))
            tc = np.tanh(c2)
            etc = 4 * U * np.abs(tc) + ec2
            h2 = so * tc
            eh2 = (so + eso) * etc + np.abs(tc) * eso + 2 * U * np.abs(h2)
            new_h.append(h2), new_eh.append(eh2), new_c.append(c2), new_ec.append(ec2)
            x_in, ex_in = h2, eh2
        ep = np.zeros((n, J))
        for b in idx:
            if T[b] > 0:
                ep[b] = EP[off[b] + min(t[b], T[b] - 1)]
        zp, ez, A = product(Wp, aWp, x_in, ex_in)
        ez = ez + 4 * U * (A + np.abs(ep))
        zp = zp + ep
        z = zp if "no_relu" in mut else np.maximum(zp, 0)
        lg, el, A = product(Wout, aWout, z, ez)
        with np.errstate(invalid="ignore"):
            el = el + 4 * U * (A + np.abs(bout))
        lg = lg + bout
        lab = lg[:, :V]
        with np.errstate(invalid="ignore", over="ignore"):
            mx = lab.max(axis=1, keepdims=True)
            lse = (mx + np.log(np.exp(lab - mx).sum(axis=1, keepdims=True)))[:, 0]
        fin = np.isfinite(lab)
        el_lab = np.where(fin, el[:, :V], 0).max(axis=1)
        last = dict(h=new_h, eh=new_eh, z=z, ez=ez, lg=lg, el=el, lse=lse, el_lab=el_lab, active=active.copy(),
                    new_plane=1 - cur.copy())
        for l in range(L):
            for b in idx:
                hp[l][1 - cur[b]][b], ehp[l][1 - cur[b]][b] = new_h[l][b], new_eh[l][b]
                cp[l][1 - cur[b]][b], ecp[l][1 - cur[b]][b] = new_c[l][b], new_ec[l][b]
        keys = np.full((n, 2), -1)
        for b in np.nonzero(active)[0]:
            li = _argmax(lab[b], last="ties_last" in mut)
            di = _argmax(lg[b, V:], last="ties_last" in mut) if not rnnt else -1
            keys[b] = (li if np.isfinite(lab[b]).any() else -1, di if (not rnnt and np.isfinite(lg[b, V:]).any()) else -1)
            margins.append(_gap(lab[b]) / (4 * el_lab[b]))
            if not rnnt:
                fd = np.isfinite(lg[b, V:])
                margins.append(_gap(lg[b, V:]) / (4 * np.where(fd, el[b, V:], 0).max()))
            skip = 0 if rnnt else inp["durations"][di]
            if li == V - 1:
                t[b] += max(skip, 1)
                nsym[b] = 0
                if "no_revert" in mut:
                    cur[b] ^= 1
            else:
                k = ntok[b]
                if k < cap:
                    if carry:
                        end = base[b] + t[b] + max(skip, 1) - 1
                    elif "unclamped" in mut:
                        end = t[b] + max(skip, 1) - 1
                    else:
                        end = min(t[b] + max(skip, 1) - 1, T[b] - 1)
                    conf = float(np.exp(lab[b, li] - lse[b]))
                    emis[b].append((li, base[b] + t[b], end, conf, el[b, li] + el_lab[b]))
                ntok[b] = k + 1
                tok[b] = li
                cur[b] ^= 1
                t[b] += skip
                if rnnt:
                    nsym[b] += 1
                    if nsym[b] >= inp["max_sym"]:
                        t[b] += 1
                        nsym[b] = 0
                if k + 1 >= cap:
                    active[b] = False
                    overflow[b] = 1
            if t[b] >= T[b]:
                active[b] = False
        last["keys"] = keys
        if not active.any() or step + 1 >= inp["max_steps"]:
            break
        step += 1
    if carry:            # exit: the committed h goes to plane 0
        for l in range(L):
            for b in idx:
                if cur[b] == 1:
                    hp[l][0][b], ehp[l][0][b] = hp[l][1][b], ehp[l][1][b]
    return dict(steps=step + 1, emis=emis, overflow=overflow, margins=np.array(margins), last=last, hp=hp, ehp=ehp,
                c=[np.stack([cp[l][cur[b]][b] for b in idx]) for l in range(L)],
                ec=[np.stack([ecp[l][cur[b]][b] for b in idx]) for l in range(L)], tok=tok.copy(), cur=cur.copy())


@functools.lru_cache(maxsize=4)
def _ref(c: Case, mut=frozenset()):
    return ref_decode(case_inputs(c), mut)


def case_ref(c, mut=frozenset()):
    return _ref(c, frozenset(mut))


# ----------------------------------------------------------------------------------------------------------- the hook
def _p(a, t=C.c_float):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def run_hook(pkg, inp, cluster=0, max_ctas=0, no_stage=False):
    """-> dict of every output (numpy), the guard count and the reported geometry."""
    L = pkg.load_library()
    E = pkg.engine
    n, P, J, V, D, Lh, cap = inp["n"], inp["P"], inp["J"], inp["V"], inp["D"], inp["L"], inp["cap"]
    hi = E.TdtHookIn()
    hi.P, hi.J, hi.V, hi.n_dur, hi.L, hi.max_sym = P, J, V, D, Lh, inp["max_sym"]
    for i, d in enumerate(inp["durations"]):
        hi.durations[i] = d
    keep = []                                   # numpy arrays referenced by pointer stay alive until the call returns

    def ptr(a, t=C.c_float):
        a = np.ascontiguousarray(a, np.float32 if t is C.c_float else np.int32)
        keep.append(a)
        return _p(a, t)

    hi.n_utt, hi.rows = n, inp["rows"]
    hi.row_off = ptr(inp["off"], C.c_int32)
    hi.EP, hi.G0 = ptr(inp["EP"]), ptr(inp["G0"])
    for l in range(Lh):
        hi.W_hh[l] = ptr(inp["Whh"][l])
        if l:
            hi.W_ih[l], hi.b_ih[l] = ptr(inp["Wih"][l]), ptr(inp["bih"][l])
    hi.W_p, hi.W_out, hi.b_out = ptr(inp["Wp"]), ptr(inp["Wout"]), ptr(inp["bout"])
    hi.cap, hi.max_steps, hi.carry = cap, inp["max_steps"], int(inp["carry"])
    if inp["carry"]:
        hi.h0, hi.c0 = ptr(inp["h0"]), ptr(inp["c0"])
        hi.tok0, hi.frame_base = ptr(inp["tok0"], C.c_int32), ptr(inp["fbase"], C.c_int32)
    hi.cluster, hi.max_ctas, hi.no_stage = cluster, max_ctas, int(no_stage)
    o = dict(tok=np.zeros((n, 1 + cap), np.int32), t_start=np.zeros((n, cap), np.int32), t_end=np.zeros((n, cap), np.int32),
             t_conf=np.zeros((n, cap), np.float32), overflow=np.zeros(n, np.int32), h_hi=np.zeros((Lh, 2, n, P), np.float32),
             h_lo=np.zeros((Lh, 2, n, P), np.float32), z_hi=np.zeros((n, J), np.float32), z_lo=np.zeros((n, J), np.float32),
             lab_val=np.zeros(n, np.float32), dur_val=np.zeros(n, np.float32), lab_idx=np.zeros(n, np.int32),
             dur_idx=np.zeros(n, np.int32), lse=np.zeros(n, np.float64), c_state=np.zeros((Lh, n, P), np.float32),
             tok_state=np.zeros(n, np.int32))
    ho = E.TdtHookOut()
    for k, a in o.items():
        t = {np.dtype(np.int32): C.c_int32, np.dtype(np.float32): C.c_float, np.dtype(np.float64): C.c_double}[a.dtype]
        setattr(ho, k, _p(a, t))
    gb = C.c_int64(-1)
    st = L.pk_kernel_tdt_decode(0, C.byref(hi), C.byref(ho), C.byref(gb))
    o["status"] = st
    o["guard_bad"] = gb.value
    o["steps"] = ho.steps
    o["geom"] = {k: getattr(ho, k) for k in ("grid", "cl", "upc", "opc", "out_in_smem", "wih_in_smem", "staged_ih", "wstage_rows")}
    return o


def fake_output(inp, ref, geom):
    """What a kernel that computed exactly `ref` (rounded as the kernel stores it) would return: lets the CPU tests run the
    checker on mutated references."""
    n, P, L, cap, V = inp["n"], inp["P"], inp["L"], inp["cap"], inp["V"]
    o = dict(status=0, guard_bad=0, steps=ref["steps"], geom=geom, overflow=ref["overflow"].astype(np.int32))
    o["tok"] = np.full((n, 1 + cap), -1, np.int32)
    o["t_start"], o["t_end"] = np.full((n, cap), -1, np.int32), np.full((n, cap), -1, np.int32)
    o["t_conf"] = np.full((n, cap), np.nan, np.float32)
    for b, em in enumerate(ref["emis"]):
        o["tok"][b, 0] = len(em)
        for k, e in enumerate(em):
            o["tok"][b, 1 + k], o["t_start"][b, k], o["t_end"][b, k], o["t_conf"][b, k] = e[0], e[1], e[2], e[3]
    hs = np.stack([np.stack(ref["hp"][l]) for l in range(L)]).astype(np.float32)
    o["h_hi"], o["h_lo"] = split(hs)
    o["z_hi"], o["z_lo"] = split(ref["last"]["z"].astype(np.float32))
    keys, lg = ref["last"]["keys"], ref["last"]["lg"]
    o["lab_idx"], o["dur_idx"] = keys[:, 0].astype(np.int32), keys[:, 1].astype(np.int32)
    o["lab_val"] = np.array([lg[b, k] if k >= 0 else np.nan for b, k in enumerate(keys[:, 0])], np.float32)
    o["dur_val"] = np.array([lg[b, V + k] if k >= 0 else np.nan for b, k in enumerate(keys[:, 1])], np.float32)
    o["lse"] = ref["last"]["lse"].copy()
    o["c_state"] = np.stack(ref["c"]).astype(np.float32)
    o["tok_state"] = ref["tok"].astype(np.int32)
    return o


# ----------------------------------------------------------------------------------------------------------- the checker
def check(inp, ref, got, check_values=True):
    """Compares a hook result with the float64 reference -> (failures, {output: max err/bound}).  Equality of every decode
    output, the exact written set, and each value within its bound."""
    fails, r = [], {}
    n, P, V, D, L, cap = inp["n"], inp["P"], inp["V"], inp["D"], inp["L"], inp["cap"]
    if got["status"] != 0:
        return [f"status {got['status']}"], r
    if got["guard_bad"] != 0:
        fails.append(f"guard_bad {got['guard_bad']}")
    if got["steps"] != ref["steps"]:
        fails.append(f"steps {got['steps']} != {ref['steps']}")
    if not np.array_equal(got["overflow"], ref["overflow"]):
        fails.append("overflow")
    g = got["geom"]
    nq = -(-g["opc"] // max(g["cl"], 1)) + 2
    conf_r = 0.0
    for b, em in enumerate(ref["emis"]):
        k = len(em)
        if got["tok"][b, 0] != k:
            fails.append(f"utt {b}: len {got['tok'][b, 0]} != {k}")
            continue
        want = np.array([e[:3] for e in em], np.int64).reshape(k, 3)
        if not (np.array_equal(got["tok"][b, 1:1 + k], want[:, 0]) and np.array_equal(got["t_start"][b, :k], want[:, 1]) and
                np.array_equal(got["t_end"][b, :k], want[:, 2])):
            fails.append(f"utt {b}: tokens / timestamps differ")
        if not (np.all(got["tok"][b, 1 + k:] == -1) and np.all(got["t_start"][b, k:] == -1) and np.all(got["t_end"][b, k:] == -1)
                and np.all(np.isnan(got["t_conf"][b, k:]))):
            fails.append(f"utt {b}: a slot past len was written")
        if check_values and k:
            cf = np.array([e[3] for e in em])
            bd = cf * np.expm1(np.array([e[4] for e in em]) + 8 * U * (nq + 16))
            conf_r = max(conf_r, ratio(got["t_conf"][b, :k], cf, bd))
    lst = ref["last"]
    if not np.array_equal(got["lab_idx"], lst["keys"][:, 0]):
        fails.append("label key index")
    if D and not np.array_equal(got["dur_idx"], lst["keys"][:, 1]):
        fails.append("duration key index")
    if not D and not np.all(got["dur_idx"] == -1):
        fails.append("RNN-T posted a duration key")
    if inp["carry"] and not np.array_equal(got["tok_state"], ref["tok"]):
        fails.append("tok_state")
    if not check_values:
        return fails, r
    r["conf"] = conf_r
    try:
        rh = 0.0
        for l in range(L):
            for s in range(2):
                rh = max(rh, check_planes(got["h_hi"][l, s], got["h_lo"][l, s], ref["hp"][l][s], ref["ehp"][l][s]))
        r["h"] = rh
        r["z"] = check_planes(got["z_hi"], got["z_lo"], lst["z"], lst["ez"])
    except AssertionError as e:
        fails.append(f"planes: {e}")
    rows = np.nonzero(lst["keys"][:, 0] >= 0)[0]
    ki = lst["keys"][rows, 0]
    r["label max"] = ratio(got["lab_val"][rows], lst["lg"][rows, ki], lst["el"][rows, ki]) if rows.size else 0.0
    if D:
        rows = np.nonzero(lst["keys"][:, 1] >= 0)[0]
        ki = V + lst["keys"][rows, 1]
        r["dur max"] = ratio(got["dur_val"][rows], lst["lg"][rows, ki], lst["el"][rows, ki]) if rows.size else 0.0
    ok = np.isfinite(lst["lse"])
    r["lse"] = ratio(got["lse"][ok], lst["lse"][ok], lst["el_lab"][ok] + 8 * U * nq + U * np.abs(lst["lse"][ok]))
    if inp["carry"]:
        r["c"] = max(ratio(got["c_state"][l], ref["c"][l], ref["ec"][l] + 2 * U * np.abs(ref["c"][l])) for l in range(L))
    return fails, r


def geometry_candidates(c: Case):
    """The plan of the launch: max_ctas SMs, the cluster size forced or the engine's (4 where the k-split allows it)."""
    CL = c.cluster or (4 if fits(c.P, c.J, 4) else 2)
    nc = c.max_ctas // CL
    return [dict(plan(c.P, c.J, c.V, c.D, c.L, c.bpad, nc, CL, c.no_stage), grid=nc * CL)]


# ----------------------------------------------------------------------------------------------------------- CPU: preconditions
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_case_preconditions(c):
    """Margins of every decision, the expected geometry under every plan the launch can choose, and the self-check of the
    checker: the reference, rounded as the kernel stores it, passes."""
    ref = case_ref(c)
    m = ref["margins"]
    assert m.size and m.min() > 1.0, f"{c.name}: a decision within 4x its bound (worst margin {m.min():.3g})"
    for gm in geometry_candidates(c):
        for k, v in c.expect:
            assert gm[k] == v, f"{c.name}: plan {gm} does not give {k} = {v}"
    inp = case_inputs(c)
    fails, r = check(inp, ref, fake_output(inp, ref, geometry_candidates(c)[0]))
    assert not fails and max(r.values()) <= 1.0, (fails, r)
    if c.name == "capacity":
        assert ref["overflow"].tolist() == [1, 0, 1] and [len(e) for e in ref["emis"]] == [c.capacity, 0, c.capacity]
    if c.name == "rnnt-ms10-forced":
        assert all(len(e) == c.max_sym * t for e, t in zip(ref["emis"], c.lens))
    if c.name == "clamp-tdt":
        assert any(e[2] == t - 1 and e[1] + 1 < t for em, t in zip(ref["emis"], c.lens) for e in em if t), "no end frame was clamped"
    if c.name == "carry-tdt":
        fb = case_inputs(c)["fbase"]
        assert any(e[2] > fb[b] + t - 1 for b, (em, t) in enumerate(zip(ref["emis"], c.lens)) for e in em), "no end frame past the chunk"
    if c.name.startswith("one-step"):
        assert ref["steps"] == 1 and all(len(e) == 1 for e in ref["emis"])


def test_geometry_coverage_planned():
    """Together the cases reach every branch of the launch geometry (the GPU test asserts the same of the reported one)."""
    seen = [dict(g, L=c.L, bpad=c.bpad) for c in CASES for g in geometry_candidates(c)[:1]]
    _assert_coverage(seen)


def _assert_coverage(seen):
    has = lambda **kw: any(all(g[k] == v if not callable(v) else v(g[k]) for k, v in kw.items()) for g in seen)  # noqa: E731
    assert has(cl=4) and has(cl=2)
    assert has(out_in_smem=1) and has(out_in_smem=0, wstage_rows=lambda x: x > 0) and has(out_in_smem=0, wstage_rows=0)
    assert has(L=lambda x: x > 1, wih_in_smem=1) and has(staged_ih=1, L=2) and has(staged_ih=1, L=lambda x: x > 2)
    assert has(L=lambda x: x > 1, wih_in_smem=0, staged_ih=0, wstage_rows=lambda x: x > 0)     # W_ih from L2 beside a tile
    assert has(L=lambda x: x > 1, wih_in_smem=0, staged_ih=0, out_in_smem=1)                   # W_ih from L2, no tile
    assert has(upc=lambda x: x > 20) and has(bpad=lambda x: x > 64)
    assert has(bpad=lambda x: x > 64, out_in_smem=0, wstage_rows=lambda x: x > 0)


# ----------------------------------------------------------------------------------------------------------- CPU: pinning to the oracle
def _oracle_weights(inp, d_model, rng, prefix):
    """An oracle checkpoint whose G0 and EP are exactly the reference's inputs."""
    P, J, V, D, L = inp["P"], inp["J"], inp["V"], inp["D"], inp["L"]
    W = {}
    f = lambda a: np.asarray(a, np.float32)  # noqa: E731
    E = f(rng.normal(0, 1, (V, P)))
    for l in range(L):
        q = f"prediction_.lstm_.cells_.{l}."
        W[q + "hidden_proj_.weight"] = inp["Whh"][l]
        W[q + "input_proj_.weight"] = f(rng.uniform(-1, 1, (4 * P, P)) / math.sqrt(P)) if l == 0 else inp["Wih"][l]
        W[q + "input_proj_.bias"] = f(rng.normal(0, 0.3, 4 * P)) if l == 0 else inp["bih"][l]
    W["prediction_.embed_.weight"] = E
    W[prefix + "enc_proj_.weight"] = f(rng.uniform(-1, 1, (J, d_model)) / math.sqrt(d_model))
    W[prefix + "enc_proj_.bias"] = f(rng.normal(0, 0.5, J))
    W[prefix + "pred_proj_.weight"] = inp["Wp"]
    if D:
        W[prefix + "label_proj_.weight"], W[prefix + "label_proj_.bias"] = inp["Wout"][:V], inp["bout"][:V]
        W[prefix + "duration_proj_.weight"], W[prefix + "duration_proj_.bias"] = inp["Wout"][V:], inp["bout"][V:]
    else:
        W[prefix + "out_proj_.weight"], W[prefix + "out_proj_.bias"] = inp["Wout"], inp["bout"]
    q = "prediction_.lstm_.cells_.0."
    G0 = (E.astype(np.float64) @ W[q + "input_proj_.weight"].T.astype(np.float64) + W[q + "input_proj_.bias"]).astype(np.float32)
    return W, G0


def _pin_inputs(c, seed, d_model=32, extra=()):
    inp = dict(case_inputs(c))
    rng = np.random.default_rng(seed)
    prefix = "tdt_joint_." if inp["D"] else "joint_."
    W, G0 = _oracle_weights(inp, d_model, rng, prefix)
    enc = [np.asarray(rng.normal(0, 1, (t, d_model)), np.float32) for t in c.lens]
    EP = np.concatenate([e.astype(np.float64) @ W[prefix + "enc_proj_.weight"].T.astype(np.float64) + W[prefix + "enc_proj_.bias"]
                         for e in enc]).astype(np.float32)
    inp.update(G0=G0, EP=EP, rows=EP.shape[0], **dict(extra))
    return inp, W, enc


def _ocfg(O, inp):
    return O.Config(vocab=inp["V"], pred_hidden=inp["P"], joint_hidden=inp["J"], lstm_layers=inp["L"], durations=inp["durations"],
                    joint_prefix="tdt_joint_." if inp["D"] else "joint_.")


PIN_TDT = Case("pin-tdt", P=64, J=96, V=33, L=2, lens=(6, 9, 1), seed=31, blank_bias=-3.0)
PIN_RNNT = Case("pin-rnnt", P=64, J=64, V=33, L=2, durations=(), max_sym=3, lens=(5, 7), seed=32, blank_bias=-0.5)


def test_reference_matches_oracle_tdt_greedy_decode(O):
    inp, W, enc = _pin_inputs(PIN_TDT, 1)
    ref = ref_decode(inp)
    assert ref["margins"].min() > 1.0
    cfg = _ocfg(O, inp)
    for b, e in enumerate(enc):
        want = O.tdt_greedy_decode(W, e, cfg, with_timestamps=True)
        got = ref["emis"][b]
        assert [w[:3] for w in want] == [tuple(int(v) for v in g[:3]) for g in got]
        assert np.allclose([w[3] for w in want], [g[3] for g in got], rtol=1e-4)
    assert sum(len(e) for e in ref["emis"]) >= 5


def test_reference_matches_oracle_stream_decode_chunk(O):
    """Two chunks with carried state against stream_decode_chunk: frame numbering, unclamped end frames, the state handed on."""
    c = dataclasses.replace(PIN_TDT, durations=(1, 2, 4, 6, 8), lens=(5, 7))
    inp, W, enc = _pin_inputs(c, 2)
    cfg = _ocfg(O, inp)
    st = O.StreamDecodeState(cfg)
    L, P = inp["L"], inp["P"]
    h0, c0 = np.zeros((L, 1, P), np.float32), np.zeros((L, 1, P), np.float32)
    tok0, fbase, row = np.array([cfg.vocab - 1], np.int32), np.array([0], np.int32), 0
    for k, e in enumerate(enc):
        want = O.stream_decode_chunk(W, e, st, cfg)
        T = e.shape[0]
        one = dict(inp, n=1, off=np.array([0, T], np.int32), EP=inp["EP"][row:row + T], rows=T, carry=True, h0=h0, c0=c0, tok0=tok0,
                   fbase=fbase, cap=3 * T + 8, max_steps=4 * T + 10)
        ref = ref_decode(one)
        assert ref["margins"].min() > 1.0
        assert [w[:3] for w in want] == [tuple(int(v) for v in g[:3]) for g in ref["emis"][0]], f"chunk {k}"
        h0 = np.stack([ref["hp"][l][0] for l in range(L)]).astype(np.float32)
        c0 = np.stack(ref["c"]).astype(np.float32)
        tok0, fbase, row = ref["tok"].astype(np.int32), fbase + T, row + T
        for l in range(L):
            assert np.allclose(st.states[l][0], h0[l, 0], atol=1e-5) and np.allclose(st.states[l][1], c0[l, 0], atol=1e-5)
        assert tok0[0] == st.token
    assert any(w[2] > w[1] for w in want)


def test_reference_matches_oracle_rnnt_greedy_decode(O):
    inp, W, enc = _pin_inputs(PIN_RNNT, 3)
    ref = ref_decode(inp)
    assert ref["margins"].min() > 1.0
    cfg = O.Config(vocab=inp["V"], pred_hidden=inp["P"], joint_hidden=inp["J"], lstm_layers=inp["L"], durations=(), has_ctc=False,
                   joint_prefix="joint_.")
    for b, e in enumerate(enc):
        want = RO.rnnt_greedy_decode(W, e, cfg, max_symbols=inp["max_sym"], with_timestamps=True)
        got = ref["emis"][b]
        assert [w[:3] for w in want] == [tuple(int(v) for v in g[:3]) for g in got]
        assert np.allclose([w[3] for w in want], [g[3] for g in got], rtol=1e-4)
    assert any(len(e) for e in ref["emis"])


def test_first_argmax_rules(O):
    row = np.array([1.0, 3.0, 3.0, -2.0])
    assert _argmax(row) == O.first_argmax(row) == first_argmax64(row) == 1
    assert _argmax(row, last=True) == 2
    assert _argmax(np.full(5, -np.inf)) == O.first_argmax(np.full(5, -np.inf)) == 0


# ----------------------------------------------------------------------------------------------------------- CPU: sensitivity
MUTATION_CASES = {"gate_if": "110m-n1-cl4", "no_revert": "110m-n33-cl4", "no_relu": "P640-J384", "h_hi_only": "upc64-L2",
                  "zero_c": "carry-tdt", "unclamped": "clamp-tdt", "ties_last": "tie-label-cluster"}


@pytest.mark.parametrize("mut", MUTATIONS)
def test_checker_rejects_mutated_reference(mut):
    """A kernel that computed the mutated reference fails the checks: an output differs or exceeds its bound."""
    if mut == "ties_last":
        c, inp = tie_inputs(MUTATION_CASES[mut])
        ref, bad = ref_decode(inp), ref_decode(inp, {mut})
    else:
        c = BY_NAME[MUTATION_CASES[mut]]
        inp, ref, bad = case_inputs(c), case_ref(c), case_ref(c, {mut})
    fails, r = check(inp, ref, fake_output(inp, bad, geometry_candidates(c)[0]))
    worst = max(r.values()) if r else float("inf")
    report(f"decode mutation {mut}: {fails[:2]}", worst)
    assert fails or worst > 1.0


# ----------------------------------------------------------------------------------------------------------- ties and -inf
def _tie_rows():
    """Head rows whose logits are made equal: one CTA, two CTAs of a cluster, two clusters (the row placement of P3: cluster
    row // OPC, CTA rank (row - cluster * OPC) % CL), for labels and durations."""
    opc = plan(640, 640, 1025, 5, 1, 32, 30, 4)["opc"]
    a, V = 3 * opc + 1, 1025
    rows = {"tie-label-cta": (a, a + 4), "tie-label-cluster-peer": (a, a + 1), "tie-label-cluster": (a, a + opc),
            "tie-dur-cta": (V, V + 4), "tie-dur-cluster-peer": (V + 1, V + 2)}
    for v in range(V - 200, V + 200):                # a vocabulary whose cluster boundary falls between two duration rows
        o = plan(640, 640, v, 5, 1, 32, 30, 4)["opc"]
        k = next((r for r in range(v + 1, v + 5) if r % o == 0), None)
        if k is not None:
            return rows, v, (k - 1, k)
    raise AssertionError("no vocabulary splits the duration rows")


TIE_ROWS, V_SPLIT, _split_rows = _tie_rows()
TIE_SEEDS = {"tie-label-cta": 40, "tie-label-cluster-peer": 41, "tie-label-cluster": 42, "tie-dur-cta": 43, "tie-dur-cluster-peer": 44,
             "tie-all-labels": 45, "no-finite-label": 46, "no-finite-dur": 48}
TIE_CASES = {k: Case(k, **M110, lens=(4, 3), cluster=4, seed=sd, durations=(1, 2, 1, 3, 1)) for k, sd in TIE_SEEDS.items()}
TIE_CASES["tie-dur-cluster"] = Case("tie-dur-cluster", P=640, J=640, V=V_SPLIT, lens=(4, 3), cluster=4, seed=47, durations=(1, 2, 1, 3, 1))
TIE_ROWS["tie-dur-cluster"] = _split_rows


def tie_inputs(name):
    c = TIE_CASES[name]
    inp = dict(case_inputs(c))
    Wout, bout = inp["Wout"].copy(), inp["bout"].copy()
    V = c.V
    if name in TIE_ROWS:
        rows = list(TIE_ROWS[name])
        Wout[rows] = 0
        bout[rows] = 30.0
    elif name == "tie-all-labels":
        Wout[:V] = 0
        bout[:V] = 1.5
    elif name == "no-finite-label":
        bout[:V] = -np.inf
    elif name == "no-finite-dur":
        bout[V:] = -np.inf
    inp.update(Wout=Wout, bout=bout)
    return c, inp


@functools.lru_cache(maxsize=16)
def tie_ref(name):
    c, inp = tie_inputs(name)
    return ref_decode(inp)


def test_tie_cases_are_exact_ties():
    for name in TIE_CASES:
        c, inp = tie_inputs(name)
        ref = tie_ref(name)
        g = geometry_candidates(c)[0]
        if name in TIE_ROWS:
            a, b = TIE_ROWS[name]
            ca, cb = a // g["opc"], b // g["opc"]
            ra, rb = (a - ca * g["opc"]) % 4, (b - cb * g["opc"]) % 4
            kind = name.rsplit("-", 1)[1] if not name.endswith("cluster-peer") else "peer"
            assert {"cta": ca == cb and ra == rb, "peer": ca == cb and ra != rb, "cluster": ca != cb}[kind], (name, ca, cb, ra, rb)
            want = a if a < c.V else a - c.V
            col = 0 if a < c.V else 1
            assert all(k in (-1, want) for k in ref["last"]["keys"][:, col])
            if a < c.V:
                assert all(e[0] == want for em in ref["emis"] for e in em) and any(ref["emis"])
        if name == "tie-all-labels":
            assert all(e[0] == 0 for em in ref["emis"] for e in em) and any(ref["emis"])
        if name == "no-finite-label":
            assert all(e[0] == 0 for em in ref["emis"] for e in em) and any(ref["emis"])
        if name == "no-finite-dur":      # durations[0] = 1 is the skip of every symbol
            assert all(e[2] == e[1] for em in ref["emis"] for e in em) and any(ref["emis"])
        m = ref["margins"]
        assert m.size and m.min() > 1.0, (name, m.min())


# ----------------------------------------------------------------------------------------------------------- GPU
RESULTS = {}


def _run_case(pkg, c):
    if c.name not in RESULTS:
        inp = case_inputs(c)
        RESULTS[c.name] = (c, run_hook(pkg, inp, c.cluster, c.max_ctas, c.no_stage))
    return RESULTS[c.name][1]


@gpu
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_decode_against_fp64(pkg, c):
    got = _run_case(pkg, c)
    assert got["status"] == 0, f"pk_kernel_tdt_decode -> {got['status']}"
    g = got["geom"]
    for k, v in c.expect:
        assert g[k] == v, f"{c.name}: geometry {g}: expected {k} = {v}"
    want = plan(c.P, c.J, c.V, c.D, c.L, c.bpad, g["grid"] // g["cl"], g["cl"], c.no_stage)
    assert {k: g[k] for k in want} == want, f"reported {g}, planned {want}"
    fails, r = check(case_inputs(c), case_ref(c), got)
    report(f"decode {c.name} {g}: " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()), max(r.values()))
    assert not fails, fails
    assert max(r.values()) <= 1.0, r


@gpu
def test_decode_geometry_coverage(pkg):
    seen = []
    for c in CASES:
        g = _run_case(pkg, c)["geom"]
        seen.append(dict(g, L=c.L, bpad=c.bpad))
    _assert_coverage(seen)


@gpu
@pytest.mark.parametrize("name", list(TIE_CASES))
def test_decode_ties_and_missing_maximum(pkg, name):
    """Equal logits in one CTA, in two CTAs of a cluster and in two clusters: the lower index wins; every label tied: index
    0; no finite label (or duration) logit: index 0, as the reference's scan."""
    c, inp = tie_inputs(name)
    got = run_hook(pkg, inp, c.cluster, c.max_ctas)
    assert got["status"] == 0
    want = geometry_candidates(c)[0]
    assert (got["geom"]["grid"], got["geom"]["opc"]) == (want["grid"], want["opc"]), got["geom"]
    ref = tie_ref(name)
    fails, r = check(inp, ref, got, check_values=not name.startswith("no-finite"))
    report(f"decode {name}", max(r.values()) if r else 0.0)
    assert not fails, fails
    assert not r or max(r.values()) <= 1.0, r


@gpu
def test_forced_cluster_size_that_does_not_fit_is_invalid(pkg):
    inp = case_inputs(BY_NAME["P96"])
    assert run_hook(pkg, inp, cluster=4)["status"] == 1         # PK_ERR_INVALID: P = 96 has no 4-way k-split


@gpu
def test_cluster_size_is_decided_per_launch(pkg):
    """A decode whose shape rules out 4-CTA clusters must not change the choice for later decodes in the process."""
    small = run_hook(pkg, case_inputs(BY_NAME["P96"]))
    assert small["status"] == 0 and small["geom"]["cl"] == 2
    c = BY_NAME["110m-n1-cl4"]
    big = run_hook(pkg, case_inputs(c))
    assert big["status"] == 0 and big["geom"]["cl"] == 4, big["geom"]
    fails, _ = check(case_inputs(c), case_ref(c), big)
    assert not fails, fails
