"""Float64 restatement of CTC forced alignment (PK_DECODER_CTC_ALIGN, DESIGN.md section 15), for the tests.

lp is one utterance's [T][V] log-probs (fp32 values, blank = V - 1), y its target ids.  align() runs the Viterbi pass with
the definition's tie rules, the forward pass, the back-trace and the greedy collapse, and records the margin of every
decision the back-trace took (the chosen predecessor against the best other one) and of the final state choice, so a test
can require every decision to be wider than what rounding could move.  brute_force() enumerates every path instead."""
from __future__ import annotations

import itertools
import math

import numpy as np

NEG = -math.inf


def extended(y, blank):
    z = [blank]
    for c in y:
        z += [int(c), blank]
    return z


def feasible(T, y):
    rep = sum(1 for i in range(len(y) - 1) if y[i] == y[i + 1])
    return T >= len(y) + rep


def _lse(xs):
    m = max(xs)
    if m == NEG:
        return NEG
    return m + math.log(sum(math.exp(x - m) for x in xs))


def collapse(labels, lp, blank):
    """The greedy CTC rule (ctc.cu ctc_collapse_row): (id, start, end, conf) per token, conf = exp(lp[start][id]) in fp32."""
    out, prev = [], -1
    for t, cur in enumerate(labels):
        if cur != prev:
            if prev != -1 and prev != blank and out:
                out[-1][2] = t - 1
            if cur != blank:
                out.append([int(cur), t, t, float(np.float32(np.exp(np.float64(lp[t, cur]))))])
        prev = cur
    if out:
        out[-1][2] = len(labels) - 1
    return [tuple(x) for x in out]


def align(lp, y):
    """-> dict(tokens, score, loglik, path (state per frame, -1 when not aligned), labels, margins [(t, margin)])."""
    lp = np.asarray(lp, np.float32)
    T, V = lp.shape
    blank = V - 1
    y = [int(c) for c in y]
    z = extended(y, blank)
    S = len(z)
    none = dict(tokens=[], score=NEG, loglik=NEG, path=[-1] * T, labels=[blank] * T, margins=[])
    if not feasible(T, y):
        return none
    if T == 0:
        return dict(tokens=[], score=0.0, loglik=0.0, path=[], labels=[], margins=[])
    X = lp.astype(np.float64)[:, z]                                 # [T][S]: lp[t][z_s]
    skip = np.array([s % 2 == 1 and s >= 3 and z[s] != z[s - 2] for s in range(S)])
    ninf1, ninf2 = np.full(1, NEG), np.full(2, NEG)
    d = np.full(S, NEG)
    d[:2] = X[0, :2]
    a = d.copy()
    hist = [d]
    with np.errstate(invalid="ignore", divide="ignore"):
        for t in range(1, T):
            p1, p2 = np.concatenate([ninf1, d[:-1]]), np.where(skip, np.concatenate([ninf2, d[:-2]]), NEG)
            m = np.where(p1 > d, p1, d)                             # ties to s, then s-1, then s-2
            m = np.where(p2 > m, p2, m)
            d = X[t] + m
            q1, q2 = np.concatenate([ninf1, a[:-1]]), np.where(skip, np.concatenate([ninf2, a[:-2]]), NEG)
            mm = np.maximum(a, np.maximum(q1, q2))
            fin = mm != NEG
            mz = np.where(fin, mm, 0.0)
            a = X[t] + np.where(fin, mz + np.log(np.exp(a - mz) + np.exp(q1 - mz) + np.exp(q2 - mz)), NEG)
            hist.append(d)
    d, a = [float(v) for v in d], [float(v) for v in a]
    end, score = S - 1, d[S - 1]
    margins = []
    if S >= 2:
        if d[S - 2] > score:
            end, score = S - 2, d[S - 2]
        margins.append((T - 1, abs(d[S - 1] - d[S - 2])))
    loglik = _lse([a[S - 1], a[S - 2]]) if S >= 2 else a[0]
    if score == NEG:
        return none
    path = [0] * T
    s = end
    for t in range(T - 1, -1, -1):
        path[t] = s
        if t == 0:
            break
        p = hist[t - 1]
        cands = [(p[s], 0)] + ([(p[s - 1], 1)] if s >= 1 else []) + ([(p[s - 2], 2)] if skip[s] else [])
        best = max(c[0] for c in cands)
        k = next(c[1] for c in cands if c[0] == best)            # ties to s, then s-1, then s-2
        others = [c[0] for c in cands if c[1] != k and c[0] != NEG]
        margins.append((t, best - max(others) if others else math.inf))
        s -= k
    labels = [z[s] for s in path]
    return dict(tokens=collapse(labels, lp, blank), score=score, loglik=loglik, path=path, labels=labels, margins=margins)


def min_margin(res):
    return min((m for _, m in res["margins"]), default=math.inf)


def margins_clear(res, lp_err=0.0, floor=1e-9):
    """Every decision wider than `floor` and than what an error of lp_err in each log-prob could move: a decision at
    frame t compares two sums of t + 1 log-probs."""
    return all(m > max(floor, 2.0 * (t + 2) * lp_err) for t, m in res["margins"])


def brute_force(lp, y):
    """Every one of the V^T label paths: -> (best score, the best paths' labels, log of the summed probability)."""
    lp = np.asarray(lp, np.float32)
    T, V = lp.shape
    blank = V - 1
    want = [int(c) for c in y]
    best, arg, tot = NEG, [], []
    for path in itertools.product(range(V), repeat=T):
        toks, prev = [], -1
        for c in path:
            if c != prev and c != blank:
                toks.append(c)
            prev = c
        if toks != want:
            continue
        sc = math.fsum(float(lp[t, c]) for t, c in enumerate(path))
        tot.append(sc)
        if sc > best:
            best, arg = sc, [list(path)]
        elif sc == best:
            arg.append(list(path))
    return best, arg, (_lse(tot) if tot else NEG)


def make_logprobs(rng, T, V, sigma=1.0, peak=2.0):
    """Random fp32 log-softmax rows with a peaked label per frame (blank-heavy like a CTC head)."""
    x = rng.normal(0.0, sigma, size=(T, V))
    if T:
        hot = rng.integers(0, V, size=T)
        hot[rng.random(T) < 0.5] = V - 1
        x[np.arange(T), hot] += peak
    x = x - x.max(axis=1, keepdims=True) if T else x
    return (x - np.log(np.exp(x).sum(axis=1, keepdims=True))).astype(np.float32) if T else np.zeros((0, V), np.float32)


def targets_with_repeats(rng, L, V, p_repeat=0.3):
    y = []
    for _ in range(L):
        if y and rng.random() < p_repeat:
            y.append(y[-1])
        else:
            y.append(int(rng.integers(0, V - 1)))
    return y


def max_feasible_len(T, y_gen):
    """The longest prefix of y_gen that T frames can align."""
    n = 0
    while n < len(y_gen) and feasible(T, y_gen[:n + 1]):
        n += 1
    return n
