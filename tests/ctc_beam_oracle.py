"""Float64 restatement of the CTC prefix beam search with word n-gram fusion (DESIGN.md section 14), an independent ARPA
reader, and the generators the tests use (seeded log-prob matrices and ARPA files).

The beam search records the margin of every decision the kernel takes (the W-th against the (W+1)-th candidate of a
frame, the lineage kept when two candidates merge, the best beam against the second at the end) with the magnitude of
the scores compared, so a test can require each decision to be wider than the kernel's rounding before it compares bytes.
"""
from __future__ import annotations

import itertools
import math

import numpy as np

SP_MARK = "▁"
NEG = -math.inf
LN10 = math.log(10.0)


def lse(a, b):
    if a == NEG:
        return b
    if b == NEG:
        return a
    m = max(a, b)
    return m + math.log1p(math.exp(-abs(a - b)))


# ------------------------------------------------------------------ ARPA
class Arpa:
    """Standard ARPA back-off: p(w | h) = prob(h w) if present, else backoff(h) + p(w | h[1:]) (backoff 0 when h is absent)."""

    def __init__(self, path):
        self.prob, self.bo, self.order = {}, {}, 0
        with open(path, encoding="utf-8") as f:
            lines = [ln.rstrip("\n") for ln in f]
        i = lines.index("\\data\\") + 1
        counts = {}
        while lines[i].startswith("ngram "):
            k, c = lines[i][6:].split("=")
            counts[int(k)] = int(c)
            i += 1
        self.order = max(counts)
        for k in range(1, self.order + 1):
            while lines[i].strip() != f"\\{k}-grams:":
                i += 1
            i += 1
            n = 0
            while n < counts[k]:
                fld = lines[i].split()
                i += 1
                if not fld:
                    continue
                g = tuple(fld[1:k + 1])
                self.prob[g] = float(fld[0])
                self.bo[g] = float(fld[k + 1]) if len(fld) > k + 1 else 0.0
                n += 1
        if ("<unk>",) not in self.prob:
            self.prob[("<unk>",)], self.bo[("<unk>",)] = -10.0, 0.0
        self.vocab = {g[0] for g in self.prob if len(g) == 1}

    def word(self, w):
        return w if w in self.vocab else "<unk>"

    def p(self, hist, w):
        hist = tuple(hist[-(self.order - 1):]) if self.order > 1 else ()
        acc = 0.0
        while True:
            if hist + (w,) in self.prob:
                return acc + self.prob[hist + (w,)]
            acc += self.bo.get(hist, 0.0)
            hist = hist[1:]

    def start(self):
        return ("<s>",) if ("<s>",) in self.prob else ()

    def sentence_log10(self, words):
        h, acc = self.start(), 0.0
        for w in words + ["</s>"]:
            w = self.word(w)
            acc += self.p(h, w)
            h = h + (w,)
        return acc


def write_arpa(path, grams, order):
    """grams: {tuple: (log10 prob, log10 backoff or None)}."""
    with open(path, "w", encoding="utf-8") as f:
        f.write("\n\\data\\\n")
        for k in range(1, order + 1):
            f.write(f"ngram {k}={sum(1 for g in grams if len(g) == k)}\n")
        for k in range(1, order + 1):
            f.write(f"\n\\{k}-grams:\n")
            for g, (p, b) in grams.items():
                if len(g) == k:
                    f.write(f"{p:.6f}\t{' '.join(g)}" + (f"\t{b:.6f}" if b is not None else "") + "\n")
        f.write("\n\\end\\\n")


def make_arpa(path, words, order, seed, per_order=200, unk=True):
    """A seeded ARPA file of `order` over `words` (plus <s>, </s>, and <unk> when asked); higher-order n-grams extend
    random lower-order ones, so their contexts exist and back-off chains of every length occur."""
    rng = np.random.default_rng(seed)
    grams = {}
    uni = list(words) + ["</s>"] + (["<unk>"] if unk else [])
    for w in uni:
        grams[(w,)] = (float(rng.uniform(-4, -0.5)), float(rng.uniform(-1, 0)) if order > 1 else None)
    grams[("<s>",)] = (-99.0, float(rng.uniform(-1, 0)) if order > 1 else None)
    for k in range(2, order + 1):
        ctxs = [g for g in grams if len(g) == k - 1 and g[-1] != "</s>" and "<s>" not in g[1:]]
        n, tries = 0, 0
        while n < per_order and tries < 20 * per_order:
            tries += 1
            c = ctxs[int(rng.integers(len(ctxs)))]
            w = uni[int(rng.integers(len(uni)))]
            if w == "<unk>" or c + (w,) in grams:
                continue
            grams[c + (w,)] = (float(rng.uniform(-3, -0.05)), float(rng.uniform(-1, 0)) if k < order else None)
            n += 1
    write_arpa(path, grams, order)
    return grams


# ------------------------------------------------------------------ inputs
def make_logprobs(rng, T, V, sigma=1.0, peak=4.0, p_blank=0.5, p_repeat=0.3):
    """[T][V] float32 log-probs with controlled entropy: per frame a dominant token (the blank with p_blank, the previous
    dominant token with p_repeat, else a random one) raised by `peak` over normal(0, sigma) logits."""
    x = rng.normal(0.0, sigma, (T, V))
    prev = V - 1
    for t in range(T):
        u = rng.random()
        d = V - 1 if u < p_blank else (prev if u < p_blank + p_repeat else int(rng.integers(V - 1)))
        x[t, d] += peak
        prev = d
    x -= x.max(axis=1, keepdims=True)
    x -= np.log(np.exp(x).sum(axis=1, keepdims=True))
    return x.astype(np.float32)


def greedy(lp):
    """CTC greedy token ids (first maximum, blank = V - 1)."""
    V = lp.shape[1]
    out, prev = [], -1
    for t in range(lp.shape[0]):
        c = int(np.argmax(lp[t]))
        if c != prev and c != V - 1:
            out.append(c)
        prev = c
    return out


def piece_table(pieces):
    """Per token (starts a word, word bytes of the piece without the leading mark)."""
    tab = []
    for p in pieces:
        st = p.startswith(SP_MARK)
        tab.append((st, (p[1:] if st else p).encode("utf-8")))
    return tab


# ------------------------------------------------------------------ the decode
def beam_search(lp, W, lm=None, pieces=None, alpha=0.5, beta=1.0, extend_all=False, keep_all=False):
    """CTC prefix beam search on one utterance's [T][V] log-probs (blank = V - 1) in float64.

    W: beam width; extend_all: extend by every finite non-blank token instead of the W best; keep_all: keep every
    candidate (no pruning).  lm: an Arpa; pieces: the vocabulary's pieces (needed with lm); alpha / beta as float32.
    Returns dict(tokens=[(id, start, end, conf)], score, prefix, margins=[(gap, scale)], merges, beams)."""
    lp = np.asarray(lp, np.float32)
    T, V = lp.shape
    blank = V - 1
    a_ln10 = float(np.float32(alpha)) * LN10
    bt = float(np.float32(beta))
    tab = piece_table(pieces) if lm is not None else None
    beams = [dict(p=(), pb=0.0, pnb=NEG, lm=0.0, hist=lm.start() if lm else (), word=b"", starts=())]
    margins, merges = [], 0

    def word_term(b):
        """LM term and history after completing b's unfinished word."""
        w = lm.word(b["word"].decode("utf-8", "surrogateescape"))
        return a_ln10 * lm.p(b["hist"], w) + bt, b["hist"] + (w,)

    for t in range(T):
        row = lp[t].astype(np.float64)
        ids = [v for v in range(blank) if row[v] > NEG]
        ids.sort(key=lambda v: (-row[v], v))
        if not extend_all:
            ids = ids[:W]
        cands, index = [], {}
        for b in beams:
            last = b["p"][-1] if b["p"] else -1
            pb = lse(b["pb"], b["pnb"]) + row[blank]
            pnb = b["pnb"] + row[last] if last >= 0 else NEG
            c = dict(b, pb=pb, pnb=pnb, own=lse(pb, pnb))
            index[c["p"]] = len(cands)
            cands.append(c)
        for b in beams:
            last = b["p"][-1] if b["p"] else -1
            base = lse(b["pb"], b["pnb"])
            for v in ids:
                term = (b["pb"] if v == last else base) + row[v]
                p = b["p"] + (v,)
                if p in index:
                    c = cands[index[p]]
                    merges += 1
                    if term > NEG and c["own"] > NEG:
                        margins.append((abs(term - c["own"]), max(abs(term), abs(c["own"]))))
                    if term > c["own"]:
                        c["starts"] = b["starts"] + (t,)
                    c["pnb"] = lse(c["pnb"], term)
                    continue
                c = dict(p=p, pb=NEG, pnb=term, lm=b["lm"], hist=b["hist"], word=b["word"], starts=b["starts"] + (t,))
                if lm is not None:
                    st, wb = tab[v]
                    if st:
                        if b["word"]:
                            d, c["hist"] = word_term(b)
                            c["lm"] = b["lm"] + d
                        c["word"] = wb
                    else:
                        c["word"] = b["word"] + wb
                index[p] = len(cands)
                cands.append(c)
        scored = [(lse(c["pb"], c["pnb"]) + c["lm"], k) for k, c in enumerate(cands)]
        scored = [s for s in scored if s[0] > NEG]
        scored.sort(key=lambda s: (-s[0], s[1]))
        if not keep_all and len(scored) > W:
            margins.append((scored[W - 1][0] - scored[W][0], max(abs(scored[W - 1][0]), abs(scored[W][0]))))
            scored = scored[:W]
        beams = [cands[k] for _, k in scored]
        if not beams:
            break
    finals = []
    for b in beams:
        s = lse(b["pb"], b["pnb"]) + b["lm"]
        if lm is not None:
            h, e = b["hist"], 0.0
            if b["word"]:
                w = lm.word(b["word"].decode("utf-8", "surrogateescape"))
                e += lm.p(h, w)
                h = h + (w,)
                s += bt
            s += a_ln10 * (e + lm.p(h, lm.word("</s>")))
        finals.append(s)
    if len(finals) >= 2:
        srt = sorted(finals, reverse=True)
        if srt[1] > NEG:
            margins.append((srt[0] - srt[1], max(abs(srt[0]), abs(srt[1]))))
    if not beams or T == 0 or max(finals) == NEG:
        return dict(tokens=[], score=NEG, prefix=(), margins=margins, merges=merges, beams=beams)
    best = int(np.argmax(finals))              # first maximum: ties to the lower slot
    b = beams[best]
    toks = []
    for k, (v, s) in enumerate(zip(b["p"], b["starts"])):
        e = b["starts"][k + 1] - 1 if k + 1 < len(b["p"]) else T - 1
        toks.append((v, s, e, math.exp(float(lp[s, v]))))
    return dict(tokens=toks, score=finals[best], prefix=b["p"], margins=margins, merges=merges, beams=beams)


def min_margin_ratio(res, T, rel=1e-11):
    """The narrowest decision over its rounding bound rel (1 + scale) (T + 1): the kernel keeps scores in double, each
    frame adds a few roundings of relative size 2^-53 to every score."""
    if not res["margins"]:
        return math.inf
    return min(g / (rel * (1.0 + s) * (T + 1)) for g, s in res["margins"])


def margins_clear(res, T, lp_err):
    """Every decision wider than 4x the error of a sum of T + 1 log-probs that are each off by at most lp_err (the device's
    log-probs against the oracle's, when the decode runs on the device's own)."""
    return all(g > 4 * lp_err * (T + 1) for g, _ in res["margins"])


def brute_force(lp):
    """Best collapsed prefix and its ln-probability by enumerating all V^T alignments."""
    lp = np.asarray(lp, np.float64)
    T, V = lp.shape
    tot = {}
    for path in itertools.product(range(V), repeat=T):
        p, prev = [], -1
        for c in path:
            if c != prev and c != V - 1:
                p.append(c)
            prev = c
        s = sum(lp[t, c] for t, c in enumerate(path))
        tot[tuple(p)] = lse(tot.get(tuple(p), NEG), s)
    best = max(tot.items(), key=lambda kv: kv[1])
    return best[0], best[1], tot
