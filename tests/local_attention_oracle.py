"""Float64 and fp32 references of limited-context (banded) relative-position attention, DESIGN.md section 16.

With a band (left, right) query frame i attends to key j only when -right <= i - j <= left and 0 <= j < T; the score,
the softmax over the keys that remain and the rest of the Conformer block are those of full attention.

ref_attention_local: the kernel-level float64 reference of test_kernels_fp64.ref_attention restricted to the band, with the
  same per-element bound, computed block by block over the keys a block of queries can see (so a 45,001-row utterance
  needs no T x T matrix).  The bound's fp32 sum term counts the keys a query tile visits, at most left + right + 192.
encoder_forward_local: oracle.encoder_forward with the band mask added to oracle.conformer_attention, computed block by block
  (attention over each query block's keys, the subsampling over chunks of frames), so it runs on an hour of audio.
"""
from __future__ import annotations

import math

import numpy as np

import oracle as O
from test_kernels_fp64 import U

F32 = np.float32


def band_mask(T, left, right, Tk=None):
    """[T, Tk] True where query i may attend to key j."""
    i = np.arange(T)[:, None]
    j = np.arange(T if Tk is None else Tk)[None, :]
    return (i - j <= left) & (j - i <= right)


def ref_attention_local(qkv, pp, u, v, row_off, n_utt, d, H, tmax, left, right, kernel, drop_u=False, widen=(0, 0), blocks=None,
                        block=256):
    """-> (out, bound, checked): float64 ctx and bound for the rows of the query blocks computed (every block, or those whose
    start is in `blocks`), checked = the rows computed.  Mutations: widen = (dl, dr) moves the band edges, drop_u drops u."""
    hd = d // H
    rows = qkv.shape[0]
    out, bound = np.zeros((rows, d)), np.zeros((rows, d))
    checked = np.zeros(rows, bool)
    q64 = qkv.astype(np.float64)
    lm, rm = left + widen[0], right + widen[1]
    n_vis = left + right + 192                           # keys a 64-query tile can visit (tiles start on multiples of 64)
    for b in range(n_utt):
        r0, r1 = int(row_off[b]), int(row_off[b + 1])
        T = r1 - r0
        for q0 in range(0, T, block):
            if blocks is not None and q0 not in blocks:
                continue
            q1 = min(T, q0 + block)
            k0, k1 = max(0, q0 - max(lm, 0)), min(T, q1 + max(rm, 0))
            i = np.arange(q0, q1)[:, None]
            j = np.arange(k0, k1)[None, :]
            dij = i - j
            mask = (dij <= lm) & (-dij <= rm)
            prow = np.clip(dij + tmax - 1, 0, 2 * tmax - 2)
            nk = min(T, n_vis)
            checked[r0 + q0:r0 + q1] = True
            for h in range(H):
                cs = slice(h * hd, (h + 1) * hd)
                q = q64[r0 + q0:r0 + q1, cs]
                k = q64[r0 + k0:r0 + k1, d + h * hd:d + (h + 1) * hd]
                V = q64[r0 + k0:r0 + k1, 2 * d + h * hd:2 * d + (h + 1) * hd]
                qu = q + (0.0 if drop_u else u[cs].astype(np.float64))
                qv = q + v[cs].astype(np.float64)
                PPh = pp[:, cs].astype(np.float64)
                G, Ga = qv @ PPh.T, np.abs(qv) @ np.abs(PPh).T
                s = (qu @ k.T + np.take_along_axis(G, prow, axis=1)) / math.sqrt(hd)
                sa = (np.abs(qu) @ np.abs(k).T + np.take_along_axis(Ga, prow, axis=1)) / math.sqrt(hd)
                s = np.where(mask, s, -np.inf)
                sa = np.where(mask, sa, 0.0)
                m = s.max(axis=1, keepdims=True)
                p = np.exp(s - m)
                p /= p.sum(axis=1, keepdims=True)
                out[r0 + q0:r0 + q1, cs] = p @ V
                if kernel == 0:
                    eps_s, eps_pv = hd * U * 2, nk * U * 2
                else:
                    eps_s, eps_pv = 3 * 2.0 ** -16 + hd * U, 3 * 2.0 ** -16 + nk * U + 2.0 ** -21
                D = eps_s * sa.max(axis=1, keepdims=True)
                vmax = np.abs(V).max(axis=0, keepdims=True)
                bound[r0 + q0:r0 + q1, cs] = 4.0 * (2 * D + eps_pv) * vmax
    return out, bound, checked


def brute_attention_local(qkv, pp, u, v, T, d, H, tmax, left, right):
    """Dense float64 masked full attention of one utterance (rows 0..T): the definition, for small T."""
    hd = d // H
    q64 = qkv.astype(np.float64)
    out = np.zeros((T, d))
    mask = band_mask(T, left, right)
    for h in range(H):
        cs = slice(h * hd, (h + 1) * hd)
        q, k, V = q64[:T, cs], q64[:T, d + h * hd:d + (h + 1) * hd], q64[:T, 2 * d + h * hd:2 * d + (h + 1) * hd]
        s = np.empty((T, T))
        for i in range(T):
            for j in range(T):
                if mask[i, j]:
                    s[i, j] = ((q[i] + u[cs]) @ k[j] + (q[i] + v[cs]) @ pp[i - j + tmax - 1, cs].astype(np.float64)) / math.sqrt(hd)
                else:
                    s[i, j] = -np.inf
        p = np.exp(s - s.max(axis=1, keepdims=True))
        out[:, cs] = (p / p.sum(axis=1, keepdims=True)) @ V
    return out


def conformer_attention_local(W, p, x, pos_emb, cfg, left, right, block=512):
    """oracle.conformer_attention with the band, query block by query block over the keys the block can see (no T x T
    matrix).  pos_emb is oracle.sinusoidal_position_embedding(T, d): row r <-> relative position T - 1 - r."""
    T, d = x.shape
    H = cfg.n_heads
    hd = d // H
    h = O.layer_norm(x, W[p + "norm_.weight"], W[p + "norm_.bias"])
    q = O.linear(h, W[p + "mha_.q_proj.weight"], W[p + "mha_.q_proj.bias"]).reshape(T, H, hd).transpose(1, 0, 2)
    k = O.linear(h, W[p + "mha_.k_proj.weight"], W[p + "mha_.k_proj.bias"]).reshape(T, H, hd).transpose(1, 0, 2)
    v = O.linear(h, W[p + "mha_.v_proj.weight"], W[p + "mha_.v_proj.bias"]).reshape(T, H, hd).transpose(1, 0, 2)
    u = W[p + "pos_bias_u_"].reshape(H, 1, hd)
    vb = W[p + "pos_bias_v_"].reshape(H, 1, hd)
    Wd = min(max(left, right), T - 1)                                 # relative positions -Wd..Wd are all a band can use
    pe = pos_emb[T - 1 - Wd:T + Wd]                                   # row r <-> position Wd - r
    pp = O.linear(pe, W[p + "pos_proj_.weight"]).reshape(2 * Wd + 1, H, hd).transpose(1, 0, 2)
    o = np.zeros((H, T, hd), F32)
    for q0 in range(0, T, block):
        q1 = min(T, q0 + block)
        k0, k1 = max(0, q0 - left), min(T, q1 + right)
        i = np.arange(q0, q1)[:, None]
        j = np.arange(k0, k1)[None, :]
        dij = i - j
        mask = (dij <= left) & (-dij <= right)
        prow = np.clip(Wd - dij, 0, 2 * Wd)
        ac = (q[:, q0:q1] + u) @ k[:, k0:k1].transpose(0, 2, 1)
        g = (q[:, q0:q1] + vb) @ pp.transpose(0, 2, 1)                 # (H, nq, 2 Wd + 1)
        bd = np.take_along_axis(g, np.broadcast_to(prow, (H,) + prow.shape), axis=2)
        scores = ((ac + bd) * F32(1.0 / math.sqrt(hd))).astype(F32)
        scores = np.where(mask[None], scores, -np.inf).astype(F32)
        o[:, q0:q1] = O.softmax(scores, axis=-1) @ v[:, k0:k1]
    o = o.transpose(1, 0, 2).reshape(T, d)
    o = O.linear(o, W[p + "mha_.out_proj.weight"], W[p + "mha_.out_proj.bias"])
    return (x + o).astype(F32)


def conv_subsampling_chunked(W, feats, cfg, rows=2048):
    """oracle.conv_subsampling over chunks of `rows` output frames, so an hour of mel frames never makes a whole-utterance
    stage tensor.  Output frame t reads mel frames 8t - 7 .. 8t + 7: a chunk of outputs [a, b) runs on mel frames
    [8a - 8, 8b + 8) and drops its first output (a > 0), whose window the chunk's zero padding cuts."""
    F = feats.shape[0]
    T = O.encoder_len(F)
    out = []
    for a in range(0, T, rows):
        b = min(T, a + rows)
        s = 8 * a - 8 if a else 0
        y = O.conv_subsampling(W, feats[s:min(F, 8 * b + 8)], cfg)
        y = y[1:] if a else y
        out.append(y[:b - a])
    return np.concatenate(out, axis=0)


def encoder_forward_local(W, feats, cfg, left, right):
    """oracle.encoder_forward with banded attention in every block, blockwise throughout (an hour runs in bounded memory)."""
    x = conv_subsampling_chunked(W, feats, cfg)
    pos = O.sinusoidal_position_embedding(x.shape[0], x.shape[1])
    for i in range(cfg.n_layers):
        p = f"encoder_.layers_.{i}."
        x = O.feed_forward(W, p + "ffn1_.", x)
        x = conformer_attention_local(W, p + "attn_.", x, pos, cfg, left, right)
        x = O.conformer_conv(W, p + "conv_.", x, cfg)
        x = O.feed_forward(W, p + "ffn2_.", x)
        x = O.layer_norm(x, W[p + "final_norm_.weight"], W[p + "final_norm_.bias"])
    return x
