"""numpy restatement of the reference's word -> speaker attribution, diarize_transcription (src/diarize.cpp:10-48).

For each word and each segment, in the order of the segment list, the overlap min(word.end, seg.end) - max(word.start,
seg.start) is taken in float32; only overlaps > 0 count, summed per speaker in float32 (so a zero-length word never gets a
speaker).  The speaker with the largest sum wins; none: -1.

Tie rule: the reference keeps the sums in a std::unordered_map<int, float> and picks with a strict `>` while iterating it.
libstdc++ hashes an int to itself and, while the map holds at most 13 keys below 13, gives each key its own bucket and
links every new key in front of the others, so the iteration runs in reverse order of first insertion: on an exact tie
the speaker whose first positive overlap comes LATEST in the segment list wins.  Speaker ids >= 13 could share a bucket,
so they are refused here (the models have at most a few speakers).  The golden file pins the rule against the compiled
reference (tests/golden/make_golden_diarized.py).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def assign_speakers(word_start, word_end, seg_spk, seg_start, seg_end):
    """-> int32 speaker per word (-1: no segment overlaps it)."""
    ws, we = np.asarray(word_start, F32), np.asarray(word_end, F32)
    spk = np.asarray(seg_spk, np.int64)
    ss, se = np.asarray(seg_start, F32), np.asarray(seg_end, F32)
    if len(spk) and (spk.min() < 0 or spk.max() >= 13):
        raise ValueError("diarize_oracle: speaker ids must lie in [0, 13) for the tie rule it restates")
    out = np.full(len(ws), -1, np.int32)
    for w in range(len(ws)):
        sums = {}            # speaker -> float32 sum; dict order = order of first insertion
        for k in range(len(spk)):
            ov = F32(min(we[w], se[k])) - F32(max(ws[w], ss[k]))
            if ov > F32(0):
                s = int(spk[k])
                sums[s] = F32(sums.get(s, F32(0)) + ov)
        best = F32(0)
        for s in reversed(list(sums)):     # the container's iteration order
            if sums[s] > best:
                best, out[w] = sums[s], s
    return out


def exact_tie(word_start, word_end, seg_spk, seg_start, seg_end):
    """Per word: True when two or more speakers share the largest positive sum (the tie rule decides the word)."""
    ws, we = np.asarray(word_start, F32), np.asarray(word_end, F32)
    res = []
    for w in range(len(ws)):
        sums = {}
        for k in range(len(seg_spk)):
            ov = F32(min(we[w], F32(seg_end[k]))) - F32(max(ws[w], F32(seg_start[k])))
            if ov > F32(0):
                sums[int(seg_spk[k])] = F32(sums.get(int(seg_spk[k]), F32(0)) + ov)
        v = list(sums.values())
        res.append(len(v) > 1 and v.count(max(v)) > 1)
    return np.array(res, bool)
