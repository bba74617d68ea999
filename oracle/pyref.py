"""Independent pure-Python restatement of the same reference lines (small cases only).

Python floats are IEEE-754 binary64 and CPython never fuses a*b+c, so these loops have
the same arithmetic as the TypeScript.  Used to cross-check rbk_oracle.c bit-for-bit and
to generate tests/golden/*.json (tests/golden/make_golden.py).  Test infrastructure.
"""
from __future__ import annotations

import math


def cosine_similarity(a, b):
    """embedder.ts:168-184."""
    if len(a) != len(b):
        raise ValueError("Vectors must have the same length")
    dot = 0.0
    na = 0.0
    nb = 0.0
    for i in range(len(a)):
        dot += a[i] * b[i]
        na += a[i] * a[i]
        nb += b[i] * b[i]
    den = math.sqrt(na) * math.sqrt(nb)
    if den == 0.0:  # JS: x/0 -> NaN (0/0) or +-Infinity (a norm that underflows to 0 while the dot does not)
        return float("nan") if dot == 0.0 or dot != dot else math.copysign(float("inf"), dot)
    return dot / den


def find_most_similar(query, embeddings, top_k=10):
    """embedder.ts:189-202.  embeddings: list of (id, vector)."""
    scored = [(i, cosine_similarity(query, e)) for i, e in embeddings]
    scored = [s for s in scored if s[1] == s[1]]  # NaN rows dropped (DESIGN.md, edge E3)
    scored.sort(key=lambda s: -s[1])  # list.sort is stable, like V8's
    return scored[:top_k]


def vector_scan(query, rows, top_k=None, min_score=None):
    """vector-store.ts:201-221.  rows: iterable of (id, vector) in Map insertion order.

    Returns the `scored.slice(0, topK*2)` list of (id, score)."""
    top_k = top_k or 10          # :201  `options.topK || 10`
    min_score = min_score or 0.5  # :202  `options.minScore || 0.5`
    scored = []
    for rid, emb in rows:        # :210-215
        s = cosine_similarity(query, emb)
        if s >= min_score:
            scored.append((rid, s))
    scored.sort(key=lambda s: -s[1])  # :218
    return scored[: top_k * 2]        # :221


def rrf(fts_ids, vec_ids, top_k, k=60, fts_w=0.4, vec_w=0.6):
    """hybrid-search.ts:106-151."""
    scores = {}
    for i, cid in enumerate(fts_ids):
        r = fts_w * (1 / (k + i + 1))
        scores[cid] = scores.get(cid, 0.0) + r if cid in scores else r
    for i, cid in enumerate(vec_ids):
        r = vec_w * (1 / (k + i + 1))
        scores[cid] = scores[cid] + r if cid in scores else r
    out = list(scores.items())
    out.sort(key=lambda e: -e[1])
    return out[:top_k]
