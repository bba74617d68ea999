"""Oracle of maximal marginal relevance (rbk_index_search_mmr_f64), test infrastructure: the candidates from
oracle.search over the whole corpus, the greedy selection in C (tests/mmr_oracle.c) on the oracle's cosine.  The library
is built into a temporary directory, so the tree may be read-only."""
from __future__ import annotations

import ctypes as C
import hashlib
import subprocess
import tempfile
from pathlib import Path

import numpy as np

import oracle

_SRC = Path(__file__).resolve().parent / "mmr_oracle.c"
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        # the selection calls rbk_oracle_cosine: the oracle's library goes first, with its symbols global
        C.CDLL(str(oracle.build()), mode=C.RTLD_GLOBAL)
        tag = hashlib.sha256(_SRC.read_bytes()).hexdigest()[:16]
        so = Path(tempfile.gettempdir()) / f"rbk_mmr_oracle_{tag}.so"
        if not so.exists():
            tmp = so.with_suffix(f".{id(so)}.tmp")
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-std=c11", "-shared",
                            str(_SRC), "-o", str(tmp), "-lm"], check=True)
            tmp.replace(so)
        lib = C.CDLL(str(so))
        lib.rbk_oracle_mmr_select.restype = C.c_int64
        lib.rbk_oracle_mmr_select.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_double,
                                              C.c_void_p]
        _LIB = lib
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def stored_values(corpus) -> np.ndarray:
    """float64 rows of a float64 or bf16-as-uint16 corpus, as the index uses them as values."""
    if corpus.dtype == np.uint16:
        return (corpus.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return np.asarray(corpus, dtype=np.float64)


def select(rows, rel, k: int, lam: float) -> np.ndarray:
    """Candidate indices of the greedy picks over candidate rows [m, d] with relevance [m], in selection order."""
    rows = np.ascontiguousarray(rows, dtype=np.float64)
    rel = np.ascontiguousarray(rel, dtype=np.float64)
    m = rel.shape[0]
    picks = np.empty(max(min(k, m), 1), dtype=np.int64)
    n = _lib().rbk_oracle_mmr_select(_p(rows), m, rows.shape[1] if rows.ndim == 2 else 0, _p(rel), k, float(lam),
                                     _p(picks))
    assert n >= 0, "out of memory"
    return picks[:n].copy()


def mmr(corpus, query, k: int, fetch_k: int, lam: float, min_score: float | None, live=None):
    """(slots int64 [n], scores float64 [n]): the picks of query's MMR over corpus (float64, or bf16 as uint16), n =
    min(k, number of candidates); the candidates are oracle.search(corpus, query, fetch_k, min_score, live)."""
    slots, scores = oracle.search(corpus, query, fetch_k, min_score, live=live)
    if len(slots) == 0:
        return slots, scores
    picks = select(stored_values(corpus[slots]), scores, k, lam)
    return slots[picks], scores[picks]


def mmr_rows(corpus, queries, ks, fetch_ks, lams, mins, live=None):
    """mmr() per query in the [B][K] layout of Index.search_mmr (K = max(ks), tail -1 / quiet NaN):
    (slots, scores, counts)."""
    B, K = len(queries), max(ks)
    out_s = np.full((B, K), -1, dtype=np.int64)
    out_v = np.full((B, K), np.nan, dtype=np.float64)
    out_c = np.zeros(B, dtype=np.int32)
    for b in range(B):
        s, v = mmr(corpus, queries[b], ks[b], fetch_ks[b], lams[b], mins[b], live)
        out_s[b, :len(s)], out_v[b, :len(s)], out_c[b] = s, v, len(s)
    return out_s, out_v, out_c
