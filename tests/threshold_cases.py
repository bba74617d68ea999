"""Corpora and thresholds for the min_score tests: rows placed where `score >= minScore` (vector-store.ts:212) cuts, and
the thresholds themselves, all measured with the oracle (test infrastructure: numpy and the oracle only).

The scan filters on approximate scores, so a threshold is only tested where live rows sit within the scan's error bound
eps_q of it.  eps_q is computed as the proof does (DESIGN.md §6, tests/test_gpu_exact_paths.py):
(d + 8) 2^-22 + angle(q, bf16 q) + the largest angle(row, bf16 row) of a float64-backed corpus (0 for bf16 rows).

- band_corpus: for each query, rows at chosen cosines spread over [t - 3 eps, t + 3 eps], plus random rows;
- ladder: per query, thresholds taken from the oracle's score bytes (hits 1, K and K + 1, a band row, the lowest live
  score) and the float64 neighbours of each; FIXED_LADDER: the thresholds at the ends of the float64 range;
- tie_corpus: a group of exact duplicates whose common score is the threshold;
- ends_corpus: rows scoring 1 and -1 (or one ulp off), +0 and -0, zero rows.
"""
import sys

import numpy as np

K = 10                       # search()'s k_fetch in the GPU matrix: the "k-th hit" of a ladder
DBL_MAX = sys.float_info.max
FIXED_LADDER = (-np.inf, -DBL_MAX, -1e300, np.nextafter(-1.0, -2.0), -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0,
                np.nextafter(1.0, 2.0), 1.5, 1e300, DBL_MAX, np.inf)
BAND_T = (0.5, 0.62, 0.75, 0.9)   # band centres, one per query; random rows score far below 0.5 at d >= 100


def bf16_f64(x):
    """float64 -> float32 (RNE) -> bf16 (RNE), as the ingest and prep kernels round, back in float64."""
    from runbookai_b200 import synth
    with np.errstate(over="ignore"):
        return synth.bf16_round(np.asarray(x, dtype=np.float64).astype(np.float32)).astype(np.float64)


def bf16_bits(x):
    from runbookai_b200 import synth
    return synth.f32_to_bf16_bits(np.asarray(x, dtype=np.float64).astype(np.float32))


def angle_bound(x):
    """asin(||x - bf16(x)|| / ||x||) per row (0 for a zero row)."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    n = np.linalg.norm(x, axis=1)
    r = np.linalg.norm(x - bf16_f64(x), axis=1) / np.where(n > 0, n, 1.0)
    return np.arcsin(np.minimum(r, 1.0))


def eps_q(q, rows, bf16_rows):
    """The scan's error bound for each query against `rows` (float64 values of the rows the index holds)."""
    d = np.asarray(q).shape[-1]
    corpus = 0.0 if bf16_rows else angle_bound(rows).max()
    return (d + 8) * 2.0 ** -22 + angle_bound(q) + corpus


def stored(rows, bf16_rows):
    """What the oracle reads: the float64 rows of a float64-backed index, or the bf16 bits of a bf16 one."""
    return bf16_bits(rows) if bf16_rows else np.asarray(rows, dtype=np.float64)


def unit(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def at_cosines(rng, q, ts, scale=None):
    """Rows t_j q^ + sqrt(1 - t_j^2) u_j with u_j a random unit vector orthogonal to q, times a random scale."""
    qh = unit(q)
    u = rng.standard_normal((len(ts), len(q)))
    u -= (u @ qh)[:, None] * qh[None, :]
    u = unit(u)
    ts = np.asarray(ts, dtype=np.float64)
    rows = ts[:, None] * qh[None, :] + np.sqrt(1.0 - ts * ts)[:, None] * u
    s = rng.uniform(0.5, 2.0, len(ts)) if scale is None else scale
    return rows * np.reshape(s, (-1, 1))


def band_corpus(d, bf16_rows, seed, per_band=1500, n_random=1000):
    """Four queries (the even ones bf16-exact, so their bound is tight) and, for query i, per_band rows whose oracle
    score lies in [BAND_T[i] - 3 eps, BAND_T[i] + 3 eps], among n_random random rows.  Returns a dict: rows (float64, to
    append), stored (what the oracle reads), q, eps (per query, over the final rows), band (the slots of each query's
    band rows) and t."""
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((len(BAND_T), d))
    q[::2] = bf16_f64(q[::2])
    rand = rng.standard_normal((n_random, d))
    if bf16_rows:
        rand = bf16_f64(rand)
    # the bound before the band rows exist; band rows are random directions too, so the final one is no narrower
    eps0 = eps_q(q, rand, bf16_rows)
    parts, band, n = [rand], [], n_random
    for i, t in enumerate(BAND_T):
        lo, hi = t - 3 * eps0[i], t + 3 * eps0[i]
        cand = at_cosines(rng, q[i], rng.uniform(lo, hi, 4 * per_band))
        if bf16_rows:
            cand = bf16_f64(cand)
        import oracle
        sc = oracle.scores(stored(cand, bf16_rows), q[i])
        keep = np.flatnonzero((sc >= lo) & (sc <= hi))[:per_band]
        parts.append(cand[keep])
        band.append(n + np.arange(len(keep)))
        n += len(keep)
    rows = np.concatenate(parts)
    perm = rng.permutation(len(rows))           # interleave band and random rows over the slots
    inv = np.argsort(perm)
    rows = rows[perm]
    band = [np.sort(inv[b]) for b in band]
    return dict(rows=rows, stored=stored(rows, bf16_rows), q=q, eps=eps_q(q, rows, bf16_rows), band=band,
                t=np.array(BAND_T))


def hits(scores, min_score, k=None):
    """The reference's answer from one query's scores: keep `>= min_score` (None: every non-NaN score), stable sort by
    score descending (ties keep slot order), first k.  Returns (slots, scores)."""
    s = np.asarray(scores, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        keep = np.flatnonzero(~np.isnan(s) if min_score is None else s >= min_score)
    order = keep[np.argsort(-s[keep], kind="stable")]
    if k is not None:
        order = order[:k]
    return order, s[order]


def with_neighbours(values):
    """Each value and its float64 neighbours towards -inf and +inf."""
    out = []
    for v in values:
        v = np.float64(v)
        out += [v, np.nextafter(v, -np.inf), np.nextafter(v, np.inf)]
    return out


def ladder(scores, band_slots, t, k=K):
    """One query's thresholds, bytes of the oracle's scores: hits 1, k and k + 1, the band row nearest t, the lowest
    live score, and the neighbours of each."""
    s, v = hits(scores, None)
    mid = band_slots[np.argmin(np.abs(scores[band_slots] - t))]
    return with_neighbours([v[0], v[k - 1], v[k], scores[mid], v[-1]])


def tie_corpus(d, bf16_rows, seed, sizes=(5, 70, 150), above=8, near=20, n_random=2000):
    """For each group size, a query, `size` exact duplicates of one row at cosine ~0.8 (contiguous slots), `above`
    rows scoring clearly higher and `near` rows within the bound below the duplicates, among random rows.  Returns a
    dict: rows, stored, q, dup (the slots of each group), ms (each group's common score, from the oracle), eps."""
    import oracle
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((len(sizes), d))
    q[::2] = bf16_f64(q[::2])
    rand = rng.standard_normal((n_random, d))
    if bf16_rows:
        rand = bf16_f64(rand)
    eps0 = eps_q(q, rand, bf16_rows)
    parts, dup, ms, n = [rand], [], [], n_random
    for g, size in enumerate(sizes):
        u = at_cosines(rng, q[g], [0.8], scale=[1.0])
        hi = at_cosines(rng, q[g], np.linspace(0.9, 0.85, above))
        lo = at_cosines(rng, q[g], 0.8 - eps0[g] * rng.uniform(-1.0, 1.0, 20 * near))
        if bf16_rows:
            u, hi, lo = bf16_f64(u), bf16_f64(hi), bf16_f64(lo)
        ms.append(oracle.scores(stored(u, bf16_rows), q[g])[0])
        sc = oracle.scores(stored(lo, bf16_rows), q[g])
        lo = lo[np.flatnonzero((sc < ms[-1]) & (sc >= ms[-1] - eps0[g]))[:near]]   # what rounding left below
        parts.append(np.concatenate([hi, np.repeat(u, size, axis=0), lo]))
        dup.append(n + above + np.arange(size))
        n += len(parts[-1])
    rows = np.concatenate(parts)
    st = stored(rows, bf16_rows)
    ms = np.array(ms)
    return dict(rows=rows, stored=st, q=q, dup=dup, ms=ms, sizes=sizes, above=above,
                eps=eps_q(q, rows, bf16_rows))


def ends_corpus(d, bf16_rows, seed, huge=False):
    """Queries (bf16-exact, so a multiple by a power of two is exact in every tier) and rows at the cosine ends:
    positive and negative multiples of each query (scores 1 / -1 or one ulp off: whatever the oracle gives), rows
    orthogonal to every query (every product 0, so the dot is +0 and the score +0), zero rows (NaN), and random rows.
    huge=True adds rows scaled by 2^600: their squared norm overflows, so they score +0 or -0 with the sign of the dot
    (and, being outside the scan's range, send every query to the exhaustive kernel).  Returns a dict: rows, stored, q,
    multiples (slots), zero_score (slots scoring +-0), zero_rows (slots)."""
    rng = np.random.default_rng(seed)
    nq = 4
    half = d // 2
    q = np.zeros((nq, d))
    q[:, :half] = bf16_f64(rng.standard_normal((nq, half)))       # the queries live in the first half of the elements
    mult = []
    for i in range(nq):
        for c in (1.0, 2.0 ** -3, 2.0 ** 5, 3.0, 0.1, 7.3, -1.0, -2.0 ** 4, -3.0, -0.37):
            mult.append(c * q[i])
    mult = np.array(mult)
    orth = np.zeros((12, d))
    orth[:, half:] = rng.standard_normal((12, d - half))          # products q_i * 0 and 0 * r_i: all +-0
    orth[::2, :half] = -0.0                                       # -0.0 elements against positive and negative q
    zero = np.zeros((3, d))
    rand = rng.standard_normal((500, d))
    parts = [rand, mult, orth, zero]
    if huge:
        big = np.ldexp(rng.standard_normal((8, d)), 600)
        parts.append(big)
    rows = np.concatenate(parts)
    if bf16_rows:
        rows = bf16_f64(rows)
    n0 = len(rand)
    multiples = n0 + np.arange(len(mult))
    zero_score = n0 + len(mult) + np.arange(len(orth))
    zero_rows = zero_score[-1] + 1 + np.arange(3)
    if huge:
        zero_score = np.concatenate([zero_score, zero_rows[-1] + 1 + np.arange(8)])
    return dict(rows=rows, stored=stored(rows, bf16_rows), q=q, multiples=multiples, zero_score=zero_score,
                zero_rows=zero_rows)


def ends_ladder(scores):
    """The fixed ladder, plus the scores of the multiples and of +-0 with their neighbours."""
    fin = np.unique(scores[np.isfinite(scores) & (np.abs(scores) >= 0.99)])
    return list(FIXED_LADDER) + with_neighbours(list(fin) + [0.0, -0.0])
