"""CPU suite for tests/test_gpu_search_each_matrix.py: its per-query expectation against the C oracle's own search and
oracle/pyref.py, and its batch builders against what the GPU tests rely on - ladders inside each query's own band, k mixes
that reach both branches of the finalize proof, batches that straddle query 1024 with no period dividing 1024, failing
queries that are not a prefix, and a budget-split case that needs more than one query group."""
import numpy as np
import pytest

import threshold_cases as tc
from oracle import pyref
from test_gpu_exact_paths import sweep_corpus
from test_gpu_search_each_matrix import (BUDGET_SPLIT, LARGE_K, SCAN_K, SEAM, SUB_BATCH, LadderBatch, budget_groups,
                                         draw, expected, fallback_batch, group_result_cost)
from test_gpu_thresholds import Oracle


@pytest.fixture(scope="module")
def band(oracle_mod):
    c = tc.band_corpus(100, False, seed=110)
    orc = Oracle(oracle_mod, c["stored"])
    return c, orc, [orc.scores(q) for q in c["q"]]


def test_expectation_is_the_oracle_search(oracle_mod):
    """Every (k, m) the matrix uses, k above count() and thresholds of +-0, +-inf and a hit's exact bytes: the block
    builder's row b equals oracle.search and pyref's cosine ordering, padded with -1 and quiet NaN."""
    rng = np.random.default_rng(1)
    d, n = 8, 120
    rows = rng.standard_normal((n, d))
    rows[5] = 0.0                                   # a NaN row
    rows[7] = rows[9]                               # a tie
    live = np.ones(n, np.uint8)
    live[::11] = 0
    q = rng.standard_normal((6, d))
    orc = Oracle(oracle_mod, rows, live)
    hit = float(orc.hits(q[0], None)[1][3])
    ths = [None, -np.inf, np.inf, 0.0, -0.0, hit, float(np.nextafter(hit, 2.0)), 0.5]
    ks = [1, 3, 56, 112, 113, 1000, n + 7]
    B = len(ths) * len(ks)
    qi = np.array(draw(rng, B, list(range(len(q)))))
    kk = [ks[p % len(ks)] for p in range(B)]
    mm = [ths[(p // len(ks)) % len(ths)] for p in range(B)]
    es, ev, ec = expected(orc, q[qi], kk, mm)
    assert es.shape == (B, max(ks))
    for b in range(B):
        s, v = oracle_mod.search(rows, q[qi[b]], kk[b], mm[b], live=live)
        c = len(s)
        assert ec[b] == c and (es[b, :c] == s).all() and ev[b, :c].tobytes() == v.tobytes(), b
        assert (es[b, c:] == -1).all() and (ev[b, c:].view(np.uint64) == 0x7FF8000000000000).all(), b
        ref = [(i, pyref.cosine_similarity(list(q[qi[b]]), list(rows[i]))) for i in range(n) if live[i]]
        ref = [(i, x) for i, x in ref if x == x and (mm[b] is None or x >= mm[b])]
        ref.sort(key=lambda e: -e[1])
        ref = ref[:kk[b]]
        assert [i for i, _ in ref] == s.tolist() and np.array([x for _, x in ref]).tobytes() == v.tobytes(), b


@pytest.mark.parametrize("route", ["scan", "large"])
def test_ladders_sit_in_their_own_band(band, route):
    """Every rung of every query's ladder at a k within its band rows lies within 3 eps (and one ulp) of its own band
    centre, and each position's thresholds are its own query's."""
    c, orc, scores = band
    kc = SCAN_K if route == "scan" else LARGE_K
    lb = LadderBatch(np.random.default_rng(3), scores, SEAM, kc, c["band"], c["t"])
    per_band = min(len(b) for b in c["band"])
    for (i, k), lad in lb.ladders.items():
        assert len(lad) == lb.L == 15
        if k < per_band:
            lo, hi = c["t"][i] - 3 * c["eps"][i], c["t"][i] + 3 * c["eps"][i]
            assert all(np.nextafter(lo, -1.0) <= x <= np.nextafter(hi, 2.0) for x in lad), (i, k)
    for call in (0, 7):
        ms = lb.ms(call)
        for p in range(0, SEAM, 37):
            assert ms[p] in lb.ladders[(lb.qi[p], lb.ks[p])]


def test_k_mix_reaches_both_proof_branches(band):
    """On the scan route some positions end with count == k (the k-th hit's proof) and some with count < k (the
    threshold's), in the same calls."""
    c, orc, scores = band
    lb = LadderBatch(np.random.default_rng(3), scores, SEAM, SCAN_K, c["band"], c["t"])
    full = short = 0
    for call in range(lb.L):
        _, _, ec = expected(orc, c["q"][lb.qi], lb.ks, lb.ms(call))
        full += int((ec == lb.ks).sum())
        short += int((ec < lb.ks).sum())
    assert full > 1000 and short > 1000, (full, short)


@pytest.mark.parametrize("kc", [SCAN_K, LARGE_K])
def test_batches_straddle_1024_without_a_period(band, kc):
    c, orc, scores = band
    lb = LadderBatch(np.random.default_rng(5), scores, SEAM, kc, c["band"], c["t"])
    assert len(lb.qi) == SEAM > SUB_BATCH
    for call in (0, 1, 14):
        key = list(zip(lb.qi.tolist(), lb.ks.tolist(), lb.ms(call)))
        assert all(key[p] != key[p + 1] for p in range(SEAM - 1)), "adjacent positions must differ"
        for period in (2 ** e for e in range(10)):
            assert any(key[p] != key[p + period] for p in range(SEAM - period)), period
        # the first sub-batch's (k, m) are not the second's shifted by 1024
        assert key[SUB_BATCH:] != key[:SEAM - SUB_BATCH]
    ks = draw(np.random.default_rng(0), SEAM, list(kc))
    assert sorted(set(ks)) == sorted(kc) and any(ks[p] != ks[p + 4] for p in range(SEAM - 4))


def test_failing_queries_are_scattered(oracle_mod):
    """The mostly-falling-back batch: more than half its positions must fall back, and they are not a prefix."""
    for d in (511, 512):
        rng, rows, wide, narrow = sweep_corpus(d, 300 + d)
        q, ks, ms, must = fallback_batch(rng, d, rows, wide, SEAM)
        assert len(q) == len(ks) == len(ms) == SEAM
        assert len(must) > SEAM // 2
        assert must.tolist() != list(range(len(must))) and must[0] > 0
        assert (must >= SUB_BATCH).any() and len(set(ks)) > 50


def test_budget_split_needs_several_query_groups():
    """By search_large's cost formula (result blocks alone, before any candidate), the group case needs more than one
    query group, and so does the index case."""
    G, B, K = BUDGET_SPLIT["G"], BUDGET_SPLIT["B"], BUDGET_SPLIT["K"]
    assert B <= SUB_BATCH          # one count scan per member: every further scan is a query group's emit scan
    groups = budget_groups([group_result_cost(G, K)] * B)
    assert len(groups) > 1 and groups[0][0] == 0 and groups[-1][1] == B
    n = 20000
    assert len(budget_groups([16 * n + 8] * 900)) > 1
    assert budget_groups([10] * 5) == [(0, 5)]
