"""CPU suite for min_score: the case builders of threshold_cases.py deliver what the GPU suite relies on, the oracle's
threshold semantics are pinned against oracle/pyref.py, and the host mirror resolves the reference's
`options.minScore || 0.5` / `options.topK || 10` with JavaScript's `||`, where NaN falls back to the default."""
import math

import numpy as np
import pytest

import threshold_cases as tc
from common import HashEmbedder, OracleIndex
from oracle import pyref


def bits(x):
    return np.float64(x).tobytes()


def live_within(scores, ms, eps):
    """How many scores lie in [ms - eps, ms) and in [ms, ms + eps]."""
    s = scores[np.isfinite(scores)]
    return int(((s >= ms - eps) & (s < ms)).sum()), int(((s >= ms) & (s <= ms + eps)).sum())


# --------------------------------------------------------------------------- the builders
@pytest.mark.parametrize("bf16_rows", [False, True], ids=["f64", "bf16"])
@pytest.mark.parametrize("d", [100, 1536])
def test_band_corpus_puts_rows_inside_the_bound_around_each_threshold(oracle_mod, d, bf16_rows):
    c = tc.band_corpus(d, bf16_rows, seed=d)
    for i, q in enumerate(c["q"]):
        sc = oracle_mod.scores(c["stored"], q)
        lad = tc.ladder(sc, c["band"][i], c["t"][i])
        assert len(lad) == 15
        # the base thresholds are score bytes, and each neighbour is one ulp away
        for j in range(0, 15, 3):
            assert np.any(sc.view(np.int64) == np.float64(lad[j]).view(np.int64)), (i, j)
            assert lad[j + 1] == np.nextafter(lad[j], -np.inf) and lad[j + 2] == np.nextafter(lad[j], np.inf)
        mid = lad[9]
        below, above = live_within(sc, mid, c["eps"][i])
        assert below >= 200 and above >= 200, (i, below, above, c["eps"][i])
        # the hits K and K + 1 sit among the band's top rows: many rows within the bound below them too
        assert live_within(sc, lad[3], c["eps"][i])[0] >= 50, i


@pytest.mark.parametrize("bf16_rows", [False, True], ids=["f64", "bf16"])
def test_tie_groups_tie_exactly_at_their_threshold(oracle_mod, bf16_rows):
    c = tc.tie_corpus(100, bf16_rows, seed=3)
    for g, size in enumerate(c["sizes"]):
        sc = oracle_mod.scores(c["stored"], c["q"][g])
        assert len(c["dup"][g]) == size
        assert (sc[c["dup"][g]].view(np.int64) == np.float64(c["ms"][g]).view(np.int64)).all()
        # exactly `above` rows score higher, and rows within the bound score just below
        assert int((sc > c["ms"][g]).sum()) == c["above"], g
        assert int(((sc < c["ms"][g]) & (sc >= c["ms"][g] - c["eps"][g])).sum()) >= 10, g


@pytest.mark.parametrize("bf16_rows", [False, True], ids=["f64", "bf16"])
def test_ends_corpus_scores(oracle_mod, bf16_rows):
    c = tc.ends_corpus(8, bf16_rows, seed=8, huge=not bf16_rows)
    for i, q in enumerate(c["q"]):
        sc = oracle_mod.scores(c["stored"], q)
        mine = c["multiples"][10 * i:10 * i + 10]
        pos, neg = sc[mine[:6]], sc[mine[6:]]
        # multiples by powers of two are exact in every tier: 1 / -1 or one ulp off; bf16 rounds the others
        exact = np.r_[pos[:3] - 1.0, neg[:2] + 1.0]
        assert (np.abs(exact) <= 2.0 ** -52).all(), (pos, neg)
        tol = 2.0 ** -52 if not bf16_rows else 1e-5
        assert (np.abs(pos - 1.0) <= tol).all() and (np.abs(neg + 1.0) <= tol).all(), (pos, neg)
        z = sc[c["zero_score"]]
        assert (z == 0.0).all()
        # the orthogonal rows: every product is +-0, the chain starts at +0, so the score is +0 (never -0)
        assert all(bits(v) == bits(0.0) for v in z[:12])
        if not bf16_rows:   # 2^600 rows: the squared norm overflows, dot / inf is +0 or -0 with the dot's sign
            assert {bits(v) for v in z[12:]} == {bits(0.0), bits(-0.0)}, z[12:]
        assert np.isnan(sc[c["zero_rows"]]).all()
        lad = tc.ends_ladder(sc)
        assert 1.0 in lad and -1.0 in lad and any(bits(v) == bits(-0.0) for v in lad)


# --------------------------------------------------------------------------- the oracle's threshold semantics
def py_scan(rows, q, k, ms):
    """pyref's cosine, then `>= ms` taken as given, stable sort, first k."""
    scored = [(i, pyref.cosine_similarity(q.tolist(), r.tolist())) for i, r in enumerate(rows)]
    scored = [h for h in scored if h[1] >= ms]
    scored.sort(key=lambda h: -h[1])
    return scored[:k]


def small_cases():
    """A small band corpus (pure Python must score it) and the ends corpus, as float64 rows."""
    band = tc.band_corpus(24, False, seed=24, per_band=60, n_random=200)
    ends = tc.ends_corpus(8, False, seed=8, huge=True)
    for c, lad in ((band, lambda sc, i: tc.ladder(sc, band["band"][i], band["t"][i])), (ends, lambda sc, i: [])):
        yield c, lad


def test_oracle_search_and_the_score_once_derivation_agree_with_pyref_at_every_threshold(oracle_mod):
    from runbookai_b200.vector_store import js_or
    for c, lad in small_cases():
        rows = c["rows"]
        for i, q in enumerate(c["q"]):
            sc = oracle_mod.scores(rows, q)
            py = np.array([pyref.cosine_similarity(q.tolist(), r.tolist()) for r in rows])
            assert [bits(v) if v == v else b"nan" for v in sc] == [bits(v) if v == v else b"nan" for v in py]
            ths = list(tc.FIXED_LADDER) + lad(sc, i) + tc.ends_ladder(sc)
            for ms in ths:
                s, v = oracle_mod.search(rows, q, 10 ** 6, ms)
                want = py_scan(rows, q, 10 ** 6, ms)
                assert s.tolist() == [h[0] for h in want] and [bits(x) for x in v] == [bits(h[1]) for h in want], ms
                hs, hv = tc.hits(sc, ms)
                assert hs.tolist() == s.tolist() and hv.tobytes() == v.tobytes(), ms
                hs, hv = tc.hits(sc, ms, 7)
                s7, v7 = oracle_mod.search(rows, q, 7, ms)
                assert hs.tolist() == s7.tolist() and hv.tobytes() == v7.tobytes(), ms
                # vector_scan resolves `minScore || 0.5` itself: the oracle at the resolved threshold
                top = [(int(a), float(b)) for a, b in pyref.vector_scan(q.tolist(), enumerate(rows.tolist()), 5, ms)]
                s10, v10 = oracle_mod.search(rows, q, 10, js_or(ms, 0.5))
                assert top == list(zip(s10.tolist(), v10.tolist())), ms
            # no threshold: every non-NaN score
            s, v = oracle_mod.search(rows, q, 10 ** 6, None)
            assert s.tolist() == tc.hits(sc, None)[0].tolist()


# --------------------------------------------------------------------------- JavaScript's ||
def test_js_or_follows_javascript():
    from runbookai_b200.vector_store import js_or
    for falsy in (None, 0, 0.0, -0.0, math.nan, np.nan, np.float64("nan"), False, ""):
        assert js_or(falsy, 0.5) == 0.5, falsy
        assert js_or(falsy, None, 10) == 10
    for truthy in (0.3, -1.0, 1.5, math.inf, -math.inf, 5e-324, 7, True, np.float64(0.25)):
        assert js_or(truthy, 0.5) is truthy
    assert js_or(math.nan, 0.2, 0.5) == 0.2 and js_or(None, None, 0.5) == 0.5
    assert math.isnan(js_or(0.2, math.nan)) is False and math.isnan(js_or(None, math.nan))


@pytest.fixture
def store(tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    s = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda dim, dev: OracleIndex(dim))
    texts = ["redis connection pool exhausted restart", "redis connection pool failover", "kubernetes pod crashloop",
             "pod oom killed restart", "postgres replication lag", "redis cache eviction storm"]
    for j, text in enumerate(texts * 5):
        s.add_chunks([{"chunk": {"id": f"c{j}", "documentId": f"d{j % 4}", "content": f"{text} step {j}",
                                 "sectionTitle": f"S{j}"}, "documentTitle": "T", "type": "runbook",
                       "services": ["api"]}])
    yield s
    s.close()
    embedder.reset()


def test_nan_min_score_and_top_k_fall_back_like_javascript(store):
    q = "redis connection pool exhausted"
    assert store.search(q, {"minScore": math.nan}) == store.search(q, {"minScore": 0.5})
    assert store.search(q, {"minScore": -0.0, "topK": -0.0}) == store.search(q, {})
    nan_k = store.search(q, {"topK": math.nan, "minScore": 0.05})
    assert nan_k == store.search(q, {"topK": 10, "minScore": 0.05}) and len(nan_k) == 10
    assert store.search(q, {"minScore": np.float64("nan"), "topK": np.nan}) == store.search(q, {})


def test_micro_batch_of_mixed_thresholds_answers_each_caller_as_its_own_search(store):
    import itertools
    from runbookai_b200.batcher import MicroBatcher
    q = "redis connection pool exhausted"
    hit = store.search(q, {"topK": 5, "minScore": 0.05})[2].score      # one caller's threshold is a hit's score
    asks = [(q, {"minScore": math.nan}), ("pod restart", {"minScore": -0.0, "topK": 3}), (q, {"minScore": 0.3}),
            ("redis failover", {"minScore": 1.5}), (q, {"minScore": hit, "topK": 5}),
            ("redis cache", {"minScore": math.nan, "topK": math.nan})]
    want = [store.search(a, o) for a, o in asks]
    assert want[4] and want[4][-1].score == hit
    orders = list(itertools.permutations(range(len(asks))))[::97]
    for order in orders:
        mb = MicroBatcher(store, window_ms=10_000.0, max_batch=len(asks))
        futs = {i: mb.submit(*asks[i]) for i in order}
        got = {i: f.result(timeout=30) for i, f in futs.items()}
        mb.close()
        assert mb.batches == 1, order
        assert [got[i] for i in range(len(asks))] == want, order
