"""CPU suite: the reference's cosine and sort at the ends of the float64 range, in the C oracle and in oracle/pyref.py.

The table in float_range_cases.py states what each class of vector scores against an ordinary one; here both
restatements must give exactly those kinds of number, agree bit for bit (+0 vs -0 included), and order +-Infinity and
+-0 ties the way the reference's comparator `b.score - a.score` does: Infinity - Infinity and 0 - 0 are not > 0, so
such ties keep slot order."""
import numpy as np
import pytest

from float_range_cases import KIND, SCALES, SPECIAL, matches, scaled, special
from oracle import pyref

D = 24


def bits(x):
    """The float64 bytes, so that -0 and +0 differ; every NaN is one value (JS has a single NaN, and a NaN score is
    never returned)."""
    x = np.float64(x)
    return b"nan" if np.isnan(x) else x.tobytes()


def py_search(rows, q, k, min_score):
    """pyref's findMostSimilar, or its VectorStore scan with min_score taken as given (vector_scan applies the
    reference's `minScore || 0.5`, which the oracle's callers have already resolved)."""
    emb = [(i, r.tolist()) for i, r in enumerate(rows)]
    if min_score is None:
        return pyref.find_most_similar(q.tolist(), emb, k)
    scored = [(i, pyref.cosine_similarity(q.tolist(), e)) for i, e in emb]
    scored = [h for h in scored if h[1] >= min_score]
    scored.sort(key=lambda h: -h[1])
    return scored[:k]


@pytest.mark.parametrize("e", sorted(SCALES))
def test_each_scale_scores_the_stated_kind_in_both_restatements(oracle_mod, e):
    rng = np.random.default_rng(2000 + e)
    base = rng.standard_normal((40, D))
    x = scaled(base[0], e)
    kind = KIND[SCALES[e]]
    for partner in base[1:]:
        for a, b in ((x, partner), (partner, x)):          # the class on the query side and on the row side
            c = oracle_mod.cosine(a, b)
            assert bits(c) == bits(pyref.cosine_similarity(a.tolist(), b.tolist()))
            assert matches(kind, c), (e, c)
    if kind == "finite":
        # powers of two scale exactly and the class is far from both ends: the direction, and so the cosine, is kept
        # up to the last bits of the chains
        want = np.array([oracle_mod.cosine(base[0], p) for p in base[1:]])
        got = np.array([oracle_mod.cosine(x, p) for p in base[1:]])
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 if -1000 < 2 * e < 1000 else 1.0)


@pytest.mark.parametrize("name", sorted(SPECIAL))
def test_special_vectors_score_nan(oracle_mod, name):
    rng = np.random.default_rng(7)
    x = special(rng.standard_normal(D), name)
    for p in rng.standard_normal((10, D)):
        for a, b in ((x, p), (p, x)):
            c = oracle_mod.cosine(a, b)
            assert np.isnan(c) and np.isnan(pyref.cosine_similarity(a.tolist(), b.tolist()))


def test_underflowing_norm_gives_signed_infinities_and_overflowing_norm_signed_zeros(oracle_mod):
    """The pyref comment "only 0/0 can occur" was wrong: x/0 with x != 0 occurs when a norm underflows."""
    q = np.zeros(D)
    q[0], q[1] = 1.0, -1.0
    tiny = scaled(q, -565)
    row_pos, row_neg = np.eye(D)[0], np.eye(D)[1]
    assert oracle_mod.cosine(tiny, row_pos) == np.inf
    assert oracle_mod.cosine(tiny, row_neg) == -np.inf
    assert np.isnan(oracle_mod.cosine(tiny, np.eye(D)[2]))          # 0 / 0
    huge = scaled(q, 600)
    assert bits(oracle_mod.cosine(huge, row_pos)) == bits(0.0)
    assert bits(oracle_mod.cosine(huge, row_neg)) == bits(-0.0)
    assert bits(pyref.cosine_similarity(huge.tolist(), row_neg.tolist())) == bits(-0.0)


def tie_corpus(rng):
    """Rows that a 2^-565 query scores +Infinity, -Infinity, NaN and finite-but-never (none: its norm is 0), and rows
    at 2^600 that an ordinary query scores +0 and -0, interleaved so every tie spans several slots."""
    q = rng.standard_normal(D)
    rows = []
    for i in range(30):
        r = rng.standard_normal(D)
        kind = i % 5
        if kind == 0:
            r = scaled(np.abs(r) * np.sign(q), 600)        # dot > 0 with q, norm overflows: +0
        elif kind == 1:
            r = scaled(-np.abs(r) * np.sign(q), 600)       # -0
        elif kind == 2:
            r = np.zeros(D)                                # NaN: dropped
        rows.append(r)
    return q, np.array(rows)


@pytest.mark.parametrize("min_score", [None, -1.0, 0.0, 0.5])
@pytest.mark.parametrize("k", [1, 7, 30])
def test_signed_zero_and_infinity_ties_keep_slot_order(oracle_mod, min_score, k):
    rng = np.random.default_rng(k)
    q, rows = tie_corpus(rng)
    for query in (q, scaled(q, -565)):                       # ordinary query: +-0 ties; tiny query: +-Infinity ties
        s, v = oracle_mod.search(rows, query, k, min_score)
        ref = py_search(rows, query, k, min_score)
        assert s.tolist() == [h[0] for h in ref]
        assert [bits(x) for x in v] == [bits(h[1]) for h in ref]
        # the order itself: scores never increase, and equal scores (+0 == -0, inf == inf) go by slot
        for i in range(len(s) - 1):
            assert v[i] >= v[i + 1]
            if v[i] == v[i + 1]:
                assert s[i] < s[i + 1]
        if min_score is not None:
            assert all(x >= min_score for x in v)
    # an ordinary query: every 2^600 row scores +-0, and -0 and +0 tie
    s, v = oracle_mod.search(rows, q, 30, None)
    zeros = [int(x) for x, y in zip(s, v) if y == 0.0]
    assert zeros == sorted(zeros) and len(zeros) >= 12
    assert {bits(y) for y in v if y == 0.0} == {bits(0.0), bits(-0.0)}


def test_tiny_query_ranks_every_positive_dot_first_by_slot(oracle_mod):
    """A query whose normA underflows scores +Infinity on every row with a positive dot: findMostSimilar returns the
    lowest such slots, whatever the rows' real angles."""
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((200, D))
    q = scaled(rows[150], -565)
    s, v = oracle_mod.search(rows, q, 10, None)
    pos = [i for i in range(200) if float(np.dot(rows[i], rows[150])) > 0]
    assert s.tolist() == pos[:10] and (v == np.inf).all()
    s2, v2 = oracle_mod.search(rows, q, 10, 0.5)
    assert s2.tolist() == s.tolist()


@pytest.mark.parametrize("e", [-1074, -565, -140, 130, 600])
def test_batch_checkers_agree_with_the_literal_search_at_extreme_queries(oracle_mod, e):
    """search_batch_verify (the checker of large GPU runs) hoists the norms: at the range ends too it must give the
    literal search's bits."""
    from runbookai_b200 import synth
    rng = np.random.default_rng(abs(e))
    rows32 = rng.standard_normal((500, D)).astype(np.float32)
    rows = synth.bf16_round(rows32)
    rows_f64 = rows.astype(np.float64)
    bits16 = (rows.view(np.uint32) >> 16).astype(np.uint16)
    q = scaled(rng.standard_normal((5, D)), e)
    for ms in (None, 0.0, 0.5):
        vs, vv, vc = oracle_mod.search_batch_verify(bits16, q, 12, ms)
        for b in range(len(q)):
            s, v = oracle_mod.search(rows_f64, q[b], 12, ms)
            assert vc[b] == len(s) and vs[b, :len(s)].tolist() == s.tolist()
            assert vv[b, :len(s)].tobytes() == v.tobytes()
