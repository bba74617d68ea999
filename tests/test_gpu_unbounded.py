"""GPU suite (-m gpu) for the unbounded search (rbk_index_search_unbounded_f64 / rbk_group_search_unbounded_f64, any
k_fetch): the large-k search's two scans, then the candidates sorted in global memory.  Bar, against the oracle: ids
identical, fp64 scores bit-identical, tail -1 / NaN."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def check(got, es, ev, ec):
    slots, scores, counts, _ = got
    assert slots.shape == es.shape
    assert (counts == ec).all(), (counts, ec)
    for b in range(len(ec)):
        n = ec[b]
        assert (slots[b, :n] == es[b, :n]).all(), b
        assert scores[b, :n].tobytes() == ev[b, :n].tobytes(), b          # bit-exact fp64
        assert (slots[b, n:] == -1).all() and np.isnan(scores[b, n:]).all()


def oracle(oracle_mod, corpus, q, k, ms, live=None, base=0):
    """(slots, scores, counts) [B, k] of the reference; corpus: bf16 bits (uint16) or float64 rows."""
    if corpus.dtype == np.uint16:
        es, ev, ec = oracle_mod.search_batch_mt(corpus, np.asarray(q, np.float64), k, ms, live=live)
    else:
        B = q.shape[0]
        es = np.full((B, k), -1, np.int64)
        ev = np.full((B, k), np.nan)
        ec = np.zeros(B, np.int32)
        for b in range(B):
            s, v = oracle_mod.search(corpus, q[b], k, ms, live=live)
            es[b, :len(s)], ev[b, :len(s)], ec[b] = s, v, len(s)
    es = np.where(es >= 0, es + base, es)
    return es, ev, ec


def bit_equal(a, b):
    return (a[0] == b[0]).all() and a[1].tobytes() == b[1].tobytes() and (a[2] == b[2]).all()


BASE = 1_000_003   # slot_base of the bf16 index: every returned slot is global


@pytest.fixture(scope="module")
def corpora(rb):
    """A bf16-exact corpus with a nonzero slot_base and an index of arbitrary float64 rows (keep_f64), both with
    tombstones, a zero row, a zero query and planted neighbours (so that min_score 0.5 keeps thousands of rows)."""
    from runbookai_b200 import synth
    out = []
    n, d = 30_000, 256
    corpus = synth.random_corpus(n, d, 401)
    q = synth.random_queries(5, d, 402).astype(np.float64)
    synth.plant_neighbours(corpus, q.astype(np.float32), 1500, 403)
    corpus[7] = 0
    q[3] = 0.0
    dead = np.random.default_rng(404).choice(n, n // 20, replace=False)
    live = np.ones(n, np.uint8)
    live[dead] = 0
    ix = rb.Index(d)
    ix.set_slot_base(BASE)
    ix.append_bf16(corpus)
    ix.tombstone(dead)
    out.append(("bf16", ix, corpus, q, live, BASE))
    rng = np.random.default_rng(405)
    n, d = 12_000, 100
    q = rng.standard_normal((5, d))
    corpus = rng.standard_normal((n, d))
    corpus[:6000] += 1.5 * q[0]                                      # thousands of rows above 0.5 for query 0
    corpus[11] = 0
    q[3] = 0.0
    dead = rng.choice(n, 500, replace=False)
    live = np.ones(n, np.uint8)
    live[dead] = 0
    ix = rb.Index(d, keep_f64=True)
    ix.append_f64(corpus)
    ix.tombstone(dead)
    out.append(("f64", ix, corpus, q, live, 0))
    yield out
    for c in out:
        c[1].close()


@pytest.mark.parametrize("B", [1, 5])
@pytest.mark.parametrize("min_score", [None, 0.0, 0.5])
@pytest.mark.parametrize("k", ["4097", "9000", "above_count"])
def test_unbounded_matches_oracle(rb, oracle_mod, corpora, k, min_score, B):
    for kind, ix, corpus, q, live, base in corpora:
        kf = ix.count() + 777 if k == "above_count" else int(k)
        qq = q if B == 5 else (q[3:4] if kind == "bf16" else q[0:1])     # B = 1: the zero query, or query 0
        got = ix.search_unbounded(qq, kf, min_score)
        check(got, *oracle(oracle_mod, corpus, qq, kf, min_score, live=live, base=base))
        zero = 7 if kind == "bf16" else 11
        assert not np.isin(zero + base, got[0])                          # the zero row never matches
        if B == 5:
            assert got[2][3] == 0                                        # nor does the zero query


@pytest.mark.parametrize("k", [10_000, 15_000])
def test_tie_group_spanning_several_tiles(rb, oracle_mod, k):
    """12000 rows with exactly the same cosine (power-of-two multiples of the query: the fp64 arithmetic scales
    exactly) span three sort tiles and straddle the k-th position: they must come out in slot order, cut exactly."""
    from runbookai_b200 import synth
    n, d = 60_000, 128
    corpus = synth.random_corpus(n, d, 411)
    q = synth.bf16_round(synth.random_queries(2, d, 412)).astype(np.float64)
    rng = np.random.default_rng(413)
    dup = np.sort(rng.choice(n, 12_000, replace=False))
    scale = np.exp2(rng.integers(-3, 4, len(dup)))[:, None]
    corpus[dup] = synth.f32_to_bf16_bits((q[0] * scale).astype(np.float32))
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        for ms in (None, 0.5):
            got = ix.search_unbounded(q, k, ms)
            check(got, *oracle(oracle_mod, corpus, q, k, ms))
            assert len(set(got[1][0, :len(dup)].tolist())) == 1                 # one tie group ...
            assert (got[0][0, :min(k, len(dup))] == dup[:k]).all()              # ... in slot order


def test_agrees_with_the_large_k_search_and_the_exact_scores_route(rb, corpora):
    from runbookai_b200 import _native
    for kind, ix, corpus, q, live, base in corpora:
        for ms in (None, 0.5):
            for k in (200, 4096):
                assert bit_equal(ix.search_unbounded(q, k, ms), ix.search_large(q, k, ms))
            for k in (4097, 7000, ix.size() + 1):
                got = ix.search_unbounded(q, k, ms)
                old = _native._search_any_k(ix, q, k, ms)                     # exact scores + the host cut
                old_slots = np.where(old[0] >= 0, old[0] + base, old[0])
                assert (got[0] == old_slots).all() and got[1].tobytes() == old[1].tobytes() and (got[2] == old[2]).all()


def test_batch_split_into_query_groups(rb, oracle_mod):
    """200k rows x 48 queries x k_fetch 200k: the candidates and results (~8 MB per query) exceed the per-pass budget,
    so the batch is answered in several query groups - one emit scan each - and stays exact.  The groups start at
    queries that are not multiples of the scan's 128-query block (33 per group on an index, 18 on a one-GPU group);
    each group's scan must stay inside the query buffer, which the library checks before every launch.  Then the same
    for the large-k search at k_fetch 4096."""
    from runbookai_b200 import _native, synth
    n, d, B, k = 200_000, 64, 48, 200_000
    corpus = synth.random_corpus(n, d, 421)
    q = synth.random_queries(B, d, 422).astype(np.float64)
    with rb.Index(d) as ix, rb.Group(d, [0]) as g:
        ix.append_bf16(corpus)
        g.append_bf16(corpus)
        before = ix.stats()["scan_launches"]
        got = ix.search_unbounded(q, k, None)
        launches = ix.stats()["scan_launches"] - before
        assert launches >= 3, launches                                   # one count scan, at least two emit scans
        # every query against the exact-scores route (fp64 scores of every row, host cut), bit for bit; queries on
        # both sides of the group boundaries against the oracle (at k_fetch 200k it costs seconds per query)
        assert bit_equal(got, _native._search_any_k(ix, q, k, None))
        pick = [0, 17, 18, 32, 33, 47]
        check(tuple(a[pick] for a in got[:3]) + (0.0,), *oracle(oracle_mod, corpus, q[pick], k, None))
        before = g.stats()["scan_launches"]
        assert bit_equal(g.search_unbounded(q, k, None), got)
        assert g.stats()["scan_launches"] - before >= 3
    # The large-k search (k_fetch <= 4096, the cut in shared memory) keeps the same budget: 1M rows that are all
    # power-of-two multiples of one direction tie for every query along it (the fp64 arithmetic scales exactly), so
    # C_q = n and 32 queries' candidates (12 bytes each, ~380 MB) need two query groups.
    n, B, k = 1_000_000, 32, 4096
    rng = np.random.default_rng(423)
    u = synth.bf16_round(synth.random_queries(1, d, 424)[0]).astype(np.float64)
    scale = np.exp2(rng.integers(-3, 4, n))[:, None]
    corpus = synth.f32_to_bf16_bits((u * scale).astype(np.float32))
    q = u * np.exp2(rng.integers(-2, 3, B))[:, None]
    want = oracle(oracle_mod, corpus, q, k, None)
    with rb.Index(d) as ix, rb.Group(d, [0]) as g:
        for h in (ix, g):
            h.append_bf16(corpus)
            before = h.stats()["scan_launches"]
            got = h.search_large(q, k, None)
            assert h.stats()["scan_launches"] - before >= 3                # one count scan, at least two emit scans
            check(got, *want)


def test_host_rows_equal_device_rows(rb):
    rng = np.random.default_rng(431)
    n, d = 15_000, 96
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((4, d))
    rows[:5000] += q[1]
    over = rng.choice(n, 300, replace=False)
    dead = np.setdiff1d(rng.choice(n, 700, replace=False), over)
    with rb.Index(d, keep_f64=True) as dev, rb.Index(d, keep_f64=True, f64_on_host=True) as host:
        for ix in (dev, host):
            ix.append_f64(rows)
            ix.overwrite_f64_batch(over, rows[over] * 0.5 + q[2])
            ix.tombstone(dead)
        for k, ms in ((5000, None), (9000, 0.0), (20_000, 0.1)):
            assert bit_equal(dev.search_unbounded(q, k, ms), host.search_unbounded(q, k, ms))


def test_after_compact_clear_and_on_an_empty_index(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d = 20_000, 192
    corpus = synth.random_corpus(n, d, 441)
    q = synth.random_queries(3, d, 442).astype(np.float64)
    with rb.Index(d) as ix:
        s, v, c, _ = ix.search_unbounded(q, 5000, None)                   # empty index
        assert (c == 0).all() and (s == -1).all() and np.isnan(v).all()
        ix.append_bf16(corpus)
        dead = np.arange(0, n, 3)
        ix.tombstone(dead)
        live = np.ones(n, np.uint8)
        live[dead] = 0
        check(ix.search_unbounded(q, 6000, 0.0), *oracle(oracle_mod, corpus, q, 6000, 0.0, live=live))
        ix.compact()
        packed = corpus[live.astype(bool)]
        for k, ms in ((6000, 0.0), (20_000, None)):
            check(ix.search_unbounded(q, k, ms), *oracle(oracle_mod, packed, q, k, ms))
        ix.clear()
        s, v, c, _ = ix.search_unbounded(q, 5000, None)
        assert (c == 0).all() and (s == -1).all() and np.isnan(v).all()
        ix.append_bf16(corpus[:8000])                                    # appends after clear start at slot 0
        check(ix.search_unbounded(q, 7000, None), *oracle(oracle_mod, corpus[:8000], q, 7000, None))


def test_one_gpu_group_equals_a_single_index(rb):
    from runbookai_b200 import synth
    n, d = 40_000, 128
    corpus = synth.random_corpus(n, d, 451)
    q = synth.random_queries(5, d, 452).astype(np.float64)
    dead = np.arange(0, n, 13)
    with rb.Group(d, [0]) as g, rb.Index(d) as ix:
        for h in (g, ix):
            h.append_bf16(corpus)
            h.tombstone(dead)
        for k, ms in ((4097, None), (12_000, 0.0), (n + 10, None)):
            assert bit_equal(g.search_unbounded(q, k, ms), ix.search_unbounded(q, k, ms))
        assert bit_equal(g.search_any_k(q, 6000, None), ix.search_any_k(q, 6000, None))


def test_two_gpu_group_equals_a_single_index(rb):
    from common import group_devices
    from runbookai_b200 import synth
    n, d = 50_000, 128
    corpus = synth.random_corpus(n, d, 461)
    q = synth.random_queries(4, d, 462).astype(np.float64)
    with rb.Group(d, group_devices(2)) as g, rb.Index(d) as ix:
        for h in (g, ix):
            h.append_bf16(corpus)
            h.tombstone(np.arange(5, n, 17))
        for k, ms in ((5000, None), (30_000, 0.0)):
            assert bit_equal(g.search_unbounded(q, k, ms), ix.search_unbounded(q, k, ms))


def test_vector_store_top_k_3000_stays_on_the_gpu(rb, tmp_path, monkeypatch):
    from common import HashEmbedder, OracleIndex
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    try:
        words = [f"w{i}" for i in range(60)]
        rng = np.random.default_rng(471)
        chunks = [{"chunk": {"id": f"c{i}", "documentId": f"d{i % 40}",
                             "content": " ".join(rng.choice(words, 6)), "sectionTitle": "s"},
                   "documentTitle": f"D{i % 40}", "type": "runbook", "services": []} for i in range(8000)]
        gpu = VectorStore(str(tmp_path / "g.db"))
        cpu = VectorStore(str(tmp_path / "c.db"), index_factory=lambda dim, dev: OracleIndex(dim))
        gpu.add_chunks(chunks)
        cpu.add_chunks(chunks)
        monkeypatch.setattr(rb.Index, "exact_scores",
                            lambda self, q: (_ for _ in ()).throw(AssertionError("host route")))
        for query in ("w1 w2 w3", "w10 w40"):
            a = gpu.search(query, {"topK": 3000, "minScore": -1.0})        # every chunk passes: 2*topK = 6000 hits
            b = cpu.search(query, {"topK": 3000, "minScore": -1.0})
            assert len(a) == 3000
            assert [(r.id, r.score) for r in a] == [(r.id, r.score) for r in b]
        gpu.close()
        cpu.close()
    finally:
        embedder.reset()


def test_errors(rb):
    from runbookai_b200 import _native
    from runbookai_b200 import synth
    d = 64
    q = synth.random_queries(2, d, 481).astype(np.float64)
    with rb.Index(d) as ix, rb.Group(d, [0]) as g:
        ix.append_bf16(synth.random_corpus(5000, d, 482))
        g.append_bf16(synth.random_corpus(5000, d, 482))
        for h, fn in ((ix, _native.lib.rbk_index_search_unbounded_f64), (g, _native.lib.rbk_group_search_unbounded_f64)):
            with pytest.raises(rb.RbkError) as e:
                h.search_unbounded(q, 0, None)
            assert e.value.status == _native.RBK_EINVAL
            with pytest.raises(rb.DimensionError, match="Vectors must have the same length") as e:
                h.search_unbounded(np.zeros((1, d + 1)), 5000, None)
            assert e.value.status == _native.RBK_EDIM
            with pytest.raises(rb.RbkError, match="NaN"):
                h.search_unbounded(q, 5000, float("nan"))
            ms = C.c_float(0)
            st = fn(h._h, _native.ptr(q), 2, d, 5000, 0.0, None, None, None, C.byref(ms))
            assert st == _native.RBK_EINVAL and b"null output" in _native.lib.rbk_last_error()
        with pytest.raises(rb.RbkError, match=r"\[1, 4096\]"):          # the large-k search keeps its limit
            ix.search_large(q, 4097, None)
