"""GPU suite (-m gpu) for compaction (rbk_index_compact): old_to_new, the stored rows, and every search answer before
and after, through the map (slots and fp64 scores bit for bit) and against the oracle on the surviving rows."""
import ctypes as C
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KS = (1, 20, 112)
LARGE_KS = (500, 4096)
MIN_SCORES = (None, 0.05, 0.5)


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def dead_slots(pattern, n, rng):
    if pattern == "random40":
        return np.flatnonzero(rng.random(n) < 0.4)
    if pattern == "tiles":                    # whole 256-row tiles, and a partial one at the end
        return np.concatenate([np.arange(256, 512), np.arange(1024, 1536), np.arange(n - 100, n)])
    if pattern == "first_last":
        return np.array([0, n - 1])
    if pattern == "all_but_one":
        return np.setdiff1d(np.arange(n), [n // 2])
    if pattern == "all":
        return np.arange(n)
    return np.zeros(0, np.int64)             # none


def expected_map(live):
    keep = live.astype(bool)
    return np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int64)


def all_answers(ix, q):
    """Every search shape the suite compares: (k, min_score, query dtype) -> (slots, scores, counts)."""
    out = {}
    for k in KS:
        for ms in MIN_SCORES:
            out[(k, ms, "f64")] = ix.search(q, k, ms)[:3]
            out[(k, ms, "f32")] = ix.search(q.astype(np.float32), k, ms)[:3]
    for k in LARGE_KS:
        for ms in (None, 0.05):
            out[(k, ms, "large")] = ix.search_large(q, k, ms)[:3]
    return out


def assert_same_through_map(before, after, old_to_new, base=0):
    for key, (s0, v0, c0) in before.items():
        s1, v1, c1 = after[key]
        assert (c0 == c1).all(), key
        for b in range(len(c0)):
            n = c0[b]
            assert (old_to_new[s0[b, :n] - base] + base == s1[b, :n]).all(), (key, b)
            assert v0[b, :n].tobytes() == v1[b, :n].tobytes(), (key, b)
            assert (s1[b, n:] == -1).all() and np.isnan(v1[b, n:]).all()


def check_oracle(got, ref):
    slots, scores, counts = got
    es, ev, ec = ref
    assert (counts == ec).all(), (counts, ec)
    for b in range(len(ec)):
        n = ec[b]
        assert (slots[b, :n] == es[b, :n]).all(), b
        assert scores[b, :n].tobytes() == ev[b, :n].tobytes(), b


@pytest.mark.parametrize("pattern", ["random40", "tiles", "first_last", "all_but_one", "all", "none"])
def test_compaction_patterns(rb, oracle_mod, pattern):
    from runbookai_b200 import synth
    n, d = 3000, 200
    rng = np.random.default_rng(len(pattern))
    corpus = synth.random_corpus(n, d, 7)
    q = synth.random_queries(6, d, 8).astype(np.float64)
    synth.plant_neighbours(corpus, q.astype(np.float32), 30, 9)
    corpus[5] = 0                                                     # a zero row is live and keeps its place
    dead = dead_slots(pattern, n, rng)
    live = np.ones(n, np.uint8)
    live[dead] = 0
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        ix.tombstone(dead)
        before = all_answers(ix, q)
        old_to_new = ix.compact()
        assert (old_to_new == expected_map(live)).all()
        assert ix.size() == ix.count() == live.sum()
        assert (ix.read_rows_bf16(0, ix.size()) == corpus[live.astype(bool)]).all()
        after = all_answers(ix, q)
        assert_same_through_map(before, after, old_to_new)
        survivors = corpus[live.astype(bool)]
        if len(survivors) == 0:
            assert all((c == 0).all() for _, _, c in after.values())
        else:
            for k in KS:
                for ms in MIN_SCORES:
                    check_oracle(after[(k, ms, "f64")], oracle_mod.search_batch_mt(survivors, q, k, ms))
            check_oracle(after[(500, 0.05, "large")], oracle_mod.search_batch_mt(survivors, q, 500, 0.05))
        again = ix.compact()                                           # nothing left: the identity, nothing moves
        assert (again == np.arange(ix.size())).all()
        assert_same_through_map(after, all_answers(ix, q), again)


@pytest.mark.parametrize("d", [100, 67])
def test_keep_f64_rows_move_bit_exactly(rb, oracle_mod, d):
    rng = np.random.default_rng(d)
    n = 5000
    corpus = rng.standard_normal((n, d))
    corpus[9] = 0.0
    q = rng.standard_normal((4, d))
    dead = np.concatenate([np.arange(s, s + rng.integers(8, 41)) for s in rng.choice(n - 40, 80, replace=False)])
    live = np.ones(n, np.uint8)
    live[dead] = 0
    keep = live.astype(bool)
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(corpus)
        ix.tombstone(np.unique(dead))
        ex0 = ix.exact_scores(q)
        before = all_answers(ix, q)
        old_to_new = ix.compact()
        ex1 = ix.exact_scores(q)
        assert ex1.shape == (4, keep.sum())
        assert ex1.tobytes() == ex0[:, keep].tobytes()                 # the f64 rows and norms moved bit for bit
        assert_same_through_map(before, all_answers(ix, q), old_to_new)
        for k in (20, 112):
            got = ix.search(q, k, 0.05)[:3]
            es = np.full((4, k), -1, np.int64)
            ev = np.full((4, k), np.nan)
            ec = np.zeros(4, np.int32)
            for b in range(4):
                s, v = oracle_mod.search(corpus[keep], q[b], k, 0.05)
                es[b, :len(s)], ev[b, :len(s)], ec[b] = s, v, len(s)
            check_oracle(got, (es, ev, ec))


def test_planted_ties_across_dead_regions_keep_slot_order(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d = 4000, 128
    corpus = synth.random_corpus(n, d, 21)
    tie_slots = np.array([3, 255, 256, 700, 1500, 2047, 2048, 3999])
    corpus[tie_slots] = corpus[3]
    dead = np.concatenate([np.arange(4, 255), np.arange(300, 690), np.arange(1600, 2000), np.arange(2100, 3990)])
    live = np.ones(n, np.uint8)
    live[dead] = 0
    q = np.stack([synth.bf16_bits_to_f32(corpus[3])] * 3).astype(np.float64)
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        ix.tombstone(dead)
        s0 = ix.search(q, 20, 0.5)[0]
        old_to_new = ix.compact()
        s1, v1, c1, _ = ix.search(q, 20, 0.5)
        assert (s1[0, :len(tie_slots)] == old_to_new[tie_slots]).all()   # ascending slots, as before
        assert (np.diff(s1[0, :len(tie_slots)]) > 0).all()
        assert (old_to_new[s0[0, :c1[0]]] == s1[0, :c1[0]]).all()
        check_oracle((s1, v1, c1), oracle_mod.search_batch_mt(corpus[live.astype(bool)], q, 20, 0.5))


def test_large_corpus_takes_many_staging_chunks(rb, oracle_mod):
    """200k x 1536 KEEP_F64 (about 4.3k rows per 64 MB staging chunk): 46 chunks, half the rows deleted in document
    runs of 8-40 slots."""
    from runbookai_b200 import synth
    n, d = 200_000, 1536
    rng = np.random.default_rng(31)
    corpus = synth.random_corpus(n, d, 32)
    q = synth.random_queries(64, d, 33).astype(np.float64)
    synth.plant_neighbours(corpus, q.astype(np.float32), 40, 34)
    live = np.ones(n, np.uint8)
    s = 0
    while s < n:
        run = int(rng.integers(8, 41))
        if rng.random() < 0.5:
            live[s:s + run] = 0
        s += run
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_bf16(corpus)
        ix.tombstone(np.flatnonzero(live == 0))
        before = {(20, "f64"): ix.search(q, 20, 0.05)[:3], (1000, "large"): ix.search_large(q[:8], 1000, 0.05)[:3]}
        old_to_new = ix.compact()
        assert (old_to_new == expected_map(live)).all() and ix.size() == live.sum()
        after = {(20, "f64"): ix.search(q, 20, 0.05)[:3], (1000, "large"): ix.search_large(q[:8], 1000, 0.05)[:3]}
        assert_same_through_map(before, after, old_to_new)
        keep = live.astype(bool)
        assert (ix.read_rows_bf16(0, 1000) == corpus[keep][:1000]).all()
        assert (ix.read_rows_bf16(ix.size() - 1000, 1000) == corpus[keep][-1000:]).all()
        check_oracle(after[(20, "f64")], oracle_mod.search_batch_mt(corpus[keep], q, 20, 0.05))


def test_mutations_after_compaction_and_a_slot_base(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d, base = 3000, 96, 1_000_000
    corpus = synth.random_corpus(n, d, 41)
    extra = synth.random_corpus(500, d, 42)
    q = synth.random_queries(5, d, 43).astype(np.float64)
    rows = list(corpus)
    live = [True] * n
    with rb.Index(d) as ix:
        ix.set_slot_base(base)
        ix.append_bf16(corpus)
        dead = np.arange(0, n, 3)
        ix.tombstone(dead)
        for s in dead:
            live[s] = False
        before = ix.search(q, 30, None)[:3]
        m = ix.compact()
        assert_same_through_map({"a": before}, {"a": ix.search(q, 30, None)[:3]}, m, base=base)
        rows = [r for r, l in zip(rows, live) if l]
        live = [True] * len(rows)
        first = ix.append_bf16(extra)                                  # lands at count(): the reclaimed slots
        assert first == len(rows)
        rows += list(extra)
        live += [True] * len(extra)
        new_row = synth.bf16_round(q[0] * 2.0)
        ix.overwrite_f64(7, new_row)
        rows[7] = synth.f32_to_bf16_bits(new_row.astype(np.float32))
        ix.tombstone([0, 8, len(rows) - 1])
        for s in (0, 8, len(rows) - 1):
            live[s] = False
        corpus2 = np.stack(rows)
        lv = np.array(live, np.uint8)
        es, ev, ec = oracle_mod.search_batch_mt(corpus2, q, 30, None, live=lv)
        check_oracle(ix.search(q, 30, None)[:3], (np.where(es >= 0, es + base, -1), ev, ec))
        m2 = ix.compact()
        assert (m2 == expected_map(lv)).all() and ix.size() == lv.sum()
        es, ev, ec = oracle_mod.search_batch_mt(corpus2[lv.astype(bool)], q, 30, None)
        check_oracle(ix.search(q, 30, None)[:3], (np.where(es >= 0, es + base, -1), ev, ec))
        assert (ix.search(q[:1], 1, None)[0][0, 0] == base + m2[7])      # the overwritten row is the best hit


def test_graph_replayed_search_is_right_after_compaction(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d = 20_000, 256
    corpus = synth.random_corpus(n, d, 51)
    q = synth.random_queries(16, d, 52).astype(np.float64)
    synth.plant_neighbours(corpus, q.astype(np.float32), 20, 53)
    dead = np.flatnonzero(np.random.default_rng(54).random(n) < 0.5)
    live = np.ones(n, np.uint8)
    live[dead] = 0
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        ix.tombstone(dead)
        for _ in range(3):
            ix.search(q, 20, 0.05)
        assert ix.stats()["graph_replays"] >= 2
        ix.compact()
        replays = ix.stats()["graph_replays"]
        for _ in range(3):
            got = ix.search(q, 20, 0.05)[:3]
            check_oracle(got, oracle_mod.search_batch_mt(corpus[live.astype(bool)], q, 20, 0.05))
        assert ix.stats()["graph_replays"] >= replays + 2                # a new graph, captured for the new corpus


def test_vector_store_and_retriever_on_the_device_through_churning_syncs(rb, tmp_path, monkeypatch):
    from common import HashEmbedder, OracleIndex
    from test_compact_host import QUERIES, _answers, _docs
    from runbookai_b200 import embedder, retriever
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    monkeypatch.setattr(retriever, "_COMPACT_MIN_DEAD", 64)
    try:
        rnd = [0]
        vs = VectorStore(str(tmp_path / "vectors.db"))
        ref = VectorStore(str(tmp_path / "ref.db"), index_factory=lambda d, dev: OracleIndex(d))
        r = KnowledgeRetriever({"storePath": str(tmp_path / "k.db"), "sources": [lambda since: _docs(rnd[0])]},
                               vector_store=vs)
        rr = KnowledgeRetriever({"storePath": str(tmp_path / "rk.db"), "sources": [lambda since: _docs(rnd[0])]},
                                vector_store=ref)
        sizes = []
        for rnd[0] in range(6):
            r.sync()
            rr.sync()
            sizes.append(vs._index.size())
            assert _answers(vs) == _answers(ref) and _answers(vs, 60) == _answers(ref, 60)
            assert r.search(QUERIES[0]) == rr.search(QUERIES[0])
        assert isinstance(vs._index, rb.Index) and max(sizes) < 2 * vs._index.count()
        assert ref._index.size() > 4 * ref._index.count()
        r.close()
        rr.close()
    finally:
        embedder.reset()


def test_addon_compact_on_the_gpu(tmp_path, oracle_mod, native):
    from test_compact_host import check_compact_outputs, write_compact_input
    from test_napi_addon import _build_real, _write_inputs
    exe = _build_real()
    w = _write_inputs(tmp_path, [], n=6000, dim=200, nq=13, k=32)
    live = write_compact_input(tmp_path, w)
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    check_compact_outputs(tmp_path, w, oracle_mod, live)


def test_errors_leave_the_index_untouched(rb, native):
    from runbookai_b200 import synth
    n, d = 1000, 64
    corpus = synth.random_corpus(n, d, 61)
    q = synth.random_queries(3, d, 62).astype(np.float64)
    assert native.lib.rbk_index_compact(None, None, 0) == native.RBK_EINVAL
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        ix.tombstone(np.arange(0, n, 2))
        before = ix.search(q, 20, None)[:3]
        short = np.empty(n - 1, np.int64)
        st = native.lib.rbk_index_compact(ix._h, short.ctypes.data_as(C.c_void_p), n - 1)
        assert st == native.RBK_EINVAL and "old_to_new_len" in native.lib.rbk_last_error().decode()
        assert ix.size() == n and ix.count() == n // 2
        after = ix.search(q, 20, None)[:3]
        assert all(a.tobytes() == b.tobytes() for a, b in zip(before, after))
        assert native.lib.rbk_index_compact(ix._h, None, 0) == native.RBK_OK   # no map asked for
        assert ix.size() == n // 2
    with rb.Group(d, [0]) as g:                                         # group members are not compacted
        g.append_bf16(corpus)
        g.tombstone([1, 2])
        member = C.c_void_p(native.lib.rbk_group_member(g._h, 0))
        assert native.lib.rbk_index_compact(member, None, 0) == native.RBK_EINVAL
        assert g.size() == n and g.count() == n - 2
