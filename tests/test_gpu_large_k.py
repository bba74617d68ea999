"""GPU suite (-m gpu) for the large-k search (rbk_index_search_large_f64 / rbk_group_search_large_f64, k_fetch up to
4096): count scan, emit scan, exact fp64 re-rank.  Bar, against the oracle: ids identical, fp64 scores bit-identical,
tail -1 / NaN."""
import subprocess

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
    assert (counts == ec).all(), (counts, ec)
    for b in range(len(ec)):
        n = ec[b]
        assert (slots[b, :n] == es[b, :n]).all(), b
        assert scores[b, :n].tobytes() == ev[b, :n].tobytes(), b          # bit-exact fp64
        assert (slots[b, n:] == -1).all() and np.isnan(scores[b, n:]).all()


def oracle_bf16(oracle_mod, corpus, q, k, ms, live=None):
    return oracle_mod.search_batch_mt(corpus, np.asarray(q, np.float64), k, ms, live=live)


def oracle_f64(oracle_mod, corpus, q, k, ms, live=None):
    B = q.shape[0]
    es = np.full((B, k), -1, np.int64)
    ev = np.full((B, k), np.nan)
    ec = np.zeros(B, np.int32)
    for b in range(B):
        s, v = oracle_mod.search(corpus, q[b], k, ms, live=live)
        es[b, :len(s)], ev[b, :len(s)], ec[b] = s, v, len(s)
    return es, ev, ec


@pytest.mark.parametrize("n,d,b,k,min_score", [
    (255, 64, 3, 10, 0.5),          # < one tile
    (257, 72, 3, 10, None),         # d not a multiple of 64
    (5000, 100, 7, 32, 0.5),        # d % 8 != 0
    (30_000, 768, 130, 32, 0.5),    # 2 query blocks, ragged
    (20_000, 1536, 5, 112, None),   # the reference's default d, the search's largest k_fetch
])
def test_search_large_equals_search_for_small_k(rb, oracle_mod, n, d, b, k, min_score):
    from runbookai_b200 import synth
    corpus = synth.random_corpus(n, d, 100 + n % 97)
    q = synth.random_queries(b, d, 200 + d)
    synth.plant_neighbours(corpus, q, min(6, n // b), 300)
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        small = ix.search(q.astype(np.float64), k, min_score)
        large = ix.search_large(q, k, min_score)
        assert (small[0] == large[0]).all() and small[1].tobytes() == large[1].tobytes() and (small[2] == large[2]).all()
        check(large, *oracle_bf16(oracle_mod, corpus, q, k, min_score))


@pytest.fixture(scope="module")
def corpora(rb):
    """bf16 corpora (d 100 / 768 / 1536, N 300 .. 200k) with tombstones, a zero row, a zero query, and one keep_f64
    index of arbitrary doubles."""
    from runbookai_b200 import synth
    out = []
    for n, d, seed in ((300, 100, 1), (50_000, 768, 2), (200_000, 1536, 3)):
        corpus = synth.random_corpus(n, d, seed)
        q = synth.random_queries(4, d, seed + 10).astype(np.float64)
        synth.plant_neighbours(corpus, q.astype(np.float32), min(50, n // 8), seed + 20)
        corpus[7] = 0
        q[3] = 0.0
        dead = np.random.default_rng(seed).choice(n, n // 20, replace=False)
        live = np.ones(n, np.uint8)
        live[dead] = 0
        ix = rb.Index(d)
        ix.append_bf16(corpus)
        ix.tombstone(dead)
        out.append(("bf16", ix, corpus, q, live))
    rng = np.random.default_rng(5)
    n, d = 20_000, 100
    corpus = rng.standard_normal((n, d))
    corpus[11] = 0
    q = rng.standard_normal((3, d))
    dead = rng.choice(n, 500, replace=False)
    live = np.ones(n, np.uint8)
    live[dead] = 0
    ix = rb.Index(d, keep_f64=True)
    ix.append_f64(corpus)
    ix.tombstone(dead)
    out.append(("f64", ix, corpus, q, live))
    yield out
    for c in out:
        c[1].close()


@pytest.mark.parametrize("min_score", [None, 0.05, 0.5])
@pytest.mark.parametrize("k", [113, 200, 1000, 4096])
def test_large_k_matches_oracle(rb, oracle_mod, corpora, k, min_score):
    for kind, ix, corpus, q, live in corpora:
        ref = (oracle_bf16 if kind == "bf16" else oracle_f64)(oracle_mod, corpus, q, k, min_score, live=live)
        got = ix.search_large(q, k, min_score)
        check(got, *ref)
        if kind == "bf16":
            assert got[2][3] == 0                                           # the zero query matches nothing
        assert not np.isin(7 if kind == "bf16" else 11, got[0])              # nor does the zero row


@pytest.mark.parametrize("k", [200, 1000])
def test_tie_group_straddling_the_cut(rb, oracle_mod, k):
    """3000 identical rows straddle the k-th position: every one is a candidate (C_q >> k), ties in slot order."""
    from runbookai_b200 import synth
    n, d = 60_000, 256
    corpus = synth.random_corpus(n, d, 31)
    q = synth.random_queries(2, d, 32).astype(np.float64)
    dup = np.sort(np.random.default_rng(33).choice(n, 3000, replace=False))
    scale = np.linalg.norm(q[0]) / np.sqrt(d)
    dup_row = q[0] + 0.05 * scale * np.random.default_rng(36).standard_normal(d)          # cosine ~0.999
    corpus[dup] = synth.f32_to_bf16_bits(dup_row.astype(np.float32))
    best = np.random.default_rng(34).choice(np.setdiff1d(np.arange(n), dup), k // 2, replace=False)
    corpus[best] = synth.f32_to_bf16_bits((q[0] + 0.002 * scale * np.random.default_rng(35).standard_normal((k // 2, d)))
                                          .astype(np.float32))                              # closer still
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        got = ix.search_large(q, k, None)
        check(got, *oracle_bf16(oracle_mod, corpus, q, k, None))
        tail = got[0][0, k // 2:]
        assert (tail == dup[:len(tail)]).all()


def test_all_positive_adversarial_corpus(rb, oracle_mod):
    from runbookai_b200 import synth
    n, b, d = 6000, 12, 1536
    rng = np.random.Generator(np.random.Philox(900 + d))
    corpus = synth.f32_to_bf16_bits(np.abs(rng.standard_normal((n, d), dtype=np.float32)) + 0.05)
    corpus[:500] = synth.f32_to_bf16_bits(np.full((500, d), 1.0, np.float32) +
                                          rng.uniform(0, 2 ** -6, (500, d)).astype(np.float32))
    corpus[500:1000] = synth.f32_to_bf16_bits(rng.uniform(1.0, 1.99, (500, d)).astype(np.float32))
    q = synth.bf16_round(np.abs(rng.standard_normal((b, d), dtype=np.float32)) + 0.05)
    q[0] = 1.0
    q[1] = synth.bf16_round(rng.uniform(1.0, 1.99, d).astype(np.float32))
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        for ms in (None, 0.5):
            check(ix.search_large(q, 1000, ms), *oracle_bf16(oracle_mod, corpus, q, 1000, ms))


def test_edge_cases_and_errors(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d = 60_000, 384
    corpus = synth.random_corpus(n, d, 41)
    q = synth.random_queries(1100, d, 42).astype(np.float64)
    with rb.Index(d) as ix:
        s, v, c, _ = ix.search_large(q[:0], 500, None)                      # B = 0
        assert s.shape == (0, 500)
        s, v, c, _ = ix.search_large(q[:3], 500, None)                      # empty index
        assert (c == 0).all() and (s == -1).all() and np.isnan(v).all()
        ix.append_bf16(corpus)
        got = ix.search_large(q, 300, 0.05)                                 # two sub-batches (1024 + 76)
        es, ev, ec = oracle_bf16(oracle_mod, corpus, q, 300, 0.05)
        check(got, es, ev, ec)
        # append, tombstone, bulk overwrite, clear
        extra = synth.random_corpus(1000, d, 43)
        ix.append_bf16(extra)
        corpus = np.concatenate([corpus, extra])
        live = np.ones(len(corpus), np.uint8)
        dead = np.arange(0, len(corpus), 7)
        ix.tombstone(dead)
        live[dead] = 0
        over = np.arange(3, 3000, 7)
        rows = synth.bf16_round(np.random.default_rng(44).standard_normal((len(over), d)).astype(np.float32))
        ix.overwrite_f64_batch(over, rows.astype(np.float64))
        corpus[over] = synth.f32_to_bf16_bits(rows)
        check(ix.search_large(q[:5], 2000, None), *oracle_bf16(oracle_mod, corpus, q[:5], 2000, None, live=live))
        ix.clear()
        s, v, c, _ = ix.search_large(q[:2], 200, None)
        assert (c == 0).all()
        # errors: the search's wording
        for k in (0, 4097):
            with pytest.raises(rb.RbkError, match=r"k_fetch must be in \[1, 4096\]"):
                ix.search_large(q[:1], k, None)
        with pytest.raises(rb.DimensionError, match="Vectors must have the same length"):
            ix.search_large(np.zeros((1, d + 1)), 200, None)
        with pytest.raises(rb.RbkError, match="NaN"):
            ix.search_large(q[:1], 200, float("nan"))
        with pytest.raises(rb.RbkError, match=r"\[1, 112\]"):               # the search keeps its limit
            ix.search(q[:1], 113, None)


def test_search_any_k_takes_the_large_path(rb, oracle_mod, monkeypatch):
    from runbookai_b200 import synth
    n, d = 20_000, 256
    corpus = synth.random_corpus(n, d, 51)
    q = synth.random_queries(3, d, 52).astype(np.float64)
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        monkeypatch.setattr(rb.Index, "exact_scores", lambda self, q: (_ for _ in ()).throw(AssertionError("slow path")))
        before = ix.stats()["scan_launches"]
        got = ix.search_any_k(q, 500, 0.0)
        assert ix.stats()["scan_launches"] == before + 2
        check(got, *oracle_bf16(oracle_mod, corpus, q, 500, 0.0))


def test_vector_store_large_top_k_matches_the_oracle_store(rb, tmp_path):
    from common import HashEmbedder, OracleIndex
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    try:
        words = [f"w{i}" for i in range(60)]
        rng = np.random.default_rng(61)
        chunks = [{"chunk": {"id": f"c{i}", "documentId": f"d{i % 40}",
                             "content": " ".join(rng.choice(words, 6)), "sectionTitle": "s"},
                   "documentTitle": f"D{i % 40}", "type": "runbook", "services": []} for i in range(3000)]
        gpu = VectorStore(str(tmp_path / "g.db"))
        cpu = VectorStore(str(tmp_path / "c.db"), index_factory=lambda dim, dev: OracleIndex(dim))
        gpu.add_chunks(chunks)
        cpu.add_chunks(chunks)
        for top_k in (100, 1000):
            for query in ("w1 w2 w3", "w10 w40"):
                a = gpu.search(query, {"topK": top_k, "minScore": 0.05})
                b = cpu.search(query, {"topK": top_k, "minScore": 0.05})
                assert [(r.id, r.score) for r in a] == [(r.id, r.score) for r in b]
        gpu.close()
        cpu.close()
    finally:
        embedder.reset()


def test_one_gpu_group(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d = 30_000, 768
    corpus = synth.random_corpus(n, d, 71)
    q = synth.random_queries(5, d, 72).astype(np.float64)
    with rb.Group(d, [0]) as g:
        g.append_bf16(corpus)
        g.tombstone(np.arange(0, n, 11))
        live = np.ones(n, np.uint8)
        live[::11] = 0
        for k in (200, 1000):
            check(g.search_large(q, k, 0.05), *oracle_bf16(oracle_mod, corpus, q, k, 0.05, live=live))


def test_two_gpu_group(rb, oracle_mod):
    from common import group_devices
    from runbookai_b200 import synth
    n, d = 50_000, 512
    corpus = synth.random_corpus(n, d, 81)
    q = synth.random_queries(4, d, 82).astype(np.float64)
    with rb.Group(d, group_devices(2)) as g:
        g.append_bf16(corpus)
        check(g.search_large(q, 1000, None), *oracle_bf16(oracle_mod, corpus, q, 1000, None))


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_large_on_the_gpu(tmp_path, oracle_mod, native, devices):
    from test_large_k_host import check_large_outputs
    from test_napi_addon import _build_real, _write_inputs
    exe = _build_real()
    w = _write_inputs(tmp_path, devices, n=6000, dim=200, nq=13, k=32)
    ks = [300, 4096]
    (tmp_path / "large.txt").write_text(" ".join(map(str, ks)) + "\n")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    check_large_outputs(tmp_path, w, oracle_mod, ks)
