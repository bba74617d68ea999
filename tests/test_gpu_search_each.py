"""GPU suite (-m gpu) for rbk_index_search_each_f64 / rbk_group_search_each_f64: each query of a batch at its own k_fetch
and min_score.  Bar: row b is bit for bit what the existing API returns for query b alone at k_fetch[b] and min_score[b]
(search_unbounded, which equals search_large and search where they accept the k), padded with -1 / NaN to the batch's
largest k; a subset is checked against the oracle too."""
import numpy as np
import pytest

from common import HashEmbedder, group_devices

pytestmark = pytest.mark.gpu

TIERS = {
    "bf16": {},
    "f64_device": {"keep_f64": True},
    "f64_host": {"keep_f64": True, "f64_on_host": True},
    "f32": {"keep_f32": True},
    "f32_split": {"keep_f32_split": True},
    "scan_f16": {"keep_f64": True, "scan_f16": True},
}


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def f32x(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def expected(ix, q, ks, mins):
    """Every query alone through the existing API, padded to K = max(ks).  Queries that share (k, min_score) go in one
    search_unbounded call (whose rows are, by its own contract, the single-query answers)."""
    B, K = len(q), max(ks)
    es = np.full((B, K), -1, np.int64)
    ev = np.full((B, K), np.nan)
    ec = np.zeros(B, np.int32)
    keys = {}
    for b in range(B):
        keys.setdefault((int(ks[b]), None if mins[b] is None else float(mins[b])), []).append(b)
    for (k, m), idx in keys.items():
        s, v, c, _ = ix.search_unbounded(q[idx], k, m)
        es[idx, :k], ev[idx, :k], ec[idx] = s, v, c
    return es, ev, ec


def check_rows(got, want, what=""):
    slots, scores, counts, _ = got
    es, ev, ec = want
    assert slots.shape == es.shape and scores.shape == ev.shape, (what, slots.shape, es.shape)
    assert (counts == ec).all(), (what, np.flatnonzero(counts != ec)[:10])
    assert (slots == es).all(), (what, np.flatnonzero((slots != es).any(axis=1))[:10])
    assert scores.tobytes() == ev.tobytes(), (what, "fp64 score bits or the NaN tail differ")   # NaN bits included


def corpus(rb, n, d, seed, f32=False):
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((16, d))
    # planted neighbours so that thresholds of 0.5 cut inside the answers
    for i in range(16):
        rows[i * 7:i * 7 + 6] = q[i] + 0.6 * rng.standard_normal((6, d))
    return (f32x(rows), f32x(q)) if f32 else (rows, q)


K_MIXES = {
    "scan": [1, 5, 56, 112],
    "large": [1, 5, 113, 1000],
    "sorted": [5, 4096, 4097, 10**6],   # the last one above count()
}


def thresholds(ix, q):
    """None, 0.5, exactly a hit's score (the 4th hit of the query), and above every score."""
    s, v, c, _ = ix.search_unbounded(q, 4, None)
    out = []
    for b in range(len(q)):
        out.append([None, 0.5, float(v[b, 3]) if c[b] >= 4 else 0.25, 1.5][b % 4])
    return out


@pytest.mark.parametrize("tier", list(TIERS))
@pytest.mark.parametrize("mix", list(K_MIXES))
def test_rows_equal_the_single_query_search(rb, tier, mix):
    n, d = 9000, 200
    rows, q = corpus(rb, n, d, 7, f32=tier.startswith("f32"))
    with rb.Index(d, **TIERS[tier]) as ix:
        ix.append_f64(rows)
        ks = [K_MIXES[mix][b % 4] for b in range(len(q))]
        mins = thresholds(ix, q)
        st0 = ix.stats()
        got = ix.search_each(q, ks, mins)
        st1 = ix.stats()
        assert st1["searches"] - st0["searches"] == 1 and st1["queries"] - st0["queries"] == len(q)
        check_rows(got, expected(ix, q, ks, mins), f"{tier}/{mix}")
        if mix == "scan":
            assert st1["scan_launches"] - st0["scan_launches"] in (1, 2)   # one pass (+ the wide retry at most)
        else:
            assert st1["scan_launches"] - st0["scan_launches"] == 2        # count scan + one emit scan


@pytest.mark.parametrize("ks", [[1, 5, 56, 112, 24, 3] * 2, [1, 5, 56, 112, 113, 1000] * 2], ids=["scan", "large"])
def test_subset_matches_the_oracle(rb, oracle_mod, ks):
    from runbookai_b200 import synth
    n, d = 12000, 384
    corpus_bits = synth.random_corpus(n, d, 21)
    q = synth.random_queries(12, d, 22)
    synth.plant_neighbours(corpus_bits, q, 8, 23)
    mins = [None, 0.5] * 6
    with rb.Index(d) as ix:
        ix.append_bf16(corpus_bits)
        slots, scores, counts, _ = ix.search_each(q.astype(np.float64), ks, mins)
    for b in range(len(q)):
        es, ev = oracle_mod.search(corpus_bits, q[b].astype(np.float64), ks[b], mins[b])
        assert counts[b] == len(es), b
        assert (slots[b, :counts[b]] == es).all(), b
        assert scores[b, :counts[b]].tobytes() == np.asarray(ev).tobytes(), b
        assert (slots[b, counts[b]:] == -1).all() and np.isnan(scores[b, counts[b]:]).all()


def test_more_than_1024_queries(rb):
    n, d = 20000, 128
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((1100, d))
    ks = [[5, 10, 20, 40, 112][b % 5] for b in range(len(q))]
    mins = [[None, 0.05, 0.1][b % 3] for b in range(len(q))]
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        check_rows(ix.search_each(q, ks, mins), expected(ix, q, ks, mins), "scan, 1100 queries")
        ks2 = [k if b % 7 else 2000 for b, k in enumerate(ks)]
        check_rows(ix.search_each(q, ks2, mins), expected(ix, q, ks2, mins), "large-k, 1100 queries")


def test_past_the_large_k_budget(rb):
    """Candidates of 100 000 rows per large query: the queries split into several groups, each its own emit scan."""
    n, d = 120000, 64
    rng = np.random.default_rng(4)
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((200, d))
    ks = [[5, 100000, 5000, 100][b % 4] for b in range(len(q))]
    mins = [None] * len(q)
    with rb.Index(d) as ix:
        ix.append_f64(rows)
        st0 = ix.stats()
        got = ix.search_each(q, ks, mins)
        assert ix.stats()["scan_launches"] - st0["scan_launches"] > 2, "expected more than one query group"
        check_rows(got, expected(ix, q, ks, mins), "budget")


@pytest.mark.parametrize("mix", list(K_MIXES))
def test_tombstones_and_an_empty_index(rb, mix):
    n, d = 6000, 96
    rows, q = corpus(rb, n, d, 9)
    ks = [K_MIXES[mix][b % 4] for b in range(len(q))]
    mins = [[None, 0.5, 0.0, -0.2][b % 4] for b in range(len(q))]
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        ix.tombstone(np.arange(0, n, 3))
        check_rows(ix.search_each(q, ks, mins), expected(ix, q, ks, mins), "tombstones")
    with rb.Index(d) as ix:
        slots, scores, counts, _ = ix.search_each(q, ks, mins)
        assert slots.shape == (len(q), max(ks)) and (counts == 0).all() and (slots == -1).all()
        assert np.isnan(scores).all()
        check_rows((slots, scores, counts, 0.0), expected(ix, q, ks, mins), "empty")


def test_ties_send_some_queries_to_the_retry_and_the_fallback(rb):
    """150 exact duplicates at ranks 8 .. 157 of the tie queries: at k = 20 their proof fails even at k' = 128 and the
    exhaustive kernel answers them at their own k and threshold; the other queries of the batch (random, small k) keep
    their first-pass answers."""
    d = 256
    rng = np.random.default_rng(11)
    rows = [rng.standard_normal((4000, d))]
    u = rng.standard_normal(d)
    w = 0.2 * rng.standard_normal(d)
    rows.append(np.repeat(u[None, :], 150, axis=0))
    rows.append(u[None, :] + np.linspace(0.9, 0.3, 8)[:, None] * w[None, :])
    rows = np.concatenate(rows)
    tie_q = u[None, :] + w[None, :] + 0.05 * rng.standard_normal((6, d))
    rand_q = rng.standard_normal((10, d))
    q = np.concatenate([tie_q, rand_q])
    ks = [20] * 6 + [3, 5, 10, 40, 3, 5, 10, 40, 1, 2]
    mins = [None, 0.1, None, 0.1, None, 0.1] + [None] * 10
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        st0 = ix.stats()
        got = ix.search_each(q, ks, mins)
        st1 = ix.stats()
        assert st1["retry_batches"] - st0["retry_batches"] == 1
        assert st1["fallback_queries"] - st0["fallback_queries"] == 6
        check_rows(got, expected(ix, q, ks, mins), "ties")


def test_colocated_group_equals_a_single_index(rb):
    n, d = 20000, 160
    rows, q = corpus(rb, n, d, 13)
    devs = group_devices(3)
    with rb.Index(d, keep_f64=True) as ix, rb.Group(d, devs, keep_f64=True) as g:
        ix.append_f64(rows)
        g.append_f64(rows)
        ix.tombstone([3, 5000, 9000])
        g.tombstone([3, 5000, 9000])
        for mix in K_MIXES.values():
            ks = [mix[b % 4] for b in range(len(q))]
            mins = thresholds(ix, q)
            a = ix.search_each(q, ks, mins)
            b = g.search_each(q, ks, mins)
            check_rows(b, a[:3], f"group {ks[:4]}")
            check_rows(a, expected(ix, q, ks, mins), f"index {ks[:4]}")


def test_argument_checks(rb):
    d = 32
    with rb.Index(d) as ix:
        ix.append_f64(np.random.default_rng(0).standard_normal((100, d)))
        q = np.ones((2, d))
        with pytest.raises(rb.RbkError) as e:
            ix.search_each(q, [5, 0], [None, None])
        assert e.value.status == 1
        with pytest.raises(rb.RbkError) as e:
            ix.search_each(q, [5, 5], [0.5, float("nan")])
        assert e.value.status == 1
        with pytest.raises(rb.DimensionError):
            ix.search_each(np.ones((2, d + 1)), [5, 5], [None, None])
        st0 = ix.stats()
        slots, scores, counts, _ = ix.search_each(np.zeros((0, d)), [], [])
        assert slots.shape == (0, 0) and ix.stats()["searches"] == st0["searches"] + 1


def test_c_refusals_on_a_live_index(rb):
    """The library's own checks, reached through the C symbols on a real index: a k_fetch[b] < 1, a null k_fetch or
    min_score array and a NaN min_score[b] are RBK_EINVAL, the wrong query_dim RBK_EDIM, before anything is searched."""
    import ctypes as C
    from runbookai_b200 import _native as nat
    d, B = 32, 3
    with rb.Index(d) as ix, rb.Group(d, group_devices(2)) as g:
        rows = np.random.default_rng(0).standard_normal((200, d))
        ix.append_f64(rows)
        g.append_f64(rows)
        q = np.ones((B, d))
        slots, scores, counts = np.empty((B, 8), np.int64), np.empty((B, 8)), np.empty(B, np.int32)
        for fn, h in ((nat.lib.rbk_index_search_each_f64, ix._h), (nat.lib.rbk_group_search_each_f64, g._h)):
            def call(k, m, dim=d):
                ms = C.c_float(0)
                st = fn(h, nat.ptr(q), B, dim, nat.ptr(k), nat.ptr(m), nat.ptr(slots), nat.ptr(scores), nat.ptr(counts),
                        C.byref(ms))
                return st, (nat.lib.rbk_last_error() or b"").decode()
            k_ok = np.array([5, 8, 1], np.int32)
            m_ok = np.array([0.1, -np.inf, 0.0])
            st, msg = call(np.array([5, 0, 1], np.int32), m_ok)
            assert st == nat.RBK_EINVAL and msg == "k_fetch[1] must be >= 1", msg
            st, msg = call(None, m_ok)
            assert st == nat.RBK_EINVAL and "null k_fetch or min_score" in msg, msg
            st, msg = call(k_ok, None)
            assert st == nat.RBK_EINVAL and "null k_fetch or min_score" in msg, msg
            st, msg = call(k_ok, np.array([0.1, np.nan, 0.0]))
            assert st == nat.RBK_EINVAL and msg == "min_score[1] is NaN", msg
            st, msg = call(k_ok, m_ok, dim=d + 1)
            assert st == nat.RBK_EDIM and msg == "Vectors must have the same length", msg
            st, msg = call(k_ok, m_ok)
            assert st == nat.RBK_OK, msg
        assert ix.stats()["searches"] == 1 and ix.stats()["queries"] == B   # only the accepted call searched


def test_micro_batcher_serves_mixed_callers_in_one_call(rb, tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200.batcher import MicroBatcher
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(96))
    try:
        words = "api latency database pool redis memory cache gateway error logs restart pods".split()
        rng = np.random.default_rng(2)
        chunks = [{"chunk": {"id": f"c{i}", "documentId": f"d{i % 9}", "content": " ".join(rng.choice(words, 5))},
                   "documentTitle": f"doc {i % 9}", "type": "runbook", "services": ["api"]} for i in range(1500)]
        vs = VectorStore(str(tmp_path / "v.db"), shared=False)
        try:
            vs.add_chunks(chunks)
            callers = [("redis memory", {"topK": 5}), ("api latency", {"topK": 10, "minScore": 0.3}),
                       ("pool restart logs", {"topK": 20}), ("gateway error", {"topK": 50, "minScore": 0.1}),
                       ("database cache", {"topK": 1000, "minScore": 0.2}), ("pods", {"topK": 57})]
            want = [vs.search(t, o) for t, o in callers]
            mb = MicroBatcher(vs, window_ms=200.0)
            try:
                futs = [mb.submit(t, o) for t, o in callers]
                got = [f.result(timeout=60) for f in futs]
                assert mb.batches == 1 and mb.served == len(callers)
            finally:
                mb.close()
            for (t, o), a, b in zip(callers, got, want):
                assert [(r.id, r.score) for r in a] == [(r.id, r.score) for r in b], (t, o)
        finally:
            vs.close()
    finally:
        embedder.reset()


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_each_on_the_gpu_matches_the_oracle(tmp_path, oracle_mod, native, devices):
    """The N-API addon's searchEach (mock runtime, async work) against librbk_knn.so, on one device and a device list:
    row b is the oracle's answer at kFetch[b] and minScore[b]; both routes (largest k 112, then 1000)."""
    import subprocess
    from test_napi_addon import _build_real, _write_inputs
    exe = _build_real()
    for K in (112, 1000):
        d = tmp_path / f"k{K}"
        d.mkdir()
        w = _write_inputs(d, devices, n=6000, dim=200, nq=13, k=32)
        ks = [[1, 5, 56, 24, 3, K][b % 6] for b in range(w["nq"])]
        mins = [[0.05, "-inf", 0.1, -0.5][b % 4] for b in range(w["nq"])]
        (d / "each.txt").write_text("".join(f"{k} {m}\n" for k, m in zip(ks, mins)))
        r = subprocess.run([str(exe), str(d)], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        assert (d / "has_search_each.txt").read_text() == "1"
        nq = w["nq"]
        slots = np.fromfile(d / "each_slots.i64", dtype=np.int64).reshape(nq, K)
        scores = np.fromfile(d / "each_scores.f64", dtype=np.float64).reshape(nq, K)
        counts = np.fromfile(d / "each_counts.i32", dtype=np.int32)
        for b in range(nq):
            m = None if mins[b] == "-inf" else float(mins[b])
            es, ev = oracle_mod.search(w["corpus"], w["q"][b], ks[b], m, live=w["live"])
            n = len(es)
            assert counts[b] == n and (slots[b, :n] == es).all(), (K, b)
            assert scores[b, :n].tobytes() == np.asarray(ev).tobytes(), (K, b)
            assert (slots[b, n:] == -1).all() and np.isnan(scores[b, n:]).all(), (K, b)
        log = dict(line.split(" ", 1) for line in (d / "log.txt").read_text().strip().splitlines())
        assert log["err_each"].startswith("k_fetch[0] must be >= 1")
