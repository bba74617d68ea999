"""GPU suite (-m gpu) for float64 rows in pinned host memory (RBK_INDEX_F64_ON_HOST).  A host-tier index and a
device-tier KEEP_F64 index go through the same calls; every answer - slots, fp64 scores, counts, exactness flags,
compaction maps, fallback and retry counters - must be the same bits, and a subset is checked against the oracle."""
import ctypes as C
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STATS = ("searches", "queries", "fallback_queries", "retry_batches", "scan_launches", "kernel_launches",
         "graph_replays", "last_kprime")


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def answers(ix, q):
    """Every output the suite compares, keyed by call."""
    import torch
    out = {}
    for B in (1, 33, 200):                    # graph replay (B <= 128) and the ungraphed path
        for k in (1, 20, 112):
            for ms in (0.5, None):
                out[("search", B, k, ms)] = ix.search(q[:B], k, ms)[:3]
    out["search_f32"] = ix.search(q[:33].astype(np.float32), 20, None)[:3]
    for k in (113, 500, 4096):
        for ms in (0.05, None):
            out[("large", k, ms)] = ix.search_large(q[:8], k, ms)[:3]
    out["exact"] = (ix.exact_scores(q[:4]),)
    B, k = 33, 20
    qd = torch.from_numpy(np.ascontiguousarray(q[:B], dtype=np.float32)).cuda()
    s = torch.empty((B, k), dtype=torch.int64, device="cuda")
    v = torch.empty((B, k), dtype=torch.float64, device="cuda")
    c = torch.empty(B, dtype=torch.int32, device="cuda")
    f = torch.empty(B, dtype=torch.int32, device="cuda")
    ix.search_device(qd.data_ptr(), B, k, 0.05, s.data_ptr(), v.data_ptr(), c.data_ptr())
    out["device"] = (s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy())
    ix.search_device_async(qd.data_ptr(), B, k, None, s.data_ptr(), v.data_ptr(), c.data_ptr(), f.data_ptr())
    torch.cuda.synchronize()
    out["async"] = (s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy(), f.cpu().numpy())
    return out


def assert_twins(dev, host, q):
    a, b = answers(dev, q), answers(host, q)
    for key in a:
        assert all(same(x, y) for x, y in zip(a[key], b[key])), key
    sa, sb = dev.stats(), host.stats()
    assert {k: sa[k] for k in STATS} == {k: sb[k] for k in STATS}
    assert dev.size() == host.size() and dev.count() == host.count()
    return a


def check_oracle(oracle_mod, got, corpus, live, q, k, ms):
    """The float64 oracle (the reference's cosine of the float64 rows), one query at a time."""
    slots, scores, counts = got
    for b in range(len(q)):
        es, ev = oracle_mod.search(corpus, q[b], k, ms, live=live)
        assert counts[b] == len(es), b
        assert (slots[b, :len(es)] == es).all(), b
        assert scores[b, :len(es)].tobytes() == ev.tobytes(), b


def queries_near(rng, corpus, n):
    """Queries around corpus rows, so that min_score 0.5 keeps hits."""
    pick = rng.choice(len(corpus), n, replace=False)
    return corpus[pick] + 0.4 * rng.standard_normal((n, corpus.shape[1]))


def test_differential_through_every_mutation(rb, oracle_mod):
    import torch
    from runbookai_b200 import synth
    d = 160
    rng = np.random.default_rng(1)
    dev = rb.Index(d, capacity_hint=1000, keep_f64=True)
    host = rb.Index(d, capacity_hint=1000, keep_f64=True, f64_on_host=True)
    twins = (dev, host)
    corpus = np.zeros((0, d))
    live = np.zeros(0, np.uint8)
    caps = []

    def append(rows_f64, call):
        nonlocal corpus, live
        firsts = {call(ix) for ix in twins}
        assert firsts == {len(corpus)}
        corpus = np.concatenate([corpus, rows_f64])
        live = np.concatenate([live, np.ones(len(rows_f64), np.uint8)])
        caps.append(dev.storage_bytes()[0])

    def check(q):
        assert_twins(dev, host, q)
        if len(corpus):
            for k, ms in ((20, None), (112, 0.5)):
                got = [ix.search(q[:40], k, ms)[:3] for ix in twins]   # both: the counters stay comparable
                assert all(same(a, b) for a, b in zip(*got))
                check_oracle(oracle_mod, got[1], corpus, live, q[:40], k, ms)

    try:
        r64 = rng.standard_normal((1500, d))                              # arbitrary doubles, not bf16-representable
        append(r64, lambda ix: ix.append_f64(r64))
        r32 = rng.standard_normal((700, d)).astype(np.float32)
        append(r32.astype(np.float64), lambda ix: ix.append_f32(r32))
        rbf = synth.f32_to_bf16_bits(rng.standard_normal((600, d)).astype(np.float32))
        append(synth.bf16_bits_to_f32(rbf).astype(np.float64), lambda ix: ix.append_bf16(rbf))
        rdv = rng.standard_normal((2500, d))
        t = torch.from_numpy(rdv).cuda()
        append(rdv, lambda ix: ix.append_f64_device(t.data_ptr(), len(rdv)))
        assert len(set(caps)) >= 3                                        # the capacity grew several times
        q = queries_near(rng, corpus, 200)
        check(q)
        # overwrite: a slot named twice takes its last row
        rows = rng.standard_normal((3, d))
        for ix in twins:
            ix.overwrite_f64_batch([10, 50, 10], rows)
        corpus[10], corpus[50] = rows[2], rows[1]
        check(q)
        # tombstones, then an overwrite that names a tombstoned slot: same error, the live slot is written
        dead = np.unique(np.concatenate([rng.choice(len(corpus), 900, replace=False), [70]]))
        for ix in twins:
            ix.tombstone(dead)
        live[dead] = 0
        rows = rng.standard_normal((2, d))
        alive = next(s for s in range(60, len(corpus)) if live[s])
        errors = []
        for ix in twins:
            with pytest.raises(rb.RbkError) as e:
                ix.overwrite_f64_batch([alive, 70], rows)
            errors.append((e.value.status, str(e.value)))
        assert errors[0] == errors[1] and errors[0][0] == rb._native.RBK_EINVAL
        corpus[alive] = rows[0]
        check(q)
        # compaction: the same map, the same answers
        m_dev, m_host = dev.compact(), host.compact()
        assert same(m_dev, m_host)
        keep = live.astype(bool)
        corpus, live = corpus[keep], live[keep]
        check(q)
        # appends into the reclaimed slots, then clear and start again
        r64 = rng.standard_normal((800, d))
        append(r64, lambda ix: ix.append_f64(r64))
        check(q)
        for ix in twins:
            ix.clear()
        corpus, live = corpus[:0], live[:0]
        check(q)
        r64 = rng.standard_normal((1200, d))
        append(r64, lambda ix: ix.append_f64(r64))
        check(queries_near(rng, corpus, 200))
    finally:
        dev.close()
        host.close()


@pytest.mark.parametrize("ties, expect_fallback", [(150, True), (70, False)])
def test_tie_groups_take_the_same_fallback_and_retry(rb, oracle_mod, ties, expect_fallback):
    n, d = 6000, 128
    rng = np.random.default_rng(ties)
    corpus = rng.standard_normal((n, d))
    v = rng.standard_normal(d)
    corpus[rng.choice(n, ties, replace=False)] = v
    q = np.stack([v * 1.5, v + 0.01 * rng.standard_normal(d), rng.standard_normal(d)])
    live = np.ones(n, np.uint8)
    with rb.Index(d, keep_f64=True) as dev, rb.Index(d, keep_f64=True, f64_on_host=True) as host:
        for ix in (dev, host):
            ix.append_f64(corpus)
        got = [ix.search(q, 20, None)[:3] for ix in (dev, host)]
        assert all(same(a, b) for a, b in zip(*got))
        check_oracle(oracle_mod, got[1], corpus, live, q, 20, None)
        st = host.stats()
        assert st["retry_batches"] >= 1
        assert (st["fallback_queries"] >= 1) == expect_fallback
        assert {k: st[k] for k in STATS} == {k: dev.stats()[k] for k in STATS}
        got = [ix.search_large(q, 200, None)[:3] for ix in (dev, host)]
        assert all(same(a, b) for a, b in zip(*got))
        check_oracle(oracle_mod, got[1], corpus, live, q, 200, None)


def test_odd_dimension_takes_the_narrow_staging(rb, oracle_mod):
    n, d = 5000, 383
    rng = np.random.default_rng(383)
    corpus = rng.standard_normal((n, d))
    q = queries_near(rng, corpus, 200)
    with rb.Index(d, keep_f64=True) as dev, rb.Index(d, keep_f64=True, f64_on_host=True) as host:
        for ix in (dev, host):
            ix.append_f64(corpus)
            ix.tombstone(np.arange(0, n, 7))
        assert_twins(dev, host, q)
        live = np.ones(n, np.uint8)
        live[np.arange(0, n, 7)] = 0
        check_oracle(oracle_mod, host.search(q[:50], 112, None)[:3], corpus, live, q[:50], 112, None)
        check_oracle(oracle_mod, host.search_large(q[:8], 1000, None)[:3], corpus, live, q[:8], 1000, None)


def test_storage_bytes(rb):
    d = 1536
    rng = np.random.default_rng(4)
    with rb.Index(d, capacity_hint=2048, keep_f64=True) as dev, \
            rb.Index(d, capacity_hint=2048, keep_f64=True, f64_on_host=True) as host, \
            rb.Index(d, capacity_hint=2048) as plain:
        for step in range(2):
            rows = rng.standard_normal((3000, d))
            for ix in (dev, host, plain):
                ix.append_f64(rows)
            cap = 2048 * 2 ** (step + 1)                                  # the capacity doubles on each growth
            dd, dh = dev.storage_bytes()
            hd, hh = host.storage_bytes()
            assert dh == 0 and hh == cap * d * 8 and hd == dd - cap * d * 8
            pd, ph = plain.storage_bytes()
            assert ph == 0 and pd == hd
            assert dd / hd > 4.9                                          # 15,372 vs 3,084 bytes per row
        assert same(dev.search(rows[:5], 20, None)[1], host.search(rows[:5], 20, None)[1])


@pytest.mark.parametrize("n_dev", [1, 2], ids=["one_gpu", "two_gpus"])
def test_groups(rb, oracle_mod, n_dev):
    from common import group_devices
    devs = group_devices(n_dev)
    n, d = 9000, 192
    rng = np.random.default_rng(5)
    corpus = rng.standard_normal((n, d))
    q = queries_near(rng, corpus, 40)
    live = np.ones(n, np.uint8)
    live[::11] = 0
    with rb.Group(d, devs, keep_f64=True, f64_on_host=True) as g:
        g.append_f64(corpus)
        g.tombstone(np.flatnonzero(live == 0))
        for i in range(len(devs)):                                        # every member has its own pinned rows
            member = C.c_void_p(rb._native.lib.rbk_group_member(g._h, i))
            h = C.c_int64(0)
            assert rb._native.lib.rbk_index_storage_bytes(member, None, C.byref(h)) == 0 and h.value > 0
        for k, ms in ((20, None), (112, 0.5)):
            check_oracle(oracle_mod, g.search(q, k, ms)[:3], corpus, live, q, k, ms)
        check_oracle(oracle_mod, g.search_large(q[:8], 1500, None)[:3], corpus, live, q[:8], 1500, None)


def test_vector_store_and_retriever_through_churning_syncs(rb, tmp_path, monkeypatch):
    from common import HashEmbedder
    from test_compact_host import QUERIES, _answers, _docs
    from runbookai_b200 import embedder, retriever
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    monkeypatch.setattr(retriever, "_COMPACT_MIN_DEAD", 64)
    monkeypatch.setenv("RUNBOOK_KNN_SIDECAR", "0")
    try:
        rnd = [0]
        monkeypatch.setenv("RUNBOOK_KNN_F64_ON_HOST", "1")
        vs = VectorStore(str(tmp_path / "vectors.db"))
        monkeypatch.setenv("RUNBOOK_KNN_F64_ON_HOST", "0")
        ref = VectorStore(str(tmp_path / "ref.db"))
        r = KnowledgeRetriever({"storePath": str(tmp_path / "k.db"), "sources": [lambda since: _docs(rnd[0])]},
                               vector_store=vs)
        rr = KnowledgeRetriever({"storePath": str(tmp_path / "rk.db"), "sources": [lambda since: _docs(rnd[0])]},
                                vector_store=ref)
        for rnd[0] in range(6):
            r.sync()
            rr.sync()
            assert _answers(vs) == _answers(ref) and _answers(vs, 60) == _answers(ref, 60)
            assert r.search(QUERIES[0]) == rr.search(QUERIES[0])
            assert vs._index.size() == ref._index.size()
        assert vs._index.storage_bytes()[1] > 0 and ref._index.storage_bytes()[1] == 0
        assert vs._index.size() < 2 * vs._index.count()                   # compaction ran on the host tier
        r.close()
        rr.close()
    finally:
        embedder.reset()


def test_addon_with_host_rows_on_the_gpu(tmp_path, oracle_mod, native):
    from test_napi_addon import _build_real, _check_outputs, _write_inputs
    exe = _build_real()
    w = _write_inputs(tmp_path, [], n=6000, dim=200, nq=13, k=32)
    (tmp_path / "host_rows.txt").write_text("1\n")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    _check_outputs(tmp_path, w, oracle_mod)


def test_flag_errors_create_nothing(rb, native):
    lib = native.lib
    devs = np.zeros(1, np.int32)
    for flags, msg in ((native.RBK_INDEX_F64_ON_HOST, "RBK_INDEX_F64_ON_HOST requires RBK_INDEX_KEEP_F64"),
                       (4, "unknown flag"), (1 | 8, "unknown flag")):
        h = C.c_void_p(0x1234)
        assert lib.rbk_index_create_ex(64, 0, 0, flags, C.byref(h)) == native.RBK_EINVAL
        assert lib.rbk_last_error().decode() == msg and not h.value
        g = C.c_void_p(0x1234)
        assert lib.rbk_group_create(64, devs.ctypes.data_as(C.c_void_p), 1, 0, flags, C.byref(g)) == native.RBK_EINVAL
        assert lib.rbk_last_error().decode() == msg and not g.value
