"""GPU suite (-m gpu) for device storage that grows in place on reserved virtual address ranges, and for trim().

- Twins: an index that starts at 1024 rows and grows through every append route, and one whose capacity_hint means it
  never grows, must give the same bits for every search route and the same counters - on the device tier, the host
  tier and plain bf16 - before and after tombstones, compaction and trim, and after appends past the old capacity.
- Growth needs the new capacity's memory, not old + new; when doubling does not fit the capacity becomes exactly what is
  needed; when even that does not fit the append fails with RBK_ENOMEM and leaves the index as it was.
- trim() returns device memory and keeps every answer: asynchronous searches enqueued before it, graph replay, a
  one-GPU group after clear(), the VectorStore / retriever churn and the addon."""
import ctypes as C
import subprocess
from contextlib import contextmanager

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STATS = ("searches", "queries", "fallback_queries", "retry_batches", "scan_launches", "kernel_launches",
         "graph_replays", "last_kprime")
CHUNK_SLACK = 256 << 20   # a trim leaves less than one chunk of at most 256 MiB per device buffer mapped
N_BUFFERS = 5


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def storage_at(cap, d, tier):
    """rbk_index_storage_bytes's device bytes at capacity `cap`: rows | inv_norm | norm2 | tombstone bits | f64 rows."""
    dpad = (d + 63) // 64 * 64
    dev = cap * dpad * 2 + (cap + 255) // 256 * 256 * 4 + 256 * 4 + cap * 8 + (cap + 31) // 32 * 4
    return dev + (cap * d * 8 if tier == "device" else 0)


def fitted(n):
    return (max(n, 1024) + 255) // 256 * 256


def answers(ix, q):
    import torch
    out = {}
    for B in (1, 40, 200):                    # graph replay (B <= 128) and the ungraphed path
        for k, ms in ((20, None), (112, 0.3)):
            out[("search", B, k, ms)] = ix.search(q[:B], k, ms)[:3]
    out["replay"] = ix.search(q[:40], 20, None)[:3]
    for k in (500, 4096):
        out[("large", k)] = ix.search_large(q[:8], k, 0.05)[:3]
    out["unbounded"] = ix.search_unbounded(q[:3], 5000, None)[:3]
    B, k = 33, 20
    qd = torch.from_numpy(np.ascontiguousarray(q[:B], dtype=np.float32)).cuda()
    s = torch.empty((B, k), dtype=torch.int64, device="cuda")
    v = torch.empty((B, k), dtype=torch.float64, device="cuda")
    c = torch.empty(B, dtype=torch.int32, device="cuda")
    f = torch.empty(B, dtype=torch.int32, device="cuda")
    ix.search_device_async(qd.data_ptr(), B, k, None, s.data_ptr(), v.data_ptr(), c.data_ptr(), f.data_ptr())
    torch.cuda.synchronize()
    out["async"] = (s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy(), f.cpu().numpy())
    return out


def assert_twins(a, b, q):
    x, y = answers(a, q), answers(b, q)
    for key in x:
        assert all(same(u, w) for u, w in zip(x[key], y[key])), key
    sa, sb = a.stats(), b.stats()
    assert {k: sa[k] for k in STATS} == {k: sb[k] for k in STATS}
    assert a.size() == b.size() and a.count() == b.count()
    return x


def check_oracle(oracle_mod, got, corpus, live, q, k, ms):
    slots, scores, counts = got
    for b in range(len(q)):
        es, ev = oracle_mod.search(corpus, q[b], k, ms, live=live)
        assert counts[b] == len(es), b
        assert (slots[b, :len(es)] == es).all(), b
        assert scores[b, :len(es)].tobytes() == ev.tobytes(), b


@pytest.mark.parametrize("tier", ["device", "host", "bf16"])
def test_growing_twin_matches_a_presized_one(rb, oracle_mod, tier):
    import torch
    from runbookai_b200 import synth
    d = 200
    keep, on_host = tier != "bf16", tier == "host"
    rng = np.random.default_rng(7)
    grown = rb.Index(d, keep_f64=keep, f64_on_host=on_host)
    sized = rb.Index(d, capacity_hint=40000, keep_f64=keep, f64_on_host=on_host)
    twins = (grown, sized)
    corpus = np.zeros((0, d))
    live = np.zeros(0, np.uint8)
    caps = []
    trimmed = False

    def append(rows_f64, call):
        nonlocal corpus, live
        assert {call(ix) for ix in twins} == {len(corpus)}
        corpus = np.concatenate([corpus, rows_f64])
        live = np.concatenate([live, np.ones(len(rows_f64), np.uint8)])
        caps.append(grown.storage_bytes())
        if not trimmed:
            assert sized.storage_bytes()[0] == storage_at(40192, d, tier)   # never grows

    def check(q):
        assert_twins(grown, sized, q)
        got = grown.search(q[:24], 40, 0.2)[:3]
        sized.search(q[:24], 40, 0.2)                                   # keep the counters comparable
        # the oracle reads what the index stores: the f64 rows (KEEP_F64) or the bf16 rows themselves
        stored = corpus if keep else grown.read_rows_bf16(0, grown.size())
        check_oracle(oracle_mod, got, stored, live, q[:24], 40, 0.2)

    try:
        assert grown.storage_bytes()[0] == storage_at(1024, d, tier)
        r = rng.standard_normal((900, d))
        append(r, lambda ix: ix.append_f64(r))
        q = corpus[rng.choice(len(corpus), 200)] + 0.5 * rng.standard_normal((200, d))
        check(q)
        r32 = rng.standard_normal((1500, d)).astype(np.float32)
        append(r32.astype(np.float64), lambda ix: ix.append_f32(r32))
        check(q)
        rbf = synth.f32_to_bf16_bits(rng.standard_normal((2100, d)).astype(np.float32))
        append(synth.bf16_bits_to_f32(rbf).astype(np.float64), lambda ix: ix.append_bf16(rbf))
        check(q)
        rdv = rng.standard_normal((5000, d))
        t = torch.from_numpy(rdv).cuda()
        append(rdv, lambda ix: ix.append_f64_device(t.data_ptr(), len(rdv)))
        check(q)
        rb16 = synth.f32_to_bf16_bits(rng.standard_normal((9000, d)).astype(np.float32))
        tb = torch.from_numpy(rb16.view(np.int16)).cuda()
        append(synth.bf16_bits_to_f32(rb16).astype(np.float64), lambda ix: ix.append_bf16_device(tb.data_ptr(), len(rb16)))
        check(q)
        assert len({c[0] for c in caps}) >= 4                              # the capacity grew several times
        assert grown.storage_bytes()[0] == storage_at(20480, d, tier)      # doubling, whole 256-row tiles
        if on_host:
            assert grown.storage_bytes()[1] == 20480 * d * 8
        # tombstone most rows, compact and trim both: the fitted capacity, the same answers
        dead = np.setdiff1d(np.arange(len(corpus)), np.arange(0, len(corpus), 7))
        for ix in twins:
            ix.tombstone(dead)
        live[dead] = 0
        maps = [ix.compact() for ix in twins]
        assert same(maps[0], maps[1])
        corpus, live = corpus[live.astype(bool)], np.ones(int(live.sum()), np.uint8)
        trimmed = True
        for ix in twins:
            ix.trim()
            assert ix.storage_bytes()[0] == storage_at(fitted(len(corpus)), d, tier)
            if on_host:
                assert ix.storage_bytes()[1] == fitted(len(corpus)) * d * 8
        q = corpus[rng.choice(len(corpus), 200)] + 0.5 * rng.standard_normal((200, d))
        check(q)
        # past the trimmed capacity, into the range that was mapped before
        fit = fitted(len(corpus))
        r = rng.standard_normal((6000, d))
        append(r, lambda ix: ix.append_f64(r))
        check(q)
        for ix in twins:
            assert ix.storage_bytes()[0] == storage_at(fitted(max(len(corpus), 2 * fit)), d, tier)
    finally:
        for ix in twins:
            ix.close()


@contextmanager
def leave_free(nbytes):
    """Holds a torch tensor so that about `nbytes` of device memory stay free; yields the free bytes."""
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    hold = torch.empty(max(free - int(nbytes), 0), dtype=torch.uint8, device="cuda") if free > nbytes else None
    try:
        yield torch.cuda.mem_get_info()[0]
    finally:
        del hold
        torch.cuda.empty_cache()


def test_growth_needs_the_new_capacity_not_old_plus_new(rb):
    import torch
    if torch.cuda.mem_get_info()[0] < 20 << 30:
        pytest.skip("needs about 20 GB of free device memory")
    d = 1536
    cap = 1 << 19                                    # 8.06 GB of KEEP_F64 rows
    ix = rb.Index(d, capacity_hint=cap, keep_f64=True)
    try:
        block = torch.randn(1 << 16, d, dtype=torch.float64, device="cuda")
        for _ in range(cap // len(block)):
            ix.append_f64_device(block.data_ptr(), len(block))
        probe = block[:40].cpu().numpy()
        del block
        before = ix.search(probe, 8, None)[:3]
        inc = storage_at(2 * cap, d, "device") - storage_at(cap, d, "device")
        row = np.random.default_rng(3).standard_normal((1, d))
        # doubling fits in the new capacity's bytes, not in old + new (the whole new buffer)
        with leave_free(1.6 * inc) as free:
            assert 1.1 * inc < free < 2.5 * inc and free < storage_at(2 * cap, d, "device")
            assert ix.append_f64(row) == cap
        assert ix.storage_bytes()[0] == storage_at(2 * cap, d, "device")
        after = ix.search(probe, 8, None)[:3]
        assert all(same(a, b) for a, b in zip(before, after))
        assert ix.search(row, 1, None)[0][0, 0] == cap
    finally:
        ix.close()


def test_growth_falls_back_to_exact_need_then_fails_cleanly(rb):
    import torch
    if torch.cuda.mem_get_info()[0] < 20 << 30:
        pytest.skip("needs about 20 GB of free device memory")
    d, cap, more = 1536, 1 << 16, 20000
    ix = rb.Index(d, capacity_hint=cap, keep_f64=True)
    try:
        block = torch.randn(cap, d, dtype=torch.float64, device="cuda")
        ix.append_f64_device(block.data_ptr(), cap)
        extra = torch.randn(more, d, dtype=torch.float64, device="cuda")
        probe = block[:40].cpu().numpy()
        del block
        exact = (cap + more + 255) // 256 * 256
        need = storage_at(exact, d, "device") - storage_at(cap, d, "device")
        double = storage_at(2 * cap, d, "device") - storage_at(cap, d, "device")
        with leave_free(need + (double - need) // 2) as free:
            assert need < free < double
            assert ix.append_f64_device(extra.data_ptr(), more) == cap
        assert ix.storage_bytes()[0] == storage_at(exact, d, "device")
        before = ix.search(probe, 8, None)[:3]
        size, stored = ix.size(), ix.storage_bytes()
        need2 = storage_at((size + more + 255) // 256 * 256, d, "device") - stored[0]
        with leave_free(need2 // 2):
            with pytest.raises(rb.RbkError) as e:
                ix.append_f64_device(extra.data_ptr(), more)
            assert e.value.status == rb._native.RBK_ENOMEM
        assert ix.size() == size and ix.storage_bytes() == stored
        after = ix.search(probe, 8, None)[:3]
        assert all(same(a, b) for a, b in zip(before, after))
        assert ix.append_f64_device(extra.data_ptr(), more) == size   # with the memory back, the same append works
    finally:
        ix.close()


def test_capacity_hint_beyond_the_device_fails_with_enomem(rb):
    import torch
    total = torch.cuda.get_device_properties(0).total_memory
    with pytest.raises(rb.RbkError) as e:
        rb.Index(1536, capacity_hint=total // 3000, keep_f64=True)
    assert e.value.status == rb._native.RBK_ENOMEM


def test_trim_returns_memory_and_keeps_answers(rb):
    import torch
    if torch.cuda.mem_get_info()[0] < 12 << 30:
        pytest.skip("needs about 12 GB of free device memory")
    d, n, keep_every = 1536, 200000, 10
    ix = rb.Index(d, keep_f64=True)
    try:
        survivors = []
        g = torch.Generator(device="cuda").manual_seed(5)
        for first in range(0, n, 25000):
            block = torch.randn(25000, d, dtype=torch.float64, device="cuda", generator=g)
            ix.append_f64_device(block.data_ptr(), len(block))
            survivors.append(block[(-first) % keep_every::keep_every].cpu().numpy())
        del block
        corpus = np.concatenate(survivors)
        ix.tombstone(np.setdiff1d(np.arange(n), np.arange(0, n, keep_every)))
        ix.compact()
        rng = np.random.default_rng(9)
        q = corpus[rng.choice(len(corpus), 64)] + 0.05 * rng.standard_normal((64, d))
        # an asynchronous search enqueued before trim() runs first and reads the storage it had: all four outputs are
        # those of the same search without a trim behind it
        qd = torch.from_numpy(q.astype(np.float32)).cuda()
        s = torch.empty((64, 20), dtype=torch.int64, device="cuda")
        v = torch.empty((64, 20), dtype=torch.float64, device="cuda")
        c = torch.empty(64, dtype=torch.int32, device="cuda")
        f = torch.zeros(64, dtype=torch.int32, device="cuda")
        # random rows at d = 1536 are near-tied around the 20th hit, so these answers come from the retry and the
        # exhaustive fallback; the twin test above checks trimmed indexes against the oracle
        reference = ix.search(q, 20, None)[:3]
        reference_large = ix.search_large(q[:3], 300, None)[:3]
        ix.search_device_async(qd.data_ptr(), 64, 20, 0.5, s.data_ptr(), v.data_ptr(), c.data_ptr(), f.data_ptr())
        torch.cuda.synchronize()
        want = (s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy(), f.cpu().numpy())
        s.fill_(0), v.fill_(0), c.fill_(0), f.fill_(-1)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        dev_before = ix.storage_bytes()[0]
        free_before = torch.cuda.mem_get_info()[0]
        ix.search_device_async(qd.data_ptr(), 64, 20, 0.5, s.data_ptr(), v.data_ptr(), c.data_ptr(), f.data_ptr())
        ix.trim()
        torch.cuda.synchronize()
        assert all(same(a, b) for a, b in zip(want, (s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy(), f.cpu().numpy())))
        free_after = torch.cuda.mem_get_info()[0]
        dev_after = ix.storage_bytes()[0]
        assert dev_after == storage_at(fitted(len(corpus)), d, "device")
        assert free_after - free_before >= (dev_before - dev_after) - N_BUFFERS * CHUNK_SLACK
        # a trimmed index keeps answering: the graph-replayed path twice, the ungraphed path, large k
        replays = ix.stats()["graph_replays"]
        for _ in range(2):
            assert all(same(a, b) for a, b in zip(reference, ix.search(q, 20, None)[:3]))
        assert ix.stats()["graph_replays"] == replays + 2
        assert all(same(a, b) for a, b in zip(reference_large, ix.search_large(q[:3], 300, None)[:3]))
        # and grows again, in place: the new rows are found where they were appended
        extra = np.random.default_rng(4).standard_normal((30000, d))
        assert ix.append_f64(extra) == len(corpus)
        assert (ix.search(extra[:8], 1, None)[0][:, 0] == len(corpus) + np.arange(8)).all()
    finally:
        ix.close()


@pytest.mark.parametrize("n_dev", [1, 2])
def test_group_trim_after_clear(rb, oracle_mod, n_dev):
    import torch
    if torch.cuda.device_count() < n_dev:
        pytest.skip(f"needs {n_dev} GPUs")
    d = 128
    rng = np.random.default_rng(12)
    with rb.Group(d, list(range(n_dev)), keep_f64=True) as g:
        rows = rng.standard_normal((30000, d))
        g.append_f64(rows)
        g.clear()
        g.trim()
        for i in range(n_dev):                                       # every member is back at the smallest capacity
            dev = C.c_int64(0)
            lib = rb._native.lib
            assert lib.rbk_index_storage_bytes(lib.rbk_group_member(g._h, i), C.byref(dev), None) == 0
            assert dev.value == storage_at(1024, d, "device")
        g.trim()                                                     # twice: nothing left to give back
        rows = rng.standard_normal((9000, d))
        assert g.append_f64(rows) == 0
        q = rows[:16] + 0.3 * rng.standard_normal((16, d))
        check_oracle(oracle_mod, g.search(q, 30, 0.1)[:3], rows, None, q, 30, 0.1)
        g.trim()
        check_oracle(oracle_mod, g.search(q, 30, 0.1)[:3], rows, None, q, 30, 0.1)


def test_vector_store_and_retriever_trim_through_churning_syncs(rb, tmp_path, monkeypatch):
    from common import HashEmbedder, OracleIndex
    from test_compact_host import QUERIES, _answers, _docs
    from runbookai_b200 import embedder, retriever
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    monkeypatch.setattr(retriever, "_COMPACT_MIN_DEAD", 64)
    trims = []
    real_trim = rb.Index.trim

    def counting_trim(self):
        real_trim(self)
        trims.append(self.storage_bytes()[0])

    monkeypatch.setattr(rb.Index, "trim", counting_trim)
    try:
        rnd = [0]
        vs = VectorStore(str(tmp_path / "vectors.db"))
        ref = VectorStore(str(tmp_path / "ref.db"), index_factory=lambda d, dev: OracleIndex(d))
        r = KnowledgeRetriever({"storePath": str(tmp_path / "k.db"), "sources": [lambda since: _docs(rnd[0])]},
                               vector_store=vs)
        rr = KnowledgeRetriever({"storePath": str(tmp_path / "rk.db"), "sources": [lambda since: _docs(rnd[0])]},
                                vector_store=ref)
        for rnd[0] in range(6):
            r.sync()
            rr.sync()
            assert _answers(vs) == _answers(ref) and _answers(vs, 60) == _answers(ref, 60)
            assert r.search(QUERIES[0]) == rr.search(QUERIES[0])
        assert isinstance(vs._index, rb.Index) and len(trims) >= 2
        r.close()
        rr.close()
    finally:
        embedder.reset()


@pytest.mark.parametrize("devices", [[], [0]])
def test_addon_trim_on_the_gpu(tmp_path, oracle_mod, native, devices):
    from test_napi_addon import _build_real, _write_inputs
    from test_trim_host import check_trim_outputs
    exe = _build_real()
    w = _write_inputs(tmp_path, devices, n=6000, dim=200, nq=13, k=32)
    (tmp_path / "trim.txt").write_text("1\n")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    check_trim_outputs(tmp_path, w, oracle_mod)
