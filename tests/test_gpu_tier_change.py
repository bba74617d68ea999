"""GPU suite (-m gpu) for changing a float64-backed index's storage tier in place (rbk_index_set_tier /
rbk_group_set_tier).  An index is built in one tier through a mutation sequence, converted, and compared with a twin
created in the target tier and fed the same calls: every answer, the stored scan bits and the storage bytes must be the
same bits, and a subset is checked against the float64 oracle."""
import ctypes as C
import itertools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STATS = ("searches", "queries", "fallback_queries", "retry_batches", "scan_launches", "kernel_launches",
         "graph_replays", "last_kprime")
KEEP, HOST, F16 = 1, 2, 16
TIERS = {"dev_bf16": KEEP, "host_bf16": KEEP | HOST, "dev_f16": KEEP | F16, "host_f16": KEEP | HOST | F16}
PAIRS = [(a, b) for a, b in itertools.permutations(TIERS, 2)]


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def make(rb, d, flags, cap=0):
    return rb.Index(d, capacity_hint=cap, keep_f64=True, f64_on_host=bool(flags & HOST), scan_f16=bool(flags & F16))


def answers(ix, q):
    """Every output the suite compares, keyed by call (the pattern of test_gpu_host_rows.py, plus unbounded k)."""
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
    out["unbounded"] = ix.search_unbounded(q[:4], 5000, None)[:3]
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


def stats_delta(ix, before):
    now = ix.stats()
    return {k: now[k] - before[k] if k != "last_kprime" else now[k] for k in STATS}


def stored_bits(ix):
    fn = ix.read_rows_f16 if ix.flags & F16 else ix.read_rows_bf16
    return fn(0, ix.size())


def assert_twins(ix, twin, q, stats_too=False):
    """Identical answers, stored scan bits, storage bytes, size and count; with stats_too, identical stats deltas."""
    sa, sb = ix.stats(), twin.stats()
    a, b = answers(ix, q), answers(twin, q)
    for key in a:
        assert all(same(x, y) for x, y in zip(a[key], b[key])), key
    if stats_too:
        assert stats_delta(ix, sa) == stats_delta(twin, sb)
    assert ix.flags == twin.flags
    assert ix.size() == twin.size() and ix.count() == twin.count()
    assert same(stored_bits(ix), stored_bits(twin))
    assert ix.storage_bytes() == twin.storage_bytes()
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


class Sequence:
    """One mutation sequence, replayed on any number of indexes; tracks the float64 rows the oracle sees."""

    def __init__(self, d, seed, overwrite=True, compact=True):
        from runbookai_b200 import synth
        rng = np.random.default_rng(seed)
        self.d = d
        self.r64 = rng.standard_normal((600, d))                          # arbitrary doubles, not bf16-representable
        self.r32 = rng.standard_normal((300, d)).astype(np.float32)
        self.rbf = synth.f32_to_bf16_bits(rng.standard_normal((300, d)).astype(np.float32))
        self.rbf64 = synth.bf16_bits_to_f32(self.rbf).astype(np.float64)
        self.rdv = rng.standard_normal((900, d))
        self.over = rng.standard_normal((3, d)) if overwrite else None
        n = 2100
        self.dead = np.unique(np.concatenate([rng.choice(n, 400, replace=False), [70]]))
        self.compact = compact
        self.tail = rng.standard_normal((3000, d))                        # grows the capacity past 4096
        self.q = None
        self.rng = rng

    def run(self, ix):
        import torch
        ix.append_f64(self.r64)
        ix.append_f32(self.r32)
        ix.append_bf16(self.rbf)
        t = torch.from_numpy(self.rdv).cuda()
        ix.append_f64_device(t.data_ptr(), len(self.rdv))
        if self.over is not None:
            ix.overwrite_f64_batch([10, 50, 10], self.over)
        ix.tombstone(self.dead)
        if self.compact:
            ix.compact()
        ix.append_f64(self.tail)

    def oracle_rows(self):
        corpus = np.concatenate([self.r64, self.r32.astype(np.float64), self.rbf64, self.rdv])
        if self.over is not None:
            corpus[10], corpus[50] = self.over[2], self.over[1]
        live = np.ones(len(corpus), np.uint8)
        live[self.dead] = 0
        if self.compact:
            corpus, live = corpus[live.astype(bool)], live[live.astype(bool)]
        corpus = np.concatenate([corpus, self.tail])
        live = np.concatenate([live, np.ones(len(self.tail), np.uint8)])
        if self.q is None:
            self.q = queries_near(self.rng, corpus, 200)
        return corpus, live


@pytest.mark.parametrize("d", [1, 100, 768, 1536])
@pytest.mark.parametrize("src, dst", PAIRS, ids=[f"{a}-{b}" for a, b in PAIRS])
def test_every_transition_matches_a_twin(rb, oracle_mod, src, dst, d):
    seq = Sequence(d, 7 + d)
    corpus, live = seq.oracle_rows()
    with make(rb, d, TIERS[src]) as ix, make(rb, d, TIERS[dst]) as twin:
        seq.run(ix)
        seq.run(twin)
        before = ix.stats()
        ix.set_tier(f64_on_host=bool(TIERS[dst] & HOST), scan_f16=bool(TIERS[dst] & F16))
        assert ix.flags == TIERS[dst]
        after = ix.stats()                                                # the change counts no search or launch
        assert {k: after[k] for k in STATS} == {k: before[k] for k in STATS}
        assert_twins(ix, twin, seq.q)
        for k, ms in ((20, None), (112, 0.5)):
            check_oracle(oracle_mod, ix.search(seq.q[:12], k, ms)[:3], corpus, live, seq.q[:12], k, ms)
        check_oracle(oracle_mod, ix.search_large(seq.q[:3], 700, None)[:3], corpus, live, seq.q[:3], 700, None)


@pytest.mark.parametrize("src, dst", PAIRS, ids=[f"{a}-{b}" for a, b in PAIRS])
def test_stats_follow_the_twin_without_overwrites(rb, src, dst):
    seq = Sequence(100, 3, overwrite=False, compact=False)
    seq.oracle_rows()
    with make(rb, 100, TIERS[src]) as ix, make(rb, 100, TIERS[dst]) as twin:
        seq.run(ix)
        seq.run(twin)
        ix.set_tier(f64_on_host=bool(TIERS[dst] & HOST), scan_f16=bool(TIERS[dst] & F16))
        assert_twins(ix, twin, seq.q, stats_too=True)


def test_round_trip(rb, oracle_mod):
    d = 768
    seq = Sequence(d, 11)
    corpus, live = seq.oracle_rows()
    with make(rb, d, TIERS["dev_bf16"]) as ix:
        seq.run(ix)
        start = answers(ix, seq.q)
        bytes0 = ix.storage_bytes()
        ix.set_tier(f64_on_host=True, scan_f16=True)
        assert ix.flags == TIERS["host_f16"] and ix.storage_bytes()[1] > 0
        mid = answers(ix, seq.q)
        ix.set_tier(f64_on_host=False, scan_f16=False)
        assert ix.flags == TIERS["dev_bf16"]
        end = answers(ix, seq.q)
        for key in start:
            assert all(same(x, y) for x, y in zip(start[key], mid[key])), key
            assert all(same(x, y) for x, y in zip(start[key], end[key])), key
        assert ix.storage_bytes() == bytes0
        check_oracle(oracle_mod, ix.search(seq.q[:20], 20, None)[:3], corpus, live, seq.q[:20], 20, None)


def test_stream_order(rb, oracle_mod):
    import torch
    d = 256
    rng = np.random.default_rng(21)
    corpus = rng.standard_normal((40000, d))
    live = np.ones(len(corpus), np.uint8)
    q = queries_near(rng, corpus, 300)
    with make(rb, d, TIERS["dev_bf16"]) as ix:
        ix.append_f64(corpus)
        B, k = 300, 20
        qd = torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32)).cuda()
        s = torch.empty((B, k), dtype=torch.int64, device="cuda")
        v = torch.empty((B, k), dtype=torch.float64, device="cuda")
        c = torch.empty(B, dtype=torch.int32, device="cuda")
        f = torch.empty(B, dtype=torch.int32, device="cuda")
        ix.search(q[:5], k, None)                                         # a captured graph on the old tier
        ix.search_device_async(qd.data_ptr(), B, k, None, s.data_ptr(), v.data_ptr(), c.data_ptr(), f.data_ptr())
        ix.set_tier(f64_on_host=True, scan_f16=True)                      # no synchronisation in between
        torch.cuda.synchronize()
        proven = f.cpu().numpy() == 0                                     # an unproven query is re-asked, not wrong
        assert proven.mean() > 0.9
        qf = q.astype(np.float32).astype(np.float64)
        got = (s.cpu().numpy()[proven], v.cpu().numpy()[proven], c.cpu().numpy()[proven])
        check_oracle(oracle_mod, got, corpus, live, qf[proven], k, None)
        replays = ix.stats()["graph_replays"]
        got = ix.search(q[:5], k, None)[:3]                               # B <= 128: a graph again, of the new tier
        assert ix.stats()["graph_replays"] == replays + 1
        check_oracle(oracle_mod, got, corpus, live, q[:5], k, None)


def test_off_band_row_keeps_the_exhaustive_path(rb, oracle_mod):
    d = 64
    rng = np.random.default_rng(5)
    corpus = rng.standard_normal((3000, d))
    corpus[17, 3] = 1e300                                                 # outside the scan band
    live = np.ones(len(corpus), np.uint8)
    q = queries_near(rng, corpus, 8)
    order = ["dev_bf16", "host_f16", "dev_f16", "host_bf16", "dev_bf16"]
    with make(rb, d, TIERS[order[0]]) as ix:
        ix.append_f64(corpus)
        for name in order[1:]:
            ix.set_tier(f64_on_host=bool(TIERS[name] & HOST), scan_f16=bool(TIERS[name] & F16))
            with make(rb, d, TIERS[name]) as twin:
                twin.append_f64(corpus)
                for one in (ix, twin):
                    before = one.stats()["fallback_queries"]
                    got = one.search(q, 20, None)[:3]
                    assert one.stats()["fallback_queries"] - before == len(q)
                    check_oracle(oracle_mod, got, corpus, live, q, 20, None)
                assert same(stored_bits(ix), stored_bits(twin))


def test_growth_compaction_and_trim_after_a_change(rb):
    d = 192
    seq = Sequence(d, 31)
    seq.oracle_rows()
    rng = np.random.default_rng(32)
    more = rng.standard_normal((9000, d))
    for src, dst in (("dev_bf16", "host_f16"), ("host_f16", "dev_bf16"), ("dev_f16", "host_bf16")):
        with make(rb, d, TIERS[src]) as ix, make(rb, d, TIERS[dst]) as twin:
            seq.run(ix)
            seq.run(twin)
            ix.set_tier(f64_on_host=bool(TIERS[dst] & HOST), scan_f16=bool(TIERS[dst] & F16))
            for one in (ix, twin):
                one.append_f64(more)                                      # grows past the capacity of the change
                one.tombstone(np.arange(0, one.size(), 3))
            assert same(ix.compact(), twin.compact())
            for one in (ix, twin):
                one.trim()
            assert_twins(ix, twin, seq.q)


def test_refusals_leave_the_index_untouched(rb, native):
    lib = native.lib
    d = 64
    rng = np.random.default_rng(9)
    rows = rng.standard_normal((2000, d))
    q = rows[:6]
    with rb.Index(d) as plain, make(rb, d, TIERS["dev_bf16"]) as keep:
        for ix in (plain, keep):
            ix.append_f64(rows)
            ix.tombstone([3, 4])
        want = {id(ix): (ix.search(q, 20, None)[:3], ix.storage_bytes(), ix.flags, stored_bits(ix)) for ix in (plain, keep)}
        refused = [(plain, KEEP), (plain, KEEP | HOST), (plain, HOST), (plain, F16), (plain, 4),
                   (keep, 0), (keep, HOST), (keep, F16), (keep, HOST | F16), (keep, KEEP | 8)]
        for ix, flags in refused:
            assert lib.rbk_index_set_tier(ix._h, flags) == native.RBK_EINVAL, (ix.flags, flags)
            assert lib.rbk_last_error()
        assert lib.rbk_index_set_tier(None, KEEP) == native.RBK_EINVAL
        for ix in (plain, keep):                                           # the current flags: a no-op
            before = ix.stats()
            assert lib.rbk_index_set_tier(ix._h, ix.flags) == native.RBK_OK
            assert {k: ix.stats()[k] for k in STATS} == {k: before[k] for k in STATS}
        with pytest.raises(native.RbkError, match="requires RBK_INDEX_KEEP_F64") as e:
            plain.set_tier(f64_on_host=True)
        assert e.value.status == native.RBK_EINVAL
        assert lib.rbk_index_set_tier(plain._h, KEEP) == native.RBK_EINVAL
        assert "cannot add RBK_INDEX_KEEP_F64" in lib.rbk_last_error().decode()
        for ix in (plain, keep):
            s, b, f, bits = want[id(ix)]
            assert all(same(x, y) for x, y in zip(s, ix.search(q, 20, None)[:3]))
            assert ix.storage_bytes() == b and ix.flags == f and same(bits, stored_bits(ix))
    with rb.Group(d, [0], keep_f64=True) as g:
        g.append_f64(rows)
        member = C.c_void_p(lib.rbk_group_member(g._h, 0))
        assert lib.rbk_index_set_tier(member, KEEP | HOST) == native.RBK_EINVAL
        assert "rbk_group_set_tier" in lib.rbk_last_error().decode()
        assert lib.rbk_index_flags(member) == KEEP and g.flags == KEEP
        assert lib.rbk_group_set_tier(g._h, HOST) == native.RBK_EINVAL and g.flags == KEEP


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
    for src, dst in (("dev_bf16", "host_f16"), ("host_f16", "dev_f16"), ("dev_f16", "host_bf16")):
        with rb.Group(d, devs, keep_f64=True, f64_on_host=bool(TIERS[src] & HOST),
                      scan_f16=bool(TIERS[src] & F16)) as g, \
                rb.Group(d, devs, keep_f64=True, f64_on_host=bool(TIERS[dst] & HOST),
                         scan_f16=bool(TIERS[dst] & F16)) as twin:
            for one in (g, twin):
                one.append_f64(corpus)
                one.tombstone(np.flatnonzero(live == 0))
            g.set_tier(f64_on_host=bool(TIERS[dst] & HOST), scan_f16=bool(TIERS[dst] & F16))
            assert g.flags == TIERS[dst]
            for i in range(len(devs)):
                a = C.c_void_p(rb._native.lib.rbk_group_member(g._h, i))
                b = C.c_void_p(rb._native.lib.rbk_group_member(twin._h, i))
                assert rb._native.lib.rbk_index_flags(a) == TIERS[dst]
                for fn in (rb._native.lib.rbk_index_storage_bytes,):
                    x, y = (C.c_int64(0), C.c_int64(0)), (C.c_int64(0), C.c_int64(0))
                    fn(a, C.byref(x[0]), C.byref(x[1]))
                    fn(b, C.byref(y[0]), C.byref(y[1]))
                    assert (x[0].value, x[1].value) == (y[0].value, y[1].value)
            for k, ms in ((20, None), (112, 0.5)):
                got = g.search(q, k, ms)[:3]
                assert all(same(x, y) for x, y in zip(got, twin.search(q, k, ms)[:3]))
                check_oracle(oracle_mod, got, corpus, live, q, k, ms)
            got = g.search_large(q[:8], 1500, None)[:3]
            assert all(same(x, y) for x, y in zip(got, twin.search_large(q[:8], 1500, None)[:3]))
            check_oracle(oracle_mod, got, corpus, live, q[:8], 1500, None)


def test_vector_store_on_a_shared_index(rb, tmp_path, monkeypatch):
    from common import HashEmbedder
    from test_compact_host import QUERIES, _answers, _docs
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    monkeypatch.setenv("RUNBOOK_KNN_SIDECAR", "0")
    monkeypatch.delenv("RUNBOOK_KNN_F64_ON_HOST", raising=False)
    monkeypatch.delenv("RUNBOOK_KNN_SCAN_F16", raising=False)
    try:
        path = str(tmp_path / "vectors.db")
        a = VectorStore(path, shared=True)
        from runbookai_b200.retriever import KnowledgeRetriever
        r = KnowledgeRetriever({"storePath": str(tmp_path / "k.db"), "sources": [lambda since: _docs(0)]},
                               vector_store=a)
        r.sync()
        b = VectorStore(path, shared=True, f64_on_host=True, scan_f16=True)
        assert b._index is a._index
        assert (a.f64_on_host, a.scan_f16, b.f64_on_host, b.scan_f16) == (False, False, False, False)
        want = (_answers(a), _answers(a, 60))
        b.set_tier(f64_on_host=True, scan_f16=True)
        assert (a.f64_on_host, a.scan_f16, b.f64_on_host, b.scan_f16) == (True, True, True, True)
        assert a._index.storage_bytes()[1] > 0
        assert (_answers(a), _answers(a, 60)) == want and (_answers(b), _answers(b, 60)) == want
        a.set_tier(scan_f16=False)
        assert (b.f64_on_host, b.scan_f16) == (True, False)
        assert (_answers(b), _answers(b, 60)) == want
        assert r.search(QUERIES[0]) is not None
        b.close()
        r.close()
    finally:
        embedder.reset()



@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_set_tier_between_searches(tmp_path, oracle_mod, native, devices):
    import subprocess
    from test_napi_addon import _build_real, _check_outputs, _write_inputs
    exe = _build_real()
    w = _write_inputs(tmp_path, devices, n=6000, dim=200, nq=13, k=32)
    (tmp_path / "set_tier.txt").write_text("1 1\n")                       # host rows and the fp16 scan
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    log = dict(line.split(" ", 1) for line in (tmp_path / "log.txt").read_text().strip().splitlines())
    assert (log["tier_before"], log["tier_after"], log["tier_partial"]) == ("0 0", "1 1", "1 0")
    assert log["tier_identical"] == "1" and log["tier_partial_identical"] == "1"
    assert "must be a boolean" in log["err_set_tier_type"]
    nq, k = w["nq"], w["k"]
    slots = np.fromfile(tmp_path / "tier_slots.i64", dtype=np.int64).reshape(nq, k)
    scores = np.fromfile(tmp_path / "tier_scores.f64", dtype=np.float64).reshape(nq, k)
    counts = np.fromfile(tmp_path / "tier_counts.i32", dtype=np.int32)
    check_oracle(oracle_mod, (slots, scores, counts), w["corpus"], w["live"], w["q"], k, w["min_score"])
    _check_outputs(tmp_path, w, oracle_mod)


@pytest.mark.parametrize("src, dst", [("dev_bf16", "dev_f16"), ("host_f16", "host_bf16")])
def test_scan_change_alone_replays_a_new_graph(rb, oracle_mod, src, dst):
    """A change of scan type keeps every pointer the captured graph baked in: the graph must still be rebuilt, or its
    replay would run the old scan instantiation over the new rows."""
    d = 192
    rng = np.random.default_rng(41)
    corpus = rng.standard_normal((20000, d))
    live = np.ones(len(corpus), np.uint8)
    q = queries_near(rng, corpus, 24)
    with make(rb, d, TIERS[src]) as ix, make(rb, d, TIERS[dst]) as twin:
        for one in (ix, twin):
            one.append_f64(corpus)
        got0 = ix.search(q, 20, None)[:3]                                 # B <= 128: captures the graph
        ix.search(q, 20, None)                                            # ... and replays it
        replays = ix.stats()["graph_replays"]
        ix.set_tier(scan_f16=bool(TIERS[dst] & F16))
        got = ix.search(q, 20, None)[:3]
        assert ix.stats()["graph_replays"] == replays + 1
        assert all(same(x, y) for x, y in zip(got, got0))
        assert all(same(x, y) for x, y in zip(got, twin.search(q, 20, None)[:3]))
        check_oracle(oracle_mod, got, corpus, live, q, 20, None)
        dbg = ix.debug_scores(q[:4].astype(np.float32))                   # the scan itself reads the new rows
        assert np.array_equal(dbg, twin.debug_scores(q[:4].astype(np.float32)), equal_nan=True)
