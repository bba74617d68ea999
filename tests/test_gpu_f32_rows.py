"""GPU suite (-m gpu) for float32 exact rows (RBK_INDEX_KEEP_F32).  A KEEP_F32 index and a KEEP_F64 twin with the same
other flags are fed the same float32-exact rows through every mutation entry point, and every search route must give
the same bits and the same stats counters, equal to the float64 oracle.  Refused values leave the index untouched, and
tier changes between the two widths keep every answer."""
import ctypes as C

import numpy as np
import pytest

from common import HashEmbedder, group_devices

pytestmark = pytest.mark.gpu

KEEP64, HOST, KEEP32, F16 = 1, 2, 64, 16
STATS = ("searches", "queries", "fallback_queries", "retry_batches", "scan_launches", "graph_replays", "last_kprime")
OTHER = {"dev_bf16": 0, "host_bf16": HOST, "dev_f16": F16, "host_f16": HOST | F16}


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def make(rb, d, flags, cap=0):
    return rb.Index(d, capacity_hint=cap, keep_f64=bool(flags & KEEP64), keep_f32=bool(flags & KEEP32),
                    f64_on_host=bool(flags & HOST), scan_f16=bool(flags & F16))


def f32x(a):
    """float32-exact float64 values."""
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def answers(ix, q):
    """Every search route's outputs, and the stats counters each route moved."""
    import torch
    out = {}

    def rec(key, fn):
        before = ix.stats()
        res = fn()
        after = ix.stats()
        out[key] = tuple(res) + (tuple(after[k] - before[k] if k != "last_kprime" else after[k] for k in STATS),)

    for B in (1, 40, 200):                                     # graph replay (B <= 128) and the plain path
        for k in (1, 20, 112):
            for ms in (0.5, None):
                rec(("search", B, k, ms), lambda B=B, k=k, ms=ms: ix.search(q[:B], k, ms)[:3])
    rec("search_f32", lambda: ix.search(q[:40].astype(np.float32), 20, None)[:3])
    for k in (113, 700, 4096):
        rec(("large", k), lambda k=k: ix.search_large(q[:6], k, 0.05)[:3])
    rec("unbounded", lambda: ix.search_unbounded(q[:3], 5000, None)[:3])
    rec("exact", lambda: (ix.exact_scores(q[:3]),))
    rec("debug", lambda: (ix.debug_scores(np.ascontiguousarray(q[:5], dtype=np.float32)),))
    B, k = 40, 20
    qd = torch.from_numpy(np.ascontiguousarray(q[:B], dtype=np.float32)).cuda()
    s = torch.empty((B, k), dtype=torch.int64, device="cuda")
    v = torch.empty((B, k), dtype=torch.float64, device="cuda")
    c = torch.empty(B, dtype=torch.int32, device="cuda")
    f = torch.empty(B, dtype=torch.int32, device="cuda")

    def dev():
        ix.search_device(qd.data_ptr(), B, k, 0.05, s.data_ptr(), v.data_ptr(), c.data_ptr())
        return s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy()

    def dev_async():
        ix.search_device_async(qd.data_ptr(), B, k, None, s.data_ptr(), v.data_ptr(), c.data_ptr(), f.data_ptr())
        torch.cuda.synchronize()
        return s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy(), f.cpu().numpy()

    rec("device", dev)
    rec("async", dev_async)
    return out


def assert_same_answers(a, b):
    for key in a:
        assert len(a[key]) == len(b[key]), key
        for x, y in zip(a[key], b[key]):
            assert (x == y) if isinstance(x, tuple) else same(x, y), key


def check_oracle(oracle_mod, got, corpus, live, q, k, ms):
    slots, scores, counts = got
    for b in range(len(q)):
        es, ev = oracle_mod.search(corpus, q[b], k, ms, live=live)
        assert counts[b] == len(es), b
        assert (slots[b, :len(es)] == es).all(), b
        assert scores[b, :len(es)].tobytes() == ev.tobytes(), b


class Sequence:
    """Float32-exact rows through every mutation entry point; tracks the rows and liveness the oracle sees."""

    def __init__(self, d, seed, ties=True, off_band=False):
        from runbookai_b200 import synth
        rng = np.random.default_rng(seed)
        self.d = d
        self.r64 = f32x(rng.standard_normal((700, d)))
        if ties:                                               # a planted tie group: more copies than any margin holds
            self.r64[100:300] = self.r64[99]
        if off_band:
            self.r64[5, 0] = 2.0 ** 50                         # float32-exact, outside the scan band
        self.r32 = rng.standard_normal((300, d)).astype(np.float32)
        self.rbf = synth.f32_to_bf16_bits(rng.standard_normal((300, d)).astype(np.float32))
        self.rbf64 = synth.bf16_bits_to_f32(self.rbf).astype(np.float64)
        self.rdv = f32x(rng.standard_normal((900, d)))
        self.over1 = f32x(rng.standard_normal(d))
        self.over = f32x(rng.standard_normal((3, d)))
        n = 2200
        self.dead = np.unique(np.concatenate([rng.choice(np.arange(400, n), 300, replace=False), [70]]))
        self.tail = f32x(rng.standard_normal((3000, d)))       # grows the capacity past 4096
        q = np.concatenate([self.r64[99:100], rng.standard_normal((199, d))])
        self.q = q
        self.rng = rng

    def run(self, ix):
        import torch
        ix.append_f64(self.r64)
        ix.append_f32(self.r32)
        ix.append_bf16(self.rbf)
        t = torch.from_numpy(self.rdv).cuda()
        ix.append_f64_device(t.data_ptr(), len(self.rdv))
        ix.overwrite_f64(3, self.over1)
        ix.overwrite_f64_batch([10, 50, 10], self.over)
        ix.tombstone(self.dead)
        m = ix.compact()
        ix.append_f64(self.tail)
        return m

    def oracle_rows(self):
        corpus = np.concatenate([self.r64, self.r32.astype(np.float64), self.rbf64, self.rdv])
        corpus[3] = self.over1
        corpus[10], corpus[50] = self.over[2], self.over[1]
        keep = np.ones(len(corpus), bool)
        keep[self.dead] = False
        corpus = np.concatenate([corpus[keep], self.tail])
        return corpus, np.ones(len(corpus), np.uint8)


@pytest.mark.parametrize("d", [7, 768])
@pytest.mark.parametrize("tier", list(OTHER))
def test_twins_answer_alike(rb, oracle_mod, tier, d):
    seq = Sequence(d, 3 + d)
    corpus, live = seq.oracle_rows()
    with make(rb, d, KEEP32 | OTHER[tier]) as ix, make(rb, d, KEEP64 | OTHER[tier]) as twin:
        assert ix.flags == KEEP32 | OTHER[tier]
        assert same(seq.run(ix), seq.run(twin))               # compaction maps
        a, b = answers(ix, seq.q), answers(twin, seq.q)
        assert_same_answers(a, b)
        assert any(x[-1][STATS.index("fallback_queries")] > 0 for x in a.values())   # the ties reach the fallback
        assert any(x[-1][STATS.index("retry_batches")] > 0 for x in a.values())
        assert ix.size() == twin.size() and ix.count() == twin.count()
        for key in (("search", 40, 20, None), ("search", 200, 112, 0.5)):
            B, k, ms = key[1], key[2], key[3]
            check_oracle(oracle_mod, a[key][:3], corpus, live, seq.q[:B], k, ms)
        check_oracle(oracle_mod, a[("large", 700)][:3], corpus, live, seq.q[:6], 700, 0.05)
        # trim and clear, then the same again
        ix.trim(), twin.trim()
        assert ix.storage_bytes() == make_bytes(rb, d, KEEP32 | OTHER[tier], ix.size())
        assert_same_answers(answers(ix, seq.q[:40]), answers(twin, seq.q[:40]))
        ix.clear(), twin.clear()
        ix.append_f64(seq.tail), twin.append_f64(seq.tail)
        assert_same_answers(answers(ix, seq.q[:40]), answers(twin, seq.q[:40]))


def make_bytes(rb, d, flags, n):
    with make(rb, d, flags, cap=n) as fresh:
        return fresh.storage_bytes()


def test_off_band_row(rb, oracle_mod):
    d = 64
    seq = Sequence(d, 5, ties=False, off_band=True)
    corpus, live = seq.oracle_rows()
    with make(rb, d, KEEP32) as ix, make(rb, d, KEEP64) as twin:
        seq.run(ix), seq.run(twin)
        a, b = answers(ix, seq.q), answers(twin, seq.q)
        assert_same_answers(a, b)
        assert a[("search", 40, 20, None)][-1][STATS.index("fallback_queries")] == 40   # every query exhaustive
        check_oracle(oracle_mod, a[("search", 40, 20, None)][:3], corpus, live, seq.q[:40], 20, None)


def test_storage_bytes_and_ceiling(rb):
    d = 1536
    with make(rb, d, KEEP32, cap=4096) as a, make(rb, d, KEEP64, cap=4096) as b, \
            make(rb, d, KEEP32 | HOST, cap=4096) as c, make(rb, d, KEEP64 | HOST, cap=4096) as e:
        (da, _), (db, _) = a.storage_bytes(), b.storage_bytes()
        assert db - da == 4096 * d * 4
        assert c.storage_bytes() == (e.storage_bytes()[0], 4096 * d * 4)
        assert e.storage_bytes()[1] == 4096 * d * 8


@pytest.mark.parametrize("entry", ["append_f64", "append_f64_device", "overwrite_f64", "overwrite_f64_batch"])
@pytest.mark.parametrize("bad", [0.1, 1e-300, 1e39])
def test_refusal_leaves_the_index_untouched(rb, entry, bad):
    import torch
    from runbookai_b200._native import RBK_ENOTF32, NotFloat32Error
    d = 32
    rng = np.random.default_rng(9)
    rows = f32x(rng.standard_normal((500, d)))
    q = rng.standard_normal((20, d))
    with make(rb, d, KEEP32) as ix:
        ix.append_f64(rows)
        ix.tombstone([4, 9])
        before = (ix.size(), ix.count(), ix.storage_bytes(), ix.search(q, 20, None)[:3], ix.exact_scores(q[:2]),
                  ix.read_rows_bf16(0, ix.size()))
        new = f32x(rng.standard_normal((3, d)))
        new[1, 7] = bad
        with pytest.raises(NotFloat32Error) as e:
            if entry == "append_f64":
                ix.append_f64(new)
            elif entry == "append_f64_device":
                t = torch.from_numpy(new).cuda()
                ix.append_f64_device(t.data_ptr(), len(new))
            elif entry == "overwrite_f64":
                ix.overwrite_f64(11, new[1])
            else:
                ix.overwrite_f64_batch([11, 4, 12], new)       # slot 4 is tombstoned: refused before that rule
        assert e.value.status == RBK_ENOTF32
        after = (ix.size(), ix.count(), ix.storage_bytes(), ix.search(q, 20, None)[:3], ix.exact_scores(q[:2]),
                 ix.read_rows_bf16(0, ix.size()))
        assert before[:3] == after[:3]
        assert all(same(x, y) for x, y in zip(before[3], after[3]))
        assert same(before[4], after[4]) and same(before[5], after[5])


def test_accepted_special_values(rb, oracle_mod):
    d = 16
    rng = np.random.default_rng(2)
    rows = f32x(rng.standard_normal((300, d)))
    rows[1, 0], rows[2, 1], rows[3, 2], rows[4, 3] = np.nan, np.inf, -np.inf, -0.0
    rows[5, 4] = float(np.float32(1e-45))                      # a float32 subnormal
    q = rng.standard_normal((10, d))
    with make(rb, d, KEEP32) as ix, make(rb, d, KEEP64) as twin:
        ix.append_f64(rows), twin.append_f64(rows)
        ix.overwrite_f64(6, rows[5]), twin.overwrite_f64(6, rows[5])
        assert ix.size() == 300
        assert_same_answers(answers(ix, q), answers(twin, q))


def test_tier_changes_keep_every_answer(rb, oracle_mod):
    d = 768
    seq = Sequence(d, 17)
    corpus, live = seq.oracle_rows()
    path = [KEEP32, KEEP64 | HOST | F16, KEEP32 | HOST, KEEP64 | F16, KEEP32 | F16, KEEP64, KEEP32]
    with make(rb, d, path[0]) as ix:
        seq.run(ix)
        start = answers(ix, seq.q)
        for flags in path[1:]:
            ix.set_tier(exact_rows="f32" if flags & KEEP32 else "f64", f64_on_host=bool(flags & HOST),
                        scan_f16=bool(flags & F16))
            assert ix.flags == flags
            got = answers(ix, seq.q)
            for key in start:                                  # answers (the scan's own approximate debug scores
                if key != "debug":                             # follow the scan type, and the stats the graph)
                    assert all(same(x, y) for x, y in zip(start[key][:-1], got[key][:-1])), (flags, key)
            with make(rb, d, flags) as fresh:
                seq.run(fresh)
                assert ix.storage_bytes() == fresh.storage_bytes()
                bits = (lambda x: x.read_rows_f16 if flags & F16 else x.read_rows_bf16)
                assert same(bits(ix)(0, ix.size()), bits(fresh)(0, fresh.size()))
        check_oracle(oracle_mod, ix.search(seq.q[:20], 20, None)[:3], corpus, live, seq.q[:20], 20, None)


def test_narrowing_refused_by_a_tombstoned_slot(rb):
    from runbookai_b200._native import NotFloat32Error
    d = 48
    rng = np.random.default_rng(4)
    rows = f32x(rng.standard_normal((400, d)))
    rows[123, 5] = 0.1
    q = rng.standard_normal((8, d))
    with make(rb, d, KEEP64 | HOST) as ix:
        ix.append_f64(rows)
        ix.tombstone([123])
        before = (ix.flags, ix.storage_bytes(), ix.search(q, 20, None)[:3])
        with pytest.raises(NotFloat32Error):
            ix.set_tier(exact_rows="f32")
        assert (ix.flags, ix.storage_bytes()) == before[:2]
        assert all(same(x, y) for x, y in zip(before[2], ix.search(q, 20, None)[:3]))
        ix.compact()                                           # the slot is gone: now it narrows
        ix.set_tier(exact_rows="f32", f64_on_host=False)
        assert ix.flags == KEEP32


def group_answers(g, q):
    out = {}
    for B, k, ms in ((1, 20, None), (40, 112, 0.5), (200, 20, None)):
        out[("search", B, k, ms)] = g.search(q[:B], k, ms)[:3]
    out["large"] = g.search_large(q[:4], 900, 0.05)[:3]
    out["unbounded"] = g.search_unbounded(q[:2], 5000, None)[:3]
    return out


def member_state(rb, g):
    from runbookai_b200._native import lib
    h = g._h
    return [(lib.rbk_index_size(C.c_void_p(lib.rbk_group_member(h, i))),
             lib.rbk_index_count(C.c_void_p(lib.rbk_group_member(h, i)))) for i in range(lib.rbk_group_devices(h))]


@pytest.mark.parametrize("n", [2, 3, 4])
def test_groups(rb, oracle_mod, n):
    from runbookai_b200._native import NotFloat32Error
    d = 64
    rng = np.random.default_rng(30 + n)
    rows = f32x(rng.standard_normal((4096 * n + 500, d)))
    rows[1000:1200] = rows[999]
    q = np.concatenate([rows[999:1000], rng.standard_normal((199, d))])
    devs = group_devices(n)
    with rb.Group(d, devs, keep_f32=True) as g, rb.Group(d, devs, keep_f64=True) as t:
        for x in (g, t):
            x.append_f64(rows[:4096 * n - 10])
            x.append_f32(rows[4096 * n - 10:].astype(np.float32))
            x.overwrite_f64_batch([3, 4097], rows[:2])
            x.tombstone(np.arange(50, 4096 * n, 7))
        assert same(g.compact(), t.compact())
        a = group_answers(g, q)
        b = group_answers(t, q)
        for key in a:
            assert all(same(x, y) for x, y in zip(a[key], b[key])), key
        corpus = rows.copy()
        corpus[3], corpus[4097] = rows[0], rows[1]
        keep = np.ones(len(rows), bool)
        keep[np.arange(50, 4096 * n, 7)] = False
        check_oracle(oracle_mod, a[("search", 200, 20, None)], corpus[keep], np.ones(keep.sum(), np.uint8), q, 20, None)
        # a refused append whose bad row falls on the last member: no member changes
        state = (g.size(), g.count(), member_state(rb, g))
        bad = f32x(rng.standard_normal((4096 * n, d)))
        bad[-1, 0] = 0.1
        with pytest.raises(NotFloat32Error):
            g.append_f64(bad)
        with pytest.raises(NotFloat32Error):
            g.overwrite_f64_batch([0, g.size() - 1], bad[-2:])
        assert (g.size(), g.count(), member_state(rb, g)) == state
        a2 = group_answers(g, q)
        for key in a:
            assert all(same(x, y) for x, y in zip(a[key], a2[key])), key
        # rbk_group_set_tier both ways
        g.set_tier(exact_rows="f64", f64_on_host=True)
        assert g.flags == KEEP64 | HOST
        t.set_tier(exact_rows="f32")
        assert t.flags == KEEP32
        for x in (g, t):
            got = group_answers(x, q)
            for key in a:
                assert all(same(u, v) for u, v in zip(a[key], got[key])), key


class OddEmbedder(HashEmbedder):
    """float32-exact vectors, except for texts that contain 'odd'."""

    def embed_text(self, text):
        v = np.asarray(HashEmbedder.embed_text(self, text))
        v = f32x(v * 1.37)
        if "odd" in text.split():
            v[0] += 0.1
        return v.tolist()


def test_vector_store_widens_itself(rb, tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(OddEmbedder(96))
    try:
        words = "api latency database pool redis memory cache gateway error logs restart pods".split()
        rng = np.random.default_rng(1)
        chunks = [{"chunk": {"id": f"c{i}", "documentId": f"d{i % 7}", "content": " ".join(rng.choice(words, 5))},
                   "documentTitle": f"doc {i % 7}", "type": "runbook", "services": ["api"]} for i in range(300)]
        chunks[150]["chunk"]["content"] += " odd"
        stores = [VectorStore(str(tmp_path / f"{n}.db"), exact_rows=n) for n in ("f32", "f64")]
        try:
            f32s, f64s = stores
            assert f32s.exact_rows == "f32"
            for vs in stores:
                vs.add_chunks(chunks[:100])
                vs.add_chunks(chunks[100:])
                vs.add_chunks(chunks[140:160])                 # re-embedded: overwrites, one of them odd
            assert f32s.exact_rows == "f64" and f32s._index.flags & KEEP64
            for text in ("api latency", "redis memory odd", "pool restart logs"):
                for opts in ({"topK": 10}, {"topK": 50, "minScore": 0.2}):
                    ra, rb_ = f32s.search(text, opts), f64s.search(text, opts)
                    assert [(r.id, r.score) for r in ra] == [(r.id, r.score) for r in rb_]
        finally:
            for vs in stores:
                vs.close()
    finally:
        embedder.reset()
