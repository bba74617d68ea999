"""GPU suite (-m gpu) for rbk_index_search_slots_f64 / rbk_group_search_slots_f64: stored rows as queries.  Bar: row b
is bit for bit what search_each returns for the host copy of the stored values of slot b at k_fetch[b] and
min_score[b], on every storage tier, and a subset is the oracle's answer."""
import numpy as np
import pytest

from common import HashEmbedder, group_devices

pytestmark = pytest.mark.gpu

KEEP64, KEEP32, SPLIT, HOST, F16 = 1, 2, 4, 8, 16
TIERS = {"bf16": 0, "f64": KEEP64, "f64host": KEEP64 | HOST, "scan_f16": KEEP64 | F16, "f16host": KEEP64 | F16 | HOST,
         "f32": KEEP32, "f32host": KEEP32 | HOST, "f32f16": KEEP32 | F16, "split": SPLIT, "splithost": SPLIT | HOST}
WIDTHS = [1, 7, 100, 768, 1536, 2049]
SCAN_K = [1, 112, 5, 40]
ALL_K = [1, 112, 113, 4096, 4097, 10**6]   # the last one above count()


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def make(rb, d, tier, cls=None, devices=None):
    f = TIERS[tier]
    kw = dict(keep_f64=bool(f & KEEP64), keep_f32=bool(f & KEEP32), keep_f32_split=bool(f & SPLIT),
              f64_on_host=bool(f & HOST), scan_f16=bool(f & F16))
    return rb.Group(d, devices, **kw) if cls == "group" else rb.Index(d, **kw)


def rows_for(tier, n, d, seed):
    """Arbitrary float64 rows (float32 ones for the float32 tiers, with planted 0x8000 low halves), planted
    neighbours, and as the last four rows a zero row, a row with a NaN and two rows off the scan band (2^-50, 2^60)."""
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((n, d))
    for i in range(0, min(n - 4, 60), 6):
        rows[i + 1:i + 5] = rows[i] + 0.5 * rng.standard_normal((4, d))
    rows[n - 4] = 0.0
    rows[n - 3, d // 2] = np.nan
    rows[n - 2] *= 2.0 ** -50
    rows[n - 1] *= 2.0 ** 60
    if TIERS[tier] & (KEEP32 | SPLIT):
        u = rows.astype(np.float32).view(np.uint32)
        u[::3, ::2] = (u[::3, ::2] & np.uint32(0xFFFF0000)) | np.uint32(0x8000)
        rows = u.view(np.float32).astype(np.float64)
    return rows


def stored(ix, tier, rows, slots, base=0):
    """The host copy of the values the index stores for `slots`."""
    if tier == "bf16":
        bits = np.stack([ix.read_rows_bf16(int(s) - base, 1)[0] for s in slots])
        return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return rows[np.asarray(slots) - base]


def check_rows(got, want, what=""):
    slots, scores, counts, _ = got
    es, ev, ec, _ = want
    assert slots.shape == es.shape, (what, slots.shape, es.shape)
    assert (counts == ec).all(), (what, np.flatnonzero(counts != ec)[:10])
    assert (slots == es).all(), (what, np.flatnonzero((slots != es).any(axis=1))[:10])
    assert scores.tobytes() == ev.tobytes(), (what, "fp64 score bits or the NaN tail differ")


def thresholds(ix, q):
    """-inf, 0.5, exactly a hit's score (the 4th hit of the query) and above every score, in turn."""
    s, v, c, _ = ix.search_each(q, [4] * len(q), [None] * len(q))
    return [[None, 0.5, float(v[b, 3]) if c[b] >= 4 else 0.25, 1.5][b % 4] for b in range(len(q))]


def check_slots(ix, tier, rows, slots, ks, base=0, what=""):
    q = stored(ix, tier, rows, slots, base)
    mins = thresholds(ix, q)
    st0 = ix.stats()
    got = ix.search_slots(slots, ks, mins)
    st1 = ix.stats()
    assert st1["searches"] - st0["searches"] == 1 and st1["queries"] - st0["queries"] == len(slots), what
    check_rows(got, ix.search_each(q, ks, mins), what)
    return got


@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("tier", list(TIERS))
def test_rows_equal_search_each_on_the_stored_values(rb, tier, d):
    n = 1500
    rows = rows_for(tier, n, d, d)
    slots = np.concatenate([np.arange(0, 30), np.arange(n - 4, n), [700, 701, 1200]])
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        for ks_set in (SCAN_K, ALL_K):
            ks = [ks_set[b % len(ks_set)] for b in range(len(slots))]
            check_slots(ix, tier, rows, slots, ks, what=f"{tier}/{d}/{ks_set}")


def test_subset_matches_the_oracle(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d = 8000, 384
    bits = synth.random_corpus(n, d, 31)
    with rb.Index(d) as ix:
        ix.append_bf16(bits)
        slots = np.array([0, 5, 77, 4000, 7999, 123, 9, 10])
        ks = [1, 5, 112, 30, 1000, 113, 5, 20]
        mins = [None, 0.05, None, 0.1, None, 0.0, 0.9, None]
        got_s, got_v, got_c, _ = ix.search_slots(slots, ks, mins)
    for b, s in enumerate(slots):
        q = (bits[s].astype(np.uint32) << 16).view(np.float32).astype(np.float64)
        es, ev = oracle_mod.search(bits, q, ks[b], mins[b])
        assert got_c[b] == len(es) and (got_s[b, :got_c[b]] == es).all(), b
        assert got_v[b, :got_c[b]].tobytes() == np.asarray(ev).tobytes(), b
        assert got_s[b, 0] == s or mins[b] is not None   # a row is its own best hit


def test_more_than_1024_queries_and_the_large_k_budget(rb):
    n, d = 20000, 64
    rows = np.random.default_rng(3).standard_normal((n, d))
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        slots = np.arange(100, 1300)
        ks = [[5, 10, 112, 40][b % 4] for b in range(len(slots))]
        check_slots(ix, "f64", rows, slots, ks, what="1200 queries, scan")
        ks = [k if b % 9 else 3000 for b, k in enumerate(ks)]
        check_slots(ix, "f64", rows, slots, ks, what="1200 queries, large")
    # 100 000 candidates per large query: the queries split into several groups, each its own emit scan
    n = 120000
    rows = np.random.default_rng(4).standard_normal((n, d))
    with rb.Index(d) as ix:
        ix.append_f64(rows)
        big = np.arange(0, 2 * 200, 2)
        ks = [[5, 100000, 5000, 100][b % 4] for b in range(len(big))]
        st0 = ix.stats()
        got = ix.search_slots(big, ks, None)
        assert ix.stats()["scan_launches"] - st0["scan_launches"] > 2, "expected more than one query group"
        check_rows(got, ix.search_each(stored(ix, "bf16", rows, big), ks, None), "budget")


def test_every_row_pass_keeps_device_memory_at_one_chunk(rb):
    import torch
    n, d = 30000, 256
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((n, d))
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        ix.search_slots(np.arange(1024), 10, None)     # one chunk's scratch
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        slots, scores, counts, _ = ix.search_slots(np.arange(n), 10, None)
        free1 = torch.cuda.mem_get_info()[0]
        assert free0 - free1 < (8 << 20), (free0, free1)
        assert (slots[:, 0] == np.arange(n)).all() and (counts == 10).all()
        pick = np.array([0, 1023, 1024, 17000, n - 1])
        check_rows((slots[pick], scores[pick], counts[pick], 0.0), ix.search_each(rows[pick], [10] * 5, [None] * 5), "B = N")


def test_slot_base_refusals_and_tombstones(rb):
    n, d, base = 3000, 48, 1_000_000
    rows = rows_for("f64", n, d, 8)
    with rb.Index(d, keep_f64=True) as ix:
        ix.set_slot_base(base)
        ix.append_f64(rows)
        slots = base + np.array([0, 7, 2999, 1500])
        got = check_slots(ix, "f64", rows, slots, [5, 200, 1, 112], base=base, what="slot_base")
        assert got[0][0, 0] == slots[0]   # a row is its own best hit
        for bad in ([base - 1], [base + n], [-1]):
            with pytest.raises(rb.RbkError) as e:
                ix.search_slots(bad, 5, None)
            assert e.value.status == rb._native.RBK_EINVAL and "not a slot of this index" in str(e.value)
        ix.tombstone([7])
        live = slots[[0, 2, 3]]
        before = ix.search_slots(live, [20, 500, 5], None)
        for ks in (20, 500):
            with pytest.raises(rb.RbkError) as e:
                ix.search_slots([base, base + 7, base + 9], ks, None)
            assert e.value.status == rb._native.RBK_EINVAL and "tombstoned" in str(e.value)
        after = ix.search_slots(live, [20, 500, 5], None)
        check_rows(after, before[:3] + (0.0,), "after the refusal")
        check_rows(after, ix.search_each(rows[live - base], [20, 500, 5], None), "after the refusal, search_each")
        assert not (after[0] == base + 7).any()


def test_mutations_then_fresh_queries(rb):
    n, d = 5000, 96
    rows = rows_for("f64", n, d, 12)
    rng = np.random.default_rng(13)
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        slots = np.array([1, 2, 100, 4000])
        # overwrite: the new values are the query
        new = rng.standard_normal((2, d))
        ix.overwrite_f64_batch([1, 100], new)
        rows[[1, 100]] = new
        check_slots(ix, "f64", rows, slots, [5, 300, 112, 1], what="overwrite")
        # compaction: queries by the new slots give the renumbered answers
        ix.tombstone(np.arange(0, n, 5))
        old_to_new = ix.compact()
        rows = rows[old_to_new >= 0]
        new_slots = old_to_new[[1, 2, 101, 4001]]
        assert (new_slots >= 0).all() and (new_slots < [1, 2, 101, 4001]).any()
        check_slots(ix, "f64", rows, new_slots, [5, 300, 112, 1], what="compact")
        # tier round trips
        for kw in ({"f64_on_host": True}, {"scan_f16": True}, {"f64_on_host": False, "scan_f16": False}):
            ix.set_tier(**kw)
            check_slots(ix, "f64", rows, new_slots, [5, 4097, 40, 1], what=f"tier {kw}")
        # growth
        more = rng.standard_normal((20000, d))
        ix.append_f64(more)
        rows = np.concatenate([rows, more])
        check_slots(ix, "f64", rows, np.array([0, len(rows) - 1, 9000]), [5, 113, 112], what="growth")


@pytest.mark.parametrize("G", [2, 3, 8])
@pytest.mark.parametrize("tier", ["bf16", "f64", "splithost"])
def test_colocated_group_equals_a_single_index(rb, G, tier):
    n, d = 20000, 160
    rows = rows_for(tier, n, d, 17)
    with make(rb, d, tier) as ix, make(rb, d, tier, "group", group_devices(G)) as g:
        ix.append_f64(rows)
        g.append_f64(rows)
        ix.tombstone([3, 5000, 9000])
        g.tombstone([3, 5000, 9000])
        slots = np.array([0, 4096, 8192, 12288, 16384, 19999, 4100, 6000, 15000, 10])   # rows on different members
        for ks in ([5, 112, 1, 40] * 3, [5, 113, 4097, 10**6] * 3):
            ks = ks[:len(slots)]
            q = stored(ix, tier, rows, slots)
            mins = thresholds(ix, q)
            a = ix.search_slots(slots, ks, mins)
            check_rows(g.search_slots(slots, ks, mins), a, f"group {G} {ks[:4]}")
            check_rows(g.search_each(q, ks, mins), a, f"group search_each {G}")
            check_rows(a, ix.search_each(q, ks, mins), f"index {ks[:4]}")
        with pytest.raises(rb.RbkError) as e:
            g.search_slots([5000], 5, None)
        assert "tombstoned" in str(e.value)
        with pytest.raises(rb.RbkError) as e:
            g.search_slots([n], 5, None)
        assert "not a slot of this group" in str(e.value)


def test_vector_store_search_similar_equals_search(rb, tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore, buffer_to_float_array
    embedder.configure(HashEmbedder(96))
    try:
        words = "api latency database pool redis memory cache gateway error logs restart pods".split()
        rng = np.random.default_rng(2)
        chunks = [{"chunk": {"id": f"c{i}", "documentId": f"d{i % 9}", "content": " ".join(rng.choice(words, 5))},
                   "documentTitle": f"doc {i % 9}", "type": ["runbook", "postmortem"][i % 2],
                   "services": [["api"], ["db"]][i % 3 % 2]} for i in range(1500)]
        vs = VectorStore(str(tmp_path / "v.db"), shared=False)
        try:
            vs.add_chunks(chunks)
            stored_q = {r["id"]: buffer_to_float_array(r["embedding"]) for r in
                        vs.db.execute("SELECT id, embedding FROM vector_embeddings").fetchall()}

            class Fake:
                def embed_text(self, t):
                    return stored_q[t]

                def embed_texts(self, ts):
                    return [stored_q[t] for t in ts]
            embedder.configure(Fake())
            for cid in ("c0", "c17", "c1499"):
                for o in ({"topK": 5}, {"topK": 20, "minScore": 0.3, "typeFilter": ["runbook"]},
                          {"topK": 100, "serviceFilter": ["db"]}):
                    a = vs.search_similar(cid, {**o, "excludeSelf": False})
                    b = vs.search(f"vec_{cid}", o)
                    assert [(r.id, r.score) for r in a] == [(r.id, r.score) for r in b], (cid, o)
                    c = vs.search_similar(cid, o)
                    assert all(r.id != cid for r in c)
            batch = vs.search_similar_batch(["c1", "c2"], {"topK": 7})
            assert [[r.id for r in x] for x in batch] == [[r.id for r in vs.search_similar(c, {"topK": 7})]
                                                          for c in ("c1", "c2")]
        finally:
            vs.close()
    finally:
        embedder.reset()


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_slots_on_the_gpu_matches_the_oracle(tmp_path, oracle_mod, native, devices):
    """The N-API addon's searchSlots (mock runtime, async work) against librbk_knn.so, on one device and a device list:
    row b is the oracle's answer for the stored row of slots[b] at kFetch[b] and minScore[b], on both routes."""
    import subprocess
    from test_napi_addon import _build_real, _write_inputs
    from test_search_slots_host import check_slot_answers, slot_queries
    exe = _build_real()
    w = _write_inputs(tmp_path, devices, n=6000, dim=200, nq=13, k=32)
    qs, ks, mins = slot_queries(w)
    (tmp_path / "slots.txt").write_text("".join(f"{s} {k} {m}\n" for s, k, m in zip(qs, ks, mins)))
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "has_search_slots.txt").read_text() == "1"
    check_slot_answers(tmp_path, w, oracle_mod)
