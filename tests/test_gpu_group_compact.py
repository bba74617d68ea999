"""GPU suite (-m gpu) for compaction of a device group (rbk_group_compact): a one-GPU group against a single index fed
the same calls (map, stored rows, every route bit for bit), a group of two or more GPUs against a new group of the
survivors, a float64 row outside the scan's band moved to another device, the vector store and retriever over a group,
the addon on a group handle, and the error paths."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from test_gpu_compact import all_answers, assert_same_through_map, expected_map
from test_gpu_exact_paths import check

pytestmark = pytest.mark.gpu

BLOCK = 4096
TIERS = ("bf16", "device", "host", "f16")


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def make(rb, cls, d, tier, *args):
    return cls(d, *args, keep_f64=tier != "bf16", f64_on_host=tier == "host", scan_f16=tier == "f16")


def routes(h, q, unbounded_k):
    """all_answers (search f64 / f32, search_large) plus the unbounded search and the exact scores."""
    out = all_answers(h, q)
    out[(unbounded_k, None, "unbounded")] = h.search_unbounded(q, unbounded_k, None)[:3]
    out[(unbounded_k, 0.05, "unbounded")] = h.search_unbounded(q, unbounded_k, 0.05)[:3]
    return out


def bit_equal(a, b):
    return a.keys() == b.keys() and all(x.tobytes() == y.tobytes() for k in a for x, y in zip(a[k], b[k]))


def member_rows(rb, g, i, tier):
    lib = rb._native.lib
    m = C.c_void_p(lib.rbk_group_member(g._h, i))
    n = lib.rbk_index_size(m)
    out = np.empty((n, g.dim), dtype=np.uint16)
    fn = lib.rbk_index_read_rows_f16 if tier == "f16" else lib.rbk_index_read_rows_bf16
    rb._native.check(fn(m, 0, n, out.ctypes.data_as(C.c_void_p)))
    return out


def runs_dead(n, rng, frac=0.5):
    """Documents of 8-40 slots, about frac of them deleted."""
    live = np.ones(n, np.uint8)
    s = 0
    while s < n:
        run = int(rng.integers(8, 41))
        if rng.random() < frac:
            live[s:s + run] = 0
        s += run
    return live


def corpus_for(tier, n, d, seed):
    from runbookai_b200 import synth
    if tier == "bf16":
        return synth.random_corpus(n, d, seed)
    return np.random.default_rng(seed).standard_normal((n, d))


def append(h, tier, rows):
    return h.append_bf16(rows) if tier == "bf16" else h.append_f64(rows)


def oracle_check(oracle_mod, answers, rows, q):
    for (k, ms, kind), got in answers.items():
        qq = q.astype(np.float32).astype(np.float64) if kind == "f32" else q
        check(oracle_mod, got, rows, None, qq, k, ms, f"{kind} k={k} min_score={ms}")


def n_devices():
    import torch
    return torch.cuda.device_count()


# --------------------------------------------------------------------------- one GPU: the group is the index
@pytest.mark.parametrize("tier", TIERS)
def test_one_gpu_group_compacts_like_an_index(rb, oracle_mod, tier):
    """A corpus that ends mid-block, deleted in document runs and in one whole block: the group of one GPU and the
    index get the same map, store the same rows and answer every route identically, before and after."""
    from runbookai_b200 import synth
    n, d = 3 * BLOCK + 1234, 96
    corpus = corpus_for(tier, n, d, 5)
    q = synth.random_queries(6, d, 6).astype(np.float64) if tier == "bf16" else np.random.default_rng(6).standard_normal((6, d))
    live = runs_dead(n, np.random.default_rng(7))
    live[BLOCK:2 * BLOCK] = 0
    keep = live.astype(bool)
    with make(rb, rb.Group, d, tier, [0]) as g, make(rb, rb.Index, d, tier) as ix:
        for h in (g, ix):
            append(h, tier, corpus)
            h.tombstone(np.flatnonzero(~keep))
        before_g, before_i = routes(g, q, 5000), routes(ix, q, 5000)
        assert bit_equal(before_g, before_i)
        ex0 = g.exact_scores(q)
        m_g, m_i = g.compact(), ix.compact()
        assert (m_g == m_i).all() and (m_g == expected_map(live)).all()
        assert g.size() == g.count() == ix.size() == keep.sum()
        assert (member_rows(rb, g, 0, tier) == (ix.read_rows_f16 if tier == "f16" else ix.read_rows_bf16)(0, ix.size())).all()
        after_g = routes(g, q, 5000)
        assert bit_equal(after_g, routes(ix, q, 5000))
        assert_same_through_map(before_g, after_g, m_g)
        assert g.exact_scores(q).tobytes() == ex0[:, keep].tobytes()
        oracle_check(oracle_mod, after_g, corpus[keep], q)   # bf16 bits or float64 rows
        again = g.compact()                                          # nothing left: the identity, nothing moves
        assert (again == np.arange(g.size())).all() and bit_equal(routes(g, q, 5000), after_g)


def test_one_gpu_group_large_corpus_takes_many_staging_chunks(rb, oracle_mod):
    """200k x 1536 KEEP_F64: one 4096-row block per 64 MB staging chunk, 49 blocks, half the rows deleted in runs."""
    from runbookai_b200 import synth
    n, d = 200_000, 1536
    corpus = synth.random_corpus(n, d, 32)
    q = synth.random_queries(32, d, 33).astype(np.float64)
    synth.plant_neighbours(corpus, q.astype(np.float32), 40, 34)
    live = runs_dead(n, np.random.default_rng(31))
    keep = live.astype(bool)
    with rb.Group(d, [0], keep_f64=True) as g, rb.Index(d, keep_f64=True) as ix:
        for h in (g, ix):
            h.append_bf16(corpus)
            h.tombstone(np.flatnonzero(~keep))
        before = {(20, "f64"): g.search(q, 20, 0.05)[:3], (1000, "large"): g.search_large(q[:8], 1000, 0.05)[:3]}
        m_g, m_i = g.compact(), ix.compact()
        assert (m_g == m_i).all() and (m_g == expected_map(live)).all()
        after = {(20, "f64"): g.search(q, 20, 0.05)[:3], (1000, "large"): g.search_large(q[:8], 1000, 0.05)[:3]}
        assert bit_equal(after, {(20, "f64"): ix.search(q, 20, 0.05)[:3],
                                 (1000, "large"): ix.search_large(q[:8], 1000, 0.05)[:3]})
        assert_same_through_map(before, after, m_g)
        rows = member_rows(rb, g, 0, "bf16")
        assert (rows == ix.read_rows_bf16(0, ix.size())).all() and (rows == corpus[keep]).all()
        es, ev, ec = oracle_mod.search_batch_mt(corpus[keep], q, 20, 0.05)
        s, v, c = after[(20, "f64")]
        assert (c == ec).all()
        for b in range(len(q)):
            assert (s[b, :c[b]] == es[b, :c[b]]).all() and v[b, :c[b]].tobytes() == ev[b, :c[b]].tobytes()


# --------------------------------------------------------------------------- two or more members
def group_devices(n_dev):
    """n_dev members (0: every visible GPU, at least three members), co-located where the machine has too few GPUs."""
    import common
    return common.group_devices(max(n_devices(), 3) if n_dev == 0 else n_dev)


@pytest.mark.parametrize("n_dev", [2, 0], ids=["two", "all"])
def test_group_compacts_to_a_new_group_of_the_survivors(rb, oracle_mod, n_dev):
    devs = group_devices(n_dev)
    G, d = len(devs), 128
    n = G * BLOCK * 2 + 777
    rng = np.random.default_rng(G)
    corpus = rng.standard_normal((n, d))
    q = corpus[rng.choice(n, 5)] + 0.1 * rng.standard_normal((5, d))
    live = runs_dead(n, rng, 0.4)
    live[BLOCK:2 * BLOCK] = 0                                        # device 1 loses a whole block
    keep = live.astype(bool)
    with rb.Group(d, devs, keep_f64=True) as g, rb.Group(d, devs, keep_f64=True) as f:
        g.append_f64(corpus)
        g.tombstone(np.flatnonzero(~keep))
        before = routes(g, q, 3000)
        m = g.compact()
        assert (m == expected_map(live)).all()
        f.append_f64(corpus[keep])
        assert g.size() == g.count() == f.size() == keep.sum()
        lib = rb._native.lib
        for i in range(G):
            assert lib.rbk_index_size(C.c_void_p(lib.rbk_group_member(g._h, i))) == \
                lib.rbk_index_size(C.c_void_p(lib.rbk_group_member(f._h, i)))
            assert (member_rows(rb, g, i, "device") == member_rows(rb, f, i, "device")).all(), i
        after = routes(g, q, 3000)
        assert bit_equal(after, routes(f, q, 3000))
        assert_same_through_map(before, after, m)
        assert g.exact_scores(q).tobytes() == f.exact_scores(q).tobytes()
        oracle_check(oracle_mod, after, corpus[keep], q)
        again = g.compact()
        assert (again == np.arange(g.size())).all() and bit_equal(routes(g, q, 3000), after)
        # appends land at count() on the right device; overwrites, tombstones and another compaction follow
        extra = rng.standard_normal((BLOCK + 300, d))
        extra[5] = q[0] * 3.0
        for h in (g, f):
            assert h.append_f64(extra) == keep.sum()
            h.overwrite_f64(17, q[1] * 0.5)
            h.tombstone(np.arange(100, 100 + BLOCK + 50))
        assert bit_equal(routes(g, q, 3000), routes(f, q, 3000))
        m2, mf = g.compact(), f.compact()
        assert (m2 == mf).all()
        for i in range(G):
            assert (member_rows(rb, g, i, "device") == member_rows(rb, f, i, "device")).all(), i
        final = routes(g, q, 3000)
        assert bit_equal(final, routes(f, q, 3000))
        rows = np.concatenate([corpus[keep], extra])
        rows[17] = q[1] * 0.5
        alive = np.ones(len(rows), bool)
        alive[100:100 + BLOCK + 50] = False
        oracle_check(oracle_mod, final, rows[alive], q)


@pytest.mark.parametrize("n_dev", [2, 0], ids=["two", "all"])
def test_off_band_row_moved_to_another_device_still_reaches_the_exhaustive_kernel(rb, oracle_mod, n_dev):
    """A float64 row whose largest element is below the scan's band (its bf16 copy is zero) sits in block 1, on device 1;
    block 0 is deleted, so compaction moves it to device 0, whose own rows were all in the band."""
    from float_range_cases import scaled
    from test_gpu_exact_paths import counters
    from test_gpu_float_range import all_routes
    devs = group_devices(n_dev)
    G, d = len(devs), 100
    rng = np.random.default_rng(77)
    n = G * BLOCK + 2000
    rows = rng.standard_normal((n, d))
    q = rows[rng.choice(n, 4)] + 0.1 * rng.standard_normal((4, d))
    rows[BLOCK + 10] = scaled(q[0] + 0.05 * rng.standard_normal(d), -160)   # the best hit of q[0], off the band
    live = np.ones(n, np.uint8)
    live[:BLOCK] = 0
    keep = live.astype(bool)
    with rb.Group(d, devs, keep_f64=True) as g:
        g.append_f64(rows)
        g.tombstone(np.flatnonzero(~keep))
        m = g.compact()
        assert m[BLOCK + 10] == 10                                   # now in block 0: device 0
        _, f0 = counters(g)
        got = g.search(q, 10, None)
        _, f1 = counters(g)
        assert f1 > f0, "the moved off-band row must send the search to the exhaustive kernel"
        assert got[0][0, 0] == 10
        all_routes(oracle_mod, g, rows[keep], None, q, f"group on {G} GPUs after compaction", group=True)


# --------------------------------------------------------------------------- the layers above
def test_vector_store_and_retriever_over_a_group_through_churning_syncs(rb, tmp_path, monkeypatch):
    from common import HashEmbedder, OracleIndex
    from test_compact_host import QUERIES, _answers, _docs
    from runbookai_b200 import embedder, retriever
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    gpus = list(range(n_devices()))
    embedder.configure(HashEmbedder(64))
    monkeypatch.setattr(retriever, "_COMPACT_MIN_DEAD", 64)
    try:
        rnd = [0]
        vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: rb.Group(d, gpus))
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
        assert isinstance(vs._index, rb.Group) and max(sizes) < 2 * vs._index.count()
        assert ref._index.size() > 4 * ref._index.count()
        r.close()
        rr.close()
    finally:
        embedder.reset()


def test_addon_compact_on_a_group_handle(tmp_path, oracle_mod, native):
    from test_compact_host import check_compact_outputs, write_compact_input
    from test_napi_addon import _build_real, _write_inputs
    exe = _build_real()
    w = _write_inputs(tmp_path, [0], n=6000, dim=200, nq=13, k=32)
    live = write_compact_input(tmp_path, w)
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "err_compact" not in (tmp_path / "log.txt").read_text()
    check_compact_outputs(tmp_path, w, oracle_mod, live)


def test_errors_leave_the_group_untouched(rb, native):
    from runbookai_b200 import synth
    n, d = 5000, 64
    corpus = synth.random_corpus(n, d, 61)
    q = synth.random_queries(3, d, 62).astype(np.float64)
    lib = native.lib
    assert lib.rbk_group_compact(None, None, 0) == native.RBK_EINVAL
    with rb.Group(d, [0]) as g:
        g.append_bf16(corpus)
        g.tombstone(np.arange(0, n, 2))
        before = g.search(q, 20, None)[:3]
        short = np.empty(n - 1, np.int64)
        st = lib.rbk_group_compact(g._h, short.ctypes.data_as(C.c_void_p), n - 1)
        assert st == native.RBK_EINVAL and "old_to_new_len" in lib.rbk_last_error().decode()
        assert g.size() == n and g.count() == n // 2
        assert all(a.tobytes() == b.tobytes() for a, b in zip(before, g.search(q, 20, None)[:3]))
        member = C.c_void_p(lib.rbk_group_member(g._h, 0))
        assert lib.rbk_index_compact(member, None, 0) == native.RBK_EINVAL   # members only through the group
        assert g.size() == n
        assert lib.rbk_group_compact(g._h, None, 0) == native.RBK_OK        # no map asked for
        assert g.size() == g.count() == n // 2
