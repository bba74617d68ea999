"""GPU suite (-m gpu) for rbk_index_similar_pairs_f64 / rbk_group_similar_pairs_f64: every pair of stored rows at or
above a threshold.  Bar: the entries of a pass with first element a are bit for bit the entries of
search_slots([a], count(), min_score) whose slot is above a, in the same order, on every storage tier; a subset is the
oracle's pairwise cosines."""
import ctypes as C

import numpy as np
import pytest

from common import HashEmbedder, group_devices
from test_gpu_search_slots import TIERS, WIDTHS, make, rows_for

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def pair_rows(tier, n, d, seed):
    """rows_for's rows (planted neighbour groups; a zero row, a NaN row and two off-band rows at the end) with exact
    duplicates of row 2 in the middle."""
    rows = rows_for(tier, n, d, seed)
    if n >= 40:
        rows[n // 2] = rows[n // 2 + 1] = rows[2]
    return rows


def want_pairs(ix, live_slots, min_score):
    """The pairs search_slots gives: for every live a, its hits at k = count() whose slot is above a."""
    A, B, S = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)], [np.zeros(0)]
    K = ix.count()
    if K == 0:
        return A[0], B[0], S[0]
    live_slots = np.asarray(live_slots, np.int64)
    for i in range(0, len(live_slots), 512):
        sl = live_slots[i:i + 512]
        s, v, c, _ = ix.search_slots(sl, K, min_score)
        for r, a in enumerate(sl):
            ss, vv = s[r, :c[r]], v[r, :c[r]]
            m = ss > a
            A.append(np.full(int(m.sum()), a, np.int64))
            B.append(ss[m])
            S.append(vv[m])
    return np.concatenate(A), np.concatenate(B), np.concatenate(S)


def all_pairs(ix, min_score, max_pairs=None, first_slot=None, end=None):
    """Every page from first_slot on, concatenated; checks that each page ends where the next one starts."""
    end = ix.size() + getattr(ix, "slot_base", 0) if end is None else end
    A, B, S = [], [], []
    nxt = first_slot
    while True:
        a, b, s, n2 = ix.similar_pairs(min_score, nxt, max_pairs)
        assert nxt is None or n2 > nxt or (nxt == end and n2 == end)
        if len(a):
            assert a.min() >= (nxt if nxt is not None else 0) and a.max() < n2
        A.append(a), B.append(b), S.append(s)
        nxt = n2
        if nxt >= end:
            return np.concatenate(A), np.concatenate(B), np.concatenate(S)


def check_pairs(got, want, what=""):
    a, b, s = got[:3]
    ea, eb, es = want[:3]
    assert len(a) == len(ea), (what, len(a), len(ea))
    assert (a == ea).all(), (what, np.flatnonzero(a != ea)[:10])
    assert (b == eb).all(), (what, np.flatnonzero(b != eb)[:10])
    assert s.tobytes() == es.tobytes(), (what, "fp64 score bits differ")


def one_call(ix, min_score, first_slot=None):
    """The pass in one call with room for every pair (in pages of 2^22 pairs on a large index)."""
    n = ix.size()
    if n > 2000:
        return all_pairs(ix, min_score, 1 << 22, first_slot)
    a, b, s, nxt = ix.similar_pairs(min_score, first_slot, max(n * (n - 1) // 2, n, 1))
    assert nxt == ix.size() + getattr(ix, "slot_base", 0)
    return a, b, s


@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("tier", list(TIERS))
def test_pairs_equal_search_slots_on_every_tier_and_width(rb, tier, d):
    n = 600
    rows = pair_rows(tier, n, d, d + 1)
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        for m in (None, 0.5, 1.0):
            got = one_call(ix, m)
            check_pairs(got, want_pairs(ix, np.arange(n), m), f"{tier}/{d}/{m}")
            if m == 0.5 and d > 1:
                assert ((got[0] == 2) & (got[1] == n // 2)).any()   # the planted exact duplicate, at 1.0
        assert len(one_call(ix, 1.5)[0]) == 0
        check_special_rows(one_call(ix, None), n)


def check_special_rows(pairs, n):
    """At -inf: the zero row (n - 4) and the NaN row (n - 3) pair with nothing; the two off-band rows (n - 2, n - 1),
    whose queries take the emit-all path, pair with every row the reference scores, each other included."""
    a, b, s = pairs
    assert not np.isin(a, [n - 4, n - 3]).any() and not np.isin(b, [n - 4, n - 3]).any()
    assert not np.isnan(s).any()
    assert ((a == n - 2) & (b == n - 1)).any()
    assert (b == n - 2).sum() == n - 4 and (b == n - 1).sum() == n - 3


@pytest.mark.parametrize("tier", list(TIERS))
def test_pairs_past_the_first_chunk_on_every_tier(rb, tier):
    """1300 rows: the second chunk's scans start at row 1024, so every tier reads its rows, exact rows, norms and
    tombstone bits from an offset."""
    n, d = 1300, 100
    rows = pair_rows(tier, n, d, 41)
    rows[1100] = rows[1050]                       # a duplicate inside the second chunk
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        ix.tombstone([1030])
        live = np.setdiff1d(np.arange(n), [1030])
        for m in (None, 0.5):
            got = one_call(ix, m)
            check_pairs(got, want_pairs(ix, live, m), f"{tier}/{m}")
        assert ((got[0] == 1050) & (got[1] == 1100)).any()


def test_thresholds_at_a_planted_pair(rb):
    n, d = 2000, 768
    rows = pair_rows("f64", n, d, 3)
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        _, v, c, _ = ix.search_slots([6], 5, None)
        t = float(v[0, 1])        # the score of 6's best planted neighbour
        for m in (None, 0.5, t, np.nextafter(t, 2.0), np.nextafter(t, -2.0), t - 1e-4, t + 1e-4, 1.0, 1.0000001):
            check_pairs(one_call(ix, m), want_pairs(ix, np.arange(n), m), f"min_score {m!r}")
        a, b, s = one_call(ix, t)
        assert ((a == 6) & (s == t)).any() and not ((a == 6) & (s < t)).any()


def test_oracle_pairwise_cosines(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d = 3000, 384
    bits = synth.random_corpus(n, d, 31)
    bits[1000] = bits[10]
    bits[2000] = bits[10]
    with rb.Index(d) as ix:
        ix.append_bf16(bits)
        a, b, s = one_call(ix, 0.1)
    for q in (0, 10, 1000, 1999, 2999, 777):
        qv = (bits[q].astype(np.uint32) << 16).view(np.float32).astype(np.float64)
        es, ev = oracle_mod.search(bits, qv, n, 0.1)
        keep = np.asarray(es) > q
        m = a == q
        assert (b[m] == np.asarray(es)[keep]).all(), q
        assert s[m].tobytes() == np.asarray(ev)[keep].tobytes(), q
    assert ((a == 10) & (b == 1000)).any() and ((a == 1000) & (b == 2000)).any()


@pytest.mark.parametrize("n", [1, 2, 255, 257, 1023, 1025, 3001])
def test_sizes_across_the_tile_and_the_chunk(rb, n):
    d = 64
    rows = np.random.default_rng(n).standard_normal((n, d))
    for i in range(0, n - 3, 97):
        rows[i + 1] = rows[i] + 0.05 * rows[i + 2]
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        for m in ((None, 0.2, 0.9) if n <= 1100 else (0.2, 0.9)):
            want = want_pairs(ix, np.arange(n), m)
            check_pairs(one_call(ix, m), want, f"n={n} {m}")
            check_pairs(all_pairs(ix, m, max(n, 1)), want, f"n={n} {m}, smallest pages")


def test_tombstones_compaction_and_slot_base(rb):
    n, d, base = 3000, 48, 1_000_000
    rows = pair_rows("f64", n, d, 8)
    with rb.Index(d, keep_f64=True) as ix:
        ix.set_slot_base(base)
        ix.append_f64(rows)
        dead = np.array([0, 2, 7, 1023, 1024, 2999])
        ix.tombstone(dead)                        # local rows
        live = base + np.setdiff1d(np.arange(n), dead)
        for m in (None, 0.3):
            got = all_pairs(ix, m, n)
            check_pairs(got, want_pairs(ix, live, m), f"tombstones {m}")
            assert not np.isin(got[0], base + dead).any() and not np.isin(got[1], base + dead).any()
            assert got[0].min() >= base
        want = one_call(ix, 0.3)
        # mid-index and at the end
        mid = base + 1500
        a, b, s = one_call(ix, 0.3, mid)
        sel = want[0] >= mid
        check_pairs((a, b, s), (want[0][sel], want[1][sel], want[2][sel]), "first_slot mid-index")
        a, b, s, nxt = ix.similar_pairs(0.3, base + n, n)
        assert len(a) == 0 and nxt == base + n
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        ix.tombstone(dead)
        before = one_call(ix, 0.3)
        old_to_new = ix.compact()
        after = one_call(ix, 0.3)
        check_pairs(after, want_pairs(ix, np.arange(ix.size()), 0.3), "after compaction")
        # the same pairs under the new slots (the order within a row can change only through ties on the slot)
        mapped = sorted(zip(old_to_new[before[0]].tolist(), old_to_new[before[1]].tolist(), before[2].tolist()))
        assert mapped == sorted(zip(after[0].tolist(), after[1].tolist(), after[2].tolist()))


def test_paging_and_refusals(rb):
    n, d = 2500, 32
    rows = np.random.default_rng(9).standard_normal((n, d))
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        want = one_call(ix, None)
        for mp in (n, n + 1, 3 * n + 7, 100 * n):
            check_pairs(all_pairs(ix, None, mp), want, f"pages of {mp}")
        a, b, s, nxt = ix.similar_pairs(None, 0, n)   # the smallest buffer: rows until the next would not fit
        assert nxt > 0 and len(a) <= n and len(a) + (n - 1 - nxt) > n
        st0 = ix.stats()
        nat = rb._native
        out = np.empty(n, np.int64), np.empty(n, np.int64), np.empty(n)
        cnt, nx, ms = C.c_int64(-5), C.c_int64(-5), C.c_float(0)

        def raw(m, first, mp, outs=out):
            return nat.lib.rbk_index_similar_pairs_f64(ix._h, m, first, mp, *(nat.ptr(o) for o in outs),
                                                       C.byref(cnt), C.byref(nx), C.byref(ms))
        for args, msg in (((float("nan"), 0, n), "NaN"), ((0.5, -1, n), "first_slot"), ((0.5, n + 1, n), "first_slot"),
                          ((0.5, 0, n - 1), "max_pairs"), ((0.5, 0, 0), "max_pairs")):
            assert raw(*args) == nat.RBK_EINVAL and msg in nat.lib.rbk_last_error().decode(), args
        assert raw(0.5, 0, n, (out[0], None, out[2])) == nat.RBK_EINVAL
        assert cnt.value == -5 and nx.value == -5
        assert ix.stats()["searches"] == st0["searches"] and ix.stats()["kernel_launches"] == st0["kernel_launches"]
        check_pairs(one_call(ix, None), want, "after the refusals")
        # counters: one search, next_slot - first_slot queries
        st0 = ix.stats()
        a, b, s, nxt = ix.similar_pairs(0.2, 100, n)
        st1 = ix.stats()
        assert st1["searches"] - st0["searches"] == 1 and st1["queries"] - st0["queries"] == nxt - 100


def test_minus_inf_pass_over_several_budget_groups_in_bounded_memory(rb):
    import torch
    n, d = 9000, 16
    rows = np.random.default_rng(21).standard_normal((n, d))
    page = 1 << 24
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        all_pairs(ix, None, page)                 # the same pass once: every scratch buffer at its size
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        total, nxt, pages = 0, 0, 0
        while nxt < n:
            a, b, s, nxt2 = ix.similar_pairs(None, nxt, page)
            # the candidates of a page's pairs are more than one budget group (256 MB at 40 bytes each) holds
            if pages == 0:
                assert len(a) * 40 > (256 << 20), len(a)
            if pages in (0, 2):
                pick = np.unique(a)[[0, -1]]
                for q in pick:
                    sv, vv, cv, _ = ix.search_slots([q], n, None)
                    m = sv[0, :cv[0]] > q
                    assert (b[a == q] == sv[0, :cv[0]][m]).all() and s[a == q].tobytes() == vv[0, :cv[0]][m].tobytes()
            total += len(a)
            nxt, pages = nxt2, pages + 1
        free1 = torch.cuda.mem_get_info()[0]
        assert total == n * (n - 1) // 2 and pages >= 3
        assert free0 - free1 < (8 << 20), (free0, free1)


@pytest.mark.parametrize("G", [2, 3, 8])
@pytest.mark.parametrize("tier", ["bf16", "f64", "splithost"])
def test_colocated_group_equals_a_single_index(rb, G, tier):
    n, d = 20000, 160
    rows = pair_rows(tier, n, d, 17)
    with make(rb, d, tier) as ix, make(rb, d, tier, "group", group_devices(G)) as g:
        ix.append_f64(rows)
        g.append_f64(rows)
        ix.tombstone([3, 5000, 9000])
        g.tombstone([3, 5000, 9000])
        for m in (0.3, 0.9):
            want = one_call(ix, m)
            check_pairs(one_call(g, m), want, f"group {G} {m}")
            check_pairs(all_pairs(g, m, n), want, f"group {G} {m}, pages")
            sel = want[0] >= 4100
            check_pairs(one_call(g, m, 4100), (want[0][sel], want[1][sel], want[2][sel]), f"group {G} {m} mid")
        with pytest.raises(rb.RbkError):
            g.similar_pairs(0.3, n + 1, n)


def test_vector_store_similar_pairs(rb, tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(96))
    try:
        words = "api latency database pool redis memory cache gateway error logs restart pods".split()
        rng = np.random.default_rng(2)
        chunks = [{"chunk": {"id": f"c{i}", "documentId": f"d{i % 9}", "content": " ".join(rng.choice(words, 3))},
                   "documentTitle": f"doc {i % 9}", "type": "runbook", "services": ["api"]} for i in range(1500)]
        vs = VectorStore(str(tmp_path / "v.db"), shared=False)
        try:
            vs.add_chunks(chunks)
            got = vs.similar_pairs(0.95)
            ix = vs._index
            a, b, s = want_pairs(ix, np.arange(ix.size()), 0.95)
            ids = vs._ids
            assert got == [(ids[x][4:], ids[y][4:], float(v)) for x, y, v in zip(a, b, s)]
            assert len(got) > 0
            vs.delete_document("d1")
            after = vs.similar_pairs(0.95)
            assert all(not x.startswith("c") or int(x[1:]) % 9 != 1 for p in after for x in p[:2])
        finally:
            vs.close()
    finally:
        embedder.reset()


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_similar_pairs_on_the_gpu_matches_the_oracle(tmp_path, oracle_mod, native, devices):
    """The N-API addon's similarPairs (mock runtime, async work) against librbk_knn.so, on one device and a device
    list: the pages from slot 0 on, concatenated, are the oracle's pairs."""
    import subprocess
    from test_napi_addon import _build_real, _write_inputs
    from test_similar_pairs_host import check_pair_answers
    exe = _build_real()
    w = _write_inputs(tmp_path, devices, n=1200, dim=200, nq=13, k=32)
    # at d = 200 random rows score about N(0, 0.07): some 12,000 pairs, in pages of the smallest size
    (tmp_path / "pairs.txt").write_text("0.15 1200\n")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "has_similar_pairs.txt").read_text() == "1"
    check_pair_answers(tmp_path, w, oracle_mod, 0.15)
