"""GPU suite (-m gpu) for rbk_index_search_mmr_f64 / rbk_group_search_mmr_f64: diverse hits by maximal marginal
relevance.  Bar: every row is bit for bit (slots, counts, fp64 score bytes, the -1 / NaN tail) the MMR oracle's answer
on the stored values (tests/mmr_oracle.py), on every storage tier, and at lambda = 1 the search_each row."""
import numpy as np
import pytest

import mmr_oracle
from common import HashEmbedder, group_devices
from test_gpu_search_slots import TIERS, WIDTHS, check_rows, make, rows_for, thresholds

pytestmark = pytest.mark.gpu

LAMS = [0.0, 0.25, 0.5, 1.0]


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def corpus_of(ix, tier, rows):
    """What the oracle scans: the bf16 rows the index holds, or the exact rows."""
    return ix.read_rows_bf16(0, ix.size()) if tier == "bf16" else rows


def check_oracle(ix, tier, rows, q, ks, fs, lams, mins, live=None, base=0, what=""):
    st0 = ix.stats()
    got = ix.search_mmr(q, ks, fs, lams, mins)
    st1 = ix.stats()
    assert st1["searches"] - st0["searches"] == 1 and st1["queries"] - st0["queries"] == len(q), what
    s, v, c = mmr_oracle.mmr_rows(corpus_of(ix, tier, rows), q, ks, fs, lams, mins, live)
    s = np.where(s >= 0, s + base, s)
    check_rows(got, (s, v, c, 0.0), what)
    return got


def queries_for(rows, n_q, seed):
    """Stored rows, the same rows nudged, and fresh directions: many near-ties among the candidates."""
    rng = np.random.default_rng(seed)
    n, d = rows.shape
    pick = rng.integers(0, n, n_q)
    q = rows[pick].copy()
    q[1::3] += 0.05 * rng.standard_normal((len(q[1::3]), d))
    q[2::3] = rng.standard_normal((len(q[2::3]), d))
    return np.nan_to_num(q, nan=0.5)


@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("tier", list(TIERS))
def test_rows_equal_the_oracle_on_the_stored_values(rb, tier, d):
    n = 1500
    rows = rows_for(tier, n, d, d + 1)
    rows[700:710] = rows[600]          # exact duplicates: ties in s and in mmr
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        ix.tombstone([603, 1200])
        live = np.ones(n, np.uint8)
        live[[603, 1200]] = 0
        q = np.concatenate([queries_for(rows, 10, d), rows[[600, n - 4, n - 3, n - 1]]])
        q = np.nan_to_num(q, nan=0.0) if tier != "bf16" else q
        q[-3] = rows[n - 3]            # a query with a NaN
        B = len(q)
        mins = thresholds(ix, q)
        big = 40 if d > 1000 else 120
        for fs_set, ks_set in (([1, 30, 112, 8], [1, 7, 112, 2]),                 # the scan route
                               ([113, 600, 4096, 2000], [3, big, 20, 1])):         # the large-k route, past count()
            fs = [fs_set[b % 4] for b in range(B)]
            ks = [min(ks_set[(b // 4) % 4], fs[b]) for b in range(B)]
            lams = [LAMS[b % 4] for b in range(B)]
            check_oracle(ix, tier, rows, q, ks, fs, lams, mins, live, what=f"{tier}/{d}/{fs_set}")


def test_float_range_rows(rb):
    """Rows whose cosines are +-inf (norms underflow), +-0 (norms overflow) or NaN (zero rows, a NaN element)."""
    n, d = 600, 64
    rng = np.random.default_rng(9)
    rows = rng.standard_normal((n, d))
    rows[0:40] *= 2.0 ** -565
    rows[40:80] *= 2.0 ** 600
    rows[80:90] = 0.0
    rows[90:100, 3] = np.nan
    rows[100:140] = rows[140:180] + 1e-3 * rng.standard_normal((40, d))
    q = np.concatenate([rows[[0, 41, 100, 300]], rng.standard_normal((4, d)), rows[[5, 45]] * 2.0 ** 10])
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        B = len(q)
        for fs, ks in ((50, 20), (500, 60)):
            for lam in LAMS:
                check_oracle(ix, "f64", rows, q, [ks] * B, [fs] * B, [lam] * B, [None] * B, what=f"{fs}/{lam}")


def test_k_from_one_to_fetch_k_and_lambda_one_is_search_each(rb):
    n, d = 3000, 96
    rows = np.random.default_rng(10).standard_normal((n, d))
    rows[1000:1100] = rows[1100:1200] + 0.01 * np.random.default_rng(11).standard_normal((100, d))
    q = queries_for(rows, 12, 12)
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        for fs in (1, 20, 112, 113, 400):
            for k in sorted({min(2, fs), fs // 2 or 1, fs, 1}):
                check_oracle(ix, "f64", rows, q, [k] * 12, [fs] * 12, [0.5] * 12, [None] * 12, what=f"{k}/{fs}")
                s, v, c, _ = ix.search_mmr(q, k, fs, 1.0, None)
                es, ev, ec, _ = ix.search_each(q, [fs] * 12, [None] * 12)
                check_rows((s, v, c, 0), (es[:, :k], ev[:, :k], np.minimum(ec, k), 0), f"lambda 1 {k}/{fs}")
                if k == 1:
                    check_rows((s, v, c, 0), (es[:, :1], ev[:, :1], np.minimum(ec, 1), 0), f"k 1 {fs}")


def test_mixed_batch_rows_equal_each_query_alone(rb):
    n, d = 4000, 128
    rows = rows_for("f64", n, d, 13)
    q = queries_for(rows, 16, 14)
    ks = [1, 5, 10, 40, 3, 100, 7, 2] * 2
    fs = [10, 50, 112, 4000, 113, 1000, 7, 2] * 2
    lams = [0.0, 0.25, 0.5, 1.0] * 4
    mins = [None, 0.1, None, 0.0] * 4
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        s, v, c, _ = ix.search_mmr(q, ks, fs, lams, mins)
        for b in range(len(q)):
            s1, v1, c1, _ = ix.search_mmr(q[b:b + 1], ks[b], fs[b], lams[b], mins[b])
            K1 = s1.shape[1]
            assert c[b] == c1[0] and (s[b, :K1] == s1[0]).all() and v[b, :K1].tobytes() == v1[0].tobytes(), b
            assert (s[b, K1:] == -1).all() and np.isnan(v[b, K1:]).all(), b


def test_more_than_1024_queries_and_several_budget_groups(rb):
    n, d = 6000, 1536
    rng = np.random.default_rng(15)
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((1100, d))
    # 4096 candidates of 1536 float64 = 48 MiB per query: six queries per 256 MiB group
    fs = [4096 if b % 50 == 0 or b >= 1090 else 20 for b in range(1100)]
    ks = [10 if f == 4096 else 3 for f in fs]
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        s, v, c, _ = ix.search_mmr(q, ks, fs, 0.5, None)
        assert (c == ks).all()
        pick = [0, 1, 50, 1023, 1024, 1050, 1090, 1095, 1099]
        es, ev, ec = mmr_oracle.mmr_rows(rows, q[pick], [ks[b] for b in pick], [fs[b] for b in pick], [0.5] * 9,
                                         [None] * 9)
        check_rows((s[pick], v[pick], c[pick], 0), (es, ev, ec, 0), "B 1100")


def test_slot_base_refusals_and_argument_order(rb):
    n, d, base = 2000, 48, 1_000_000
    rows = rows_for("f64", n, d, 16)
    q = queries_for(rows, 6, 17)
    with rb.Index(d, keep_f64=True) as ix:
        ix.set_slot_base(base)
        ix.append_f64(rows)
        got = check_oracle(ix, "f64", rows, q, [5, 20, 1, 8, 3, 40], [50, 20, 1, 300, 4096, 200], LAMS + [0.5, 0.5],
                           [None, 0.5, None, 0.0, None, None], base=base, what="slot_base")
        assert (got[0][got[0] >= 0] >= base).all()
        E, D = rb._native.RBK_EINVAL, rb._native.RBK_EDIM

        def refused(status, text, qq, k, f, lam, m):
            with pytest.raises(rb.RbkError) as e:
                ix.search_mmr(qq, k, f, lam, m)
            assert e.value.status == status and text in str(e.value), (text, str(e.value))
        refused(E, "k[0] must be >= 1", q[:1], 0, 5, 0.5, None)
        refused(E, "fetch_k[1] must be >= k[1]", q[:2], [3, 6], [5, 5], 0.5, None)
        refused(E, "fetch_k[0] must be <= 4096", q[:1], 3, 4097, 0.5, None)
        # the checks run in order: a bad k before a wrong width before a bad lambda or a NaN threshold
        refused(E, "k[0]", q[:1, :7], 0, 5, 2.0, float("nan"))
        refused(D, "same length", q[:1, :7], 3, 5, 2.0, float("nan"))
        refused(E, "min_score[0] is NaN", q[:1], 3, 5, 2.0, float("nan"))
        for lam in (-0.01, 1.01, float("nan")):
            refused(E, "lambda_mult[0] must be in [0, 1]", q[:1], 3, 5, lam, None)
        s, v, c, ms = ix.search_mmr(q[:0], 3, 5, 0.5, None)
        assert s.shape == (0, 0) and c.shape == (0,)
    with rb.Index(8193, keep_f64=True) as wide:
        with pytest.raises(rb.RbkError) as e:
            wide.search_mmr(np.ones((1, 8193)), 1, 4096, 0.5, None)   # 4096 * 8193 > 2^25 elements
        assert e.value.status == rb._native.RBK_EINVAL and "RBK_MMR_MAX_FETCH_ELEMS" in str(e.value)
        s, v, c, _ = wide.search_mmr(np.ones((1, 8193)), 1, 4095, 0.5, None)   # the largest that fits
        assert c.tolist() == [0] and s.tolist() == [[-1]]


def test_mutations_compaction_and_tiers(rb):
    n, d = 5000, 96
    rows = rows_for("f64", n, d, 18)
    q = queries_for(rows, 8, 19)
    ks, fs, lams = [5, 10, 1, 30] * 2, [50, 112, 1000, 300] * 2, LAMS * 2
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        ix.tombstone(np.arange(0, n, 5))
        old_to_new = ix.compact()
        rows = rows[old_to_new >= 0]
        check_oracle(ix, "f64", rows, q, ks, fs, lams, [None] * 8, what="compact")
        for kw in ({"f64_on_host": True}, {"scan_f16": True}, {"f64_on_host": False, "scan_f16": False}):
            ix.set_tier(**kw)
            check_oracle(ix, "f64", rows, q, ks, fs, lams, [None] * 8, what=f"tier {kw}")


def test_repeated_calls_stay_within_the_budget_and_trim_returns_it(rb):
    import torch
    n, d = 20000, 1024
    rows = np.random.default_rng(20).standard_normal((n, d))
    q = np.random.default_rng(21).standard_normal((64, d))
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(rows)
        torch.cuda.synchronize()
        free_before = torch.cuda.mem_get_info()[0]
        first = ix.search_mmr(q, 10, 4096, 0.5, None)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        for _ in range(3):
            again = ix.search_mmr(q, 10, 4096, 0.5, None)
            check_rows(again, first, "repeat")
        free1 = torch.cuda.mem_get_info()[0]
        assert free0 - free1 < (8 << 20), (free0, free1)
        assert free_before - free1 < (512 << 20), (free_before, free1)   # staging + search scratch
        ix.trim()
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] - free1 > (200 << 20)


@pytest.mark.parametrize("G", [2, 3, 8])
@pytest.mark.parametrize("tier", ["bf16", "f64", "splithost"])
def test_colocated_group_equals_a_single_index(rb, G, tier):
    n, d = 20000, 160
    rows = rows_for(tier, n, d, 22)
    q = queries_for(rows, 12, 23)
    with make(rb, d, tier) as ix, make(rb, d, tier, "group", group_devices(G)) as g:
        ix.append_f64(rows)
        g.append_f64(rows)
        ix.tombstone([3, 5000, 9000])
        g.tombstone([3, 5000, 9000])
        mins = thresholds(ix, q)
        for fs, ks in (([5, 112, 1, 40] * 3, [2, 20, 1, 40] * 3), ([113, 1000, 4096, 300] * 3, [10, 3, 50, 1] * 3)):
            lams = LAMS * 3
            a = ix.search_mmr(q, ks, fs, lams, mins)
            check_rows(g.search_mmr(q, ks, fs, lams, mins), a, f"group {G} {fs[:4]}")
        g.trim()
        check_rows(g.search_mmr(q, ks, fs, lams, mins), a, f"group {G} after trim")


def test_vector_store_search_mmr_on_the_library(rb, tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(96))
    try:
        words = "api latency database pool redis memory cache gateway error logs restart pods".split()
        rng = np.random.default_rng(2)
        chunks = [{"chunk": {"id": f"c{i}", "documentId": f"d{i % 9}", "content": " ".join(rng.choice(words, 3))},
                   "documentTitle": f"doc {i % 9}", "type": ["runbook", "postmortem"][i % 2],
                   "services": [["api"], ["db"]][i % 3 % 2]} for i in range(1500)]
        vs = VectorStore(str(tmp_path / "v.db"), shared=False)
        try:
            vs.add_chunks(chunks)
            ix = vs._index
            for text, o in (("api latency", {}), ("redis pool error", {"topK": 20, "minScore": 0.2,
                                                                      "typeFilter": ["runbook"]}),
                            ("cache gateway", {"topK": 5, "lambdaMult": 0.9, "fetchK": 3000})):
                got = vs.search_mmr(text, o)
                top_k = o.get("topK", 10)
                fetch_k = o.get("fetchK", min(4096, 10 * top_k))
                qv = np.asarray(embedder.embed_text(text), dtype=np.float64)
                s, v, c, _ = ix.search_mmr(qv, min(2 * top_k, fetch_k), fetch_k, o.get("lambdaMult", 0.5),
                                           o.get("minScore", 0.5))
                picked = [vs._ids[int(x)].removeprefix("vec_") for x in s[0, :c[0]]]
                if "typeFilter" in o:
                    types = {ch["chunk"]["id"]: ch["type"] for ch in chunks}
                    picked = [p for p in picked if types[p] in o["typeFilter"]]
                assert [r.id for r in got] == picked[:top_k], (text, o)
                es, ev, ec = mmr_oracle.mmr_rows(ix.read_rows_bf16(0, ix.size()), qv[None], [min(2 * top_k, fetch_k)],
                                                 [fetch_k], [o.get("lambdaMult", 0.5)], [o.get("minScore", 0.5)])
                check_rows((s, v, c, 0), (es, ev, ec, 0), text)
        finally:
            vs.close()
    finally:
        embedder.reset()


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_mmr_on_the_gpu_matches_the_oracle(tmp_path, oracle_mod, native, devices):
    """The N-API addon's searchMmr (mock runtime, async work) against librbk_knn.so, on one device and a device list:
    row b is the MMR oracle's answer for query b, on both candidate routes."""
    import subprocess
    from test_napi_addon import _build_real, _write_inputs
    from test_mmr_host import check_mmr_answers, write_mmr
    exe = _build_real()
    w = _write_inputs(tmp_path, devices, n=6000, dim=200, nq=13, k=32)
    write_mmr(tmp_path, w)
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "has_search_mmr.txt").read_text() == "1"
    check_mmr_answers(tmp_path, w)
