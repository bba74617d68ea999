"""CPU suite for diverse hits by maximal marginal relevance (rbk_index_search_mmr_f64 / rbk_group_search_mmr_f64): the
header and the library's exports, the null-handle refusal, the Python plumbing, the MMR oracle on hand-built cases
whose greedy answer is known, VectorStore.search_mmr on an oracle-backed CPU stand-in index, and the addon's searchMmr
on an oracle-backed stand-in of the library, with and without the symbols."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

import mmr_oracle
from common import HashEmbedder, OracleIndex

ROOT = Path(__file__).resolve().parents[1]
MMR = ("rbk_index_search_mmr_f64", "rbk_group_search_mmr_f64")


@pytest.fixture(scope="module")
def nat(native):
    from runbookai_b200 import _native
    return _native


def test_header_declares_both_calls_and_the_fetch_limit():
    h = (ROOT / "include" / "rbk_knn.h").read_text()
    for name, handle in zip(MMR, ("rbk_index* idx", "rbk_group* grp")):
        m = re.search(name + r"\(([^;]*)\);", h)
        assert m, name
        args = " ".join(m.group(1).split())
        assert args == (handle + ", const double* queries, int32_t B, int32_t query_dim, const int32_t* k, const "
                        "int32_t* fetch_k, const double* lambda_mult, const double* min_score, int64_t* out_slots, "
                        "double* out_scores, int32_t* out_counts, float* "
                        + ("kernel_ms_out" if "index" in name else "device_ms_out")), args
    assert "#define RBK_MMR_MAX_FETCH_ELEMS (1 << 25)" in h
    assert "#define RBK_ABI_VERSION 2" in h


def test_library_exports_both_calls(nat):
    assert set(MMR) <= set(nat.SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", str(nat.LIB_PATH)], capture_output=True, text=True).stdout
    for name in MMR:
        assert re.search(r"\bT " + name + r"\b", out), name


@pytest.mark.parametrize("name", MMR)
def test_null_handle_is_refused(nat, name):
    fn = getattr(nat.lib, name)
    q = np.zeros((2, 4))
    k = np.array([5, 5], np.int32)
    f = np.array([50, 50], np.int32)
    lam = np.array([0.5, 0.5])
    m = np.array([0.5, 0.5])
    slots, scores, counts = np.empty((2, 5), np.int64), np.empty((2, 5)), np.empty(2, np.int32)
    ms = C.c_float(0)
    for B in (2, 0):
        st = fn(None, nat.ptr(q), B, 4, nat.ptr(k), nat.ptr(f), nat.ptr(lam), nat.ptr(m), nat.ptr(slots),
                nat.ptr(scores), nat.ptr(counts), C.byref(ms))
        assert st == nat.RBK_EINVAL and "null" in (nat.lib.rbk_last_error() or b"").decode()


def test_python_plumbing_through_a_recording_stand_in(nat):
    """What _search_mmr hands the C call: float64 queries, int32 k and fetch_k, float64 lambda and thresholds (None as
    -inf), scalars broadcast; the [B][K] outputs come back as the call wrote them, tail included."""
    seen = {}

    def fn(h, qp, B, dim, kp, fp, lp, mp, op, vp, cp, msp):
        seen.update(h=h, B=B, dim=dim)
        seen["q"] = np.ctypeslib.as_array(C.cast(qp, C.POINTER(C.c_double)), (B, dim)).copy()
        for key, p, t in (("k", kp, C.c_int32), ("f", fp, C.c_int32), ("l", lp, C.c_double), ("m", mp, C.c_double)):
            seen[key] = np.ctypeslib.as_array(C.cast(p, C.POINTER(t)), (B,)).copy()
        K = int(seen["k"].max())
        out_s = np.ctypeslib.as_array(C.cast(op, C.POINTER(C.c_int64)), (B, K))
        out_v = np.ctypeslib.as_array(C.cast(vp, C.POINTER(C.c_double)), (B, K))
        out_c = np.ctypeslib.as_array(C.cast(cp, C.POINTER(C.c_int32)), (B,))
        for b in range(B):
            c = min(int(seen["k"][b]), 2)
            out_s[b, :c], out_v[b, :c], out_c[b] = 7, 0.25, c
            out_s[b, c:], out_v[b, c:] = -1, np.nan
        C.cast(msp, C.POINTER(C.c_float))[0] = 2.5
        return nat.RBK_OK
    q = np.arange(12, dtype=np.float32).reshape(3, 4)
    slots, scores, counts, ms = nat._search_mmr(fn, "h", q, 3, 40, 0.25, None)
    assert seen["h"] == "h" and seen["B"] == 3 and seen["dim"] == 4 and (seen["q"] == q).all()
    assert seen["k"].tolist() == [3] * 3 and seen["f"].tolist() == [40] * 3 and (seen["l"] == 0.25).all()
    assert (seen["m"] == -np.inf).all() and ms == 2.5
    assert slots.shape == scores.shape == (3, 3) and counts.tolist() == [2, 2, 2]
    assert (slots[:, 2] == -1).all() and np.isnan(scores[:, 2]).all() and (slots[:, :2] == 7).all()
    nat._search_mmr(fn, "h", q[:2], [1, 6], [5, 60], [0.0, 1.0], [0.5, None])
    assert seen["k"].tolist() == [1, 6] and seen["f"].tolist() == [5, 60] and seen["l"].tolist() == [0.0, 1.0]
    assert seen["m"][0] == 0.5 and seen["m"][1] == -np.inf
    # the library checks the values (k < 1, lambda outside [0, 1], ...); a wrong count or a non-int32 is refused here
    nat._search_mmr(fn, "h", q[:1], 0, 5, 2.0, 0.5)
    assert seen["k"].tolist() == [0] and seen["l"].tolist() == [2.0]
    with pytest.raises(ValueError):
        nat._search_mmr(fn, "h", q[:2], [3], 40, 0.5, None)
    with pytest.raises(nat.RbkError):
        nat._search_mmr(fn, "h", q[:1], 3, 2**40, 0.5, None)
    assert hasattr(nat.Index, "search_mmr") and hasattr(nat.Group, "search_mmr")


# ---- the oracle on cases whose greedy answer is known

def test_exact_duplicates_are_never_both_picked_at_half_lambda(oracle_mod):
    # six orthonormal rows, each stored twice (s = 1 to its copy, 0 to the others) and a query with a positive part
    # along each: a copy's mmr is 0.5 * r - 0.5 <= 0 while every unpicked distinct row's is 0.5 * r > 0
    rng = np.random.default_rng(1)
    base = np.linalg.qr(rng.standard_normal((32, 6)))[0].T
    corpus = np.concatenate([base, base])
    q = np.array([1.0, 0.9, 0.7, 0.5, 0.3, 0.2]) @ base
    slots, scores = mmr_oracle.mmr(corpus, q, 6, 12, 0.5, None)
    assert len(slots) == 6 and len({int(s) % 6 for s in slots}) == 6, slots
    plain, pv = oracle_mod.search(corpus, q, 12, None)
    assert slots[0] == plain[0] and scores[0] == pv[0]


@pytest.mark.parametrize("min_score", [None, 0.0, 0.2])
def test_lambda_one_is_the_plain_ranking(oracle_mod, min_score):
    rng = np.random.default_rng(2)
    corpus = rng.standard_normal((300, 24))
    for t in range(5):
        q = rng.standard_normal(24)
        for k, fetch_k in ((1, 1), (5, 50), (50, 50), (40, 400)):
            s, v = mmr_oracle.mmr(corpus, q, k, fetch_k, 1.0, min_score)
            es, ev = oracle_mod.search(corpus, q, fetch_k, min_score)
            assert (s == es[:k]).all() and v.tobytes() == ev[:k].tobytes(), (t, k, fetch_k)


def test_ties_in_mmr_go_to_the_smaller_candidate_index():
    # candidates 1 and 2 have equal relevance and equal similarity to c_0: the smaller index wins
    rows = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0], [0.0, 1.0, 1.0]])
    rel = np.array([0.9, 0.5, 0.5, 0.1])
    assert mmr_oracle.select(rows, rel, 3, 0.5).tolist() == [0, 1, 2]
    # lambda = 0: relevance drops out, every s to c_0 is 0 -> ties everywhere, smallest index first; then the pick
    # least like the picks so far (row 3 is like row 1, row 2 is not)
    assert mmr_oracle.select(rows, rel, 3, 0.0).tolist() == [0, 1, 2]
    # +0 and -0 are one value: a*r - c with r = +-0 ties, the smaller index wins
    rows2 = np.eye(3)
    assert mmr_oracle.select(rows2, np.array([1.0, -0.0, 0.0]), 3, 0.5).tolist() == [0, 1, 2]
    assert mmr_oracle.select(rows2, np.array([1.0, 0.0, -0.0]), 3, 0.5).tolist() == [0, 1, 2]


def test_nan_similarities_rank_below_every_number():
    # row 1 is all zeros: its s is NaN against every pick, so its red stays NaN and its mmr is NaN - it goes last
    rows = np.array([[1.0, 0.0], [0.0, 0.0], [0.0, 1.0], [1.0, 1.0]])
    rel = np.array([0.9, 0.8, 0.1, 0.05])
    assert mmr_oracle.select(rows, rel, 4, 0.5).tolist() == [0, 2, 3, 1]
    # a NaN s never replaces a number: once row 3 has red = s(3, 0), a later NaN leaves it
    rows = np.array([[1.0, 0.0], [np.nan, 0.0], [0.0, 1.0]])
    rel = np.array([0.9, 0.8, 0.7])
    picks = mmr_oracle.select(rows, rel, 3, 0.5)
    assert picks.tolist() == [0, 2, 1]
    # only NaN mmr left: the smallest index
    rows = np.array([[1.0, 0.0], [0.0, 0.0], [0.0, 0.0]])
    assert mmr_oracle.select(rows, np.array([0.9, 0.8, 0.7]), 3, 0.5).tolist() == [0, 1, 2]


def test_k_one_and_empty_candidates(oracle_mod):
    rng = np.random.default_rng(3)
    corpus = rng.standard_normal((50, 8))
    q = rng.standard_normal(8)
    s, v = mmr_oracle.mmr(corpus, q, 1, 30, 0.0, None)
    es, ev = oracle_mod.search(corpus, q, 1, None)
    assert s.tolist() == es.tolist() and v.tobytes() == ev.tobytes()
    s, v = mmr_oracle.mmr(corpus, q, 5, 30, 0.5, 2.0)
    assert len(s) == 0 and len(v) == 0


# ---- VectorStore.search_mmr on an oracle-backed stand-in

class MmrOracleIndex(OracleIndex):
    """OracleIndex with search_mmr: the MMR oracle on the bf16 rows, with search_each's per-query arguments."""

    def search_mmr(self, queries, k, fetch_k, lambda_mult=0.5, min_score=0.5):
        from runbookai_b200._native import RBK_EINVAL, RbkError
        q = np.atleast_2d(np.asarray(queries, dtype=np.float64))
        B = len(q)
        per = lambda v: list(v) if np.ndim(v) else [v] * B   # noqa: E731
        ks, fs, ls, ms = per(k), per(fetch_k), per(lambda_mult), per(min_score)
        for b in range(B):
            if ks[b] < 1 or fs[b] < ks[b] or fs[b] > 4096 or not 0.0 <= ls[b] <= 1.0:
                raise RbkError(RBK_EINVAL, "bad MMR argument")
        self.calls = getattr(self, "calls", []) + [(ks, fs, ls, ms)]
        s, v, c = mmr_oracle.mmr_rows(self.rows, q, ks, fs, ls, ms, live=self.live)
        return s + self.slot_base * (s >= 0), v, c, 0.0


def _chunks(n, doc, typ, services, text):
    return [{"chunk": {"id": f"{doc}-c{i}", "documentId": doc, "content": f"{text} {doc} part {i % 3}"},
             "documentTitle": f"title {doc}", "type": typ, "services": list(services)} for i in range(n)]


ALL = (_chunks(30, "doc1", "runbook", ("api",), "api latency spike")
       + _chunks(30, "doc2", "postmortem", ("db",), "api latency redis connection pool exhausted failover")
       + _chunks(30, "doc3", "runbook", ("web", "db"), "api kubernetes pod crashloop oom"))


def _store(tmp_path, chunks=ALL):
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    store = VectorStore(str(tmp_path / "m.db"), index_factory=lambda d, dev: MmrOracleIndex(d))
    store.add_chunks(chunks)
    return store


def _want(store, query, top_k, fetch_k, lam, min_score, select, type_filter=None, service_filter=None):
    """The oracle's picks for the query's embedding, hydrated by hand: rows of the picks, filtered, in selection
    order, cut at top_k."""
    from runbookai_b200 import embedder
    ix = store._index
    q = np.asarray(embedder.embed_text(query), dtype=np.float64)
    s, v = mmr_oracle.mmr(ix.rows, q, select, fetch_k, lam, min_score, live=ix.live)
    out = []
    for slot, score in zip(s, v):
        row = store.db.execute("SELECT chunk_id, type, services FROM vector_embeddings WHERE id = ?",
                               (store._ids[int(slot)],)).fetchone()
        import json
        if type_filter and row["type"] not in type_filter:
            continue
        if service_filter and not any(x in json.loads(row["services"]) for x in service_filter):
            continue
        out.append((row["chunk_id"], float(score)))
    return out[:top_k]


def test_search_mmr_defaults_filters_and_selection_order(tmp_path):
    from runbookai_b200 import embedder
    store = _store(tmp_path)
    try:
        got = store.search_mmr("api latency spike part 1", {"minScore": 0.1})
        assert store._index.calls[-1] == ([20], [100], [0.5], [0.1])   # select min(2*topK, fetchK), fetchK 10*topK
        want = _want(store, "api latency spike part 1", 10, 100, 0.5, 0.1, 20)
        assert [(r.id, r.score) for r in got] == want and len(got) == 10
        # selection order is kept: not sorted by score
        scores = [r.score for r in got]
        assert scores != sorted(scores, reverse=True)
        # MMR spreads the picks over the documents; the plain ranking of the same store does not
        plain = store.search("api latency spike part 1", {"minScore": 0.1})
        assert len({r.id.split("-")[0] for r in got}) > len({r.id.split("-")[0] for r in plain[:3]})
        # reference defaults: topK 10, minScore 0.5 (js_or: 0 / None fall back)
        store.search_mmr("api latency spike", {"topK": 0, "minScore": 0})
        assert store._index.calls[-1] == ([20], [100], [0.5], [0.5])
        # the filters apply after the selection
        for o, tf, sf in (({"typeFilter": ["postmortem"]}, ["postmortem"], None),
                          ({"serviceFilter": ["db"]}, None, ["db"]),
                          ({"typeFilter": ["runbook"], "serviceFilter": ["web"]}, ["runbook"], ["web"])):
            o = {**o, "topK": 4, "minScore": 0.05, "lambdaMult": 0.3, "fetchK": 60}
            got = store.search_mmr("redis api pool", o)
            assert store._index.calls[-1] == ([8], [60], [0.3], [0.05])
            assert [(r.id, r.score) for r in got] == _want(store, "redis api pool", 4, 60, 0.3, 0.05, 8, tf, sf)
        # fetchK below 2*topK selects fetchK; lambdaMult 1 is search()'s ranking
        store.search_mmr("api", {"topK": 10, "fetchK": 12, "minScore": 0.05})
        assert store._index.calls[-1] == ([12], [12], [0.5], [0.05])
        a = store.search_mmr("api oom", {"topK": 7, "minScore": 0.05, "lambdaMult": 1})
        b = store.search("api oom", {"topK": 7, "minScore": 0.05})
        # (the same scores; which of several equal-scored chunks make the cut differs: search() keeps the database's
        # row order among them, MMR the candidates' slot order)
        assert [r.score for r in a] == [r.score for r in b]
        assert [(r.id, r.score) for r in a] == _want(store, "api oom", 7, 100, 1.0, 0.05, 14)
        # batch
        batch = store.search_mmr_batch(["api", "oom pod"], {"topK": 3, "minScore": 0.05})
        assert [[r.id for r in x] for x in batch] == [[r.id for r in store.search_mmr(t, {"topK": 3, "minScore": 0.05})]
                                                      for t in ("api", "oom pod")]
    finally:
        store.close()
        embedder.reset()


def test_search_mmr_refusals(tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200._native import DimensionError
    store = _store(tmp_path)
    try:
        for lam in (-0.1, 1.5, float("nan")):
            with pytest.raises(ValueError):
                store.search_mmr("api", {"lambdaMult": lam})
        embedder.reset()
        with pytest.raises(RuntimeError):
            store.search_mmr("api")
        embedder.configure(HashEmbedder(64))
        store._set("vec_odd", np.ones(5))     # another length in the Map: the reference's search throws
        with pytest.raises(DimensionError):
            store.search_mmr("api")
    finally:
        store.close()
        embedder.reset()


# ---- the N-API addon's searchMmr

@pytest.fixture(scope="module")
def shim_mmr_harness(tmp_path_factory, oracle_mod):
    from test_unbounded_host import _shim_harness
    return _shim_harness(tmp_path_factory.mktemp("shim_mmr"), "rbk_shim_mmr")


@pytest.fixture(scope="module")
def shim_without_mmr_harness(tmp_path_factory, oracle_mod):
    from test_unbounded_host import _shim_harness
    return _shim_harness(tmp_path_factory.mktemp("shim_without_mmr"), "rbk_shim_each")


def mmr_queries(nq):
    """One "k fetchK lambdaMult minScore" line per query: both routes, k from 1 to fetchK, every lambda band."""
    ks = [1, 5, 10, 30, 3, 100, 2, 8, 20]
    fs = [1, 50, 112, 30, 113, 1000, 40, 8, 300]
    lams = [0.5, 0.0, 0.25, 0.5, 1.0, 0.5, 0.9, 0.3, 0.7]
    mins = ["-inf", 0.05, "-inf", 0.1, "-inf", 0.0, -0.5, "-inf", 0.05]
    return [(ks[b % 9], fs[b % 9], lams[b % 9], mins[b % 9]) for b in range(nq)]


def write_mmr(d, w):
    lines = mmr_queries(w["nq"])
    (d / "mmr.txt").write_text("".join(f"{k} {f} {lam} {m}\n" for k, f, lam, m in lines))
    return lines


def check_mmr_answers(d, w):
    lines = mmr_queries(w["nq"])
    ks, fs, lams = [x[0] for x in lines], [x[1] for x in lines], [x[2] for x in lines]
    mins = [None if x[3] == "-inf" else float(x[3]) for x in lines]
    K = max(ks)
    slots = np.fromfile(d / "mmr_slots.i64", dtype=np.int64).reshape(w["nq"], K)
    scores = np.fromfile(d / "mmr_scores.f64", dtype=np.float64).reshape(w["nq"], K)
    counts = np.fromfile(d / "mmr_counts.i32", dtype=np.int32)
    es, ev, ec = mmr_oracle.mmr_rows(w["corpus"], w["q"], ks, fs, lams, mins, live=w["live"])
    assert (counts == ec).all() and (slots == es).all(), np.flatnonzero((slots != es).any(axis=1))
    assert scores.tobytes() == ev.tobytes()
    log = dict(line.split(" ", 1) for line in (d / "log.txt").read_text().strip().splitlines())
    assert log["err_mmr"].startswith("k[0] must be >= 1")
    assert log["err_mmr_lambda"].startswith("lambda_mult[0] must be in [0, 1]")


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_mmr_against_the_oracle_backed_stand_in(tmp_path, oracle_mod, shim_mmr_harness, devices):
    """searchMmr under the mock N-API runtime, as async work on one device and on a device list: row b is the MMR
    oracle's answer for query b; a k of 0 and a lambdaMult of 2 reject with the library's message."""
    from test_napi_addon import _write_inputs
    w = _write_inputs(tmp_path, devices, n=3000, min_score=0.05)
    write_mmr(tmp_path, w)
    r = subprocess.run([str(shim_mmr_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "has_search_mmr.txt").read_text() == "1"
    check_mmr_answers(tmp_path, w)


def test_addon_search_mmr_throws_against_a_library_without_it(tmp_path, oracle_mod, shim_without_mmr_harness):
    """A library without MMR still loads the addon: hasSearchMmr is false and searchMmr throws, after every method
    before it ran."""
    from test_napi_addon import _write_inputs
    w = _write_inputs(tmp_path, [])
    write_mmr(tmp_path, w)
    r = subprocess.run([str(shim_without_mmr_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr
    assert (tmp_path / "has_search_mmr.txt").read_text() == "0"
    err = (tmp_path / "error.txt").read_text()
    assert "searchMmr rejected" in err and "no MMR search" in err
    assert (tmp_path / "slots.i64").exists()     # search() before it ran against the same handle
