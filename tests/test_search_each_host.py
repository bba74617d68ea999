"""CPU suite for the per-query search (rbk_index_search_each_f64 / rbk_group_search_each_f64): the header and the
library's exports, the refusals that need no device, the Python plumbing, and the micro-batcher serving a window of
mixed callers through one search_each call."""
import ctypes as C
import re
import subprocess
import threading
from pathlib import Path

import numpy as np
import pytest

from common import HashEmbedder, OracleIndex

ROOT = Path(__file__).resolve().parents[1]
EACH = ("rbk_index_search_each_f64", "rbk_group_search_each_f64")


@pytest.fixture(scope="module")
def nat(native):
    from runbookai_b200 import _native
    return _native


def test_header_declares_both_calls():
    h = (ROOT / "include" / "rbk_knn.h").read_text()
    for name, handle in zip(EACH, ("rbk_index* idx", "rbk_group* grp")):
        m = re.search(name + r"\(([^;]*)\);", h)
        assert m, name
        args = " ".join(m.group(1).split())
        assert args.startswith(handle + ", const double* queries, int32_t B, int32_t query_dim, const int32_t* k_fetch, "
                                        "const double* min_score, int64_t* out_slots, double* out_scores, "
                                        "int32_t* out_counts, float*"), args
    assert "#define RBK_ABI_VERSION 2" in h


def test_library_exports_both_calls(nat):
    assert set(EACH) <= set(nat.SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", str(nat.LIB_PATH)], capture_output=True, text=True).stdout
    for name in EACH:
        assert re.search(r"\bT " + name + r"\b", out), name
    assert nat.lib.rbk_abi_version() == 2


def _call(nat, fn, h, B, dim, k, m, outs=True):
    q = np.zeros((max(B, 1), dim))
    kk = None if k is None else np.ascontiguousarray(k, dtype=np.int32)
    mm = None if m is None else np.ascontiguousarray(m, dtype=np.float64)
    K = max(int(kk.max()) if kk is not None and len(kk) else 1, 1)
    slots = np.empty((max(B, 1), K), np.int64)
    scores = np.empty((max(B, 1), K))
    counts = np.empty(max(B, 1), np.int32)
    ms = C.c_float(0)
    st = fn(h, nat.ptr(q), B, dim, nat.ptr(kk), nat.ptr(mm), nat.ptr(slots) if outs else None, nat.ptr(scores),
            nat.ptr(counts), C.byref(ms))
    return st, (nat.lib.rbk_last_error() or b"").decode()


@pytest.mark.parametrize("name", EACH)
def test_refusals_before_any_device_work(nat, name):
    fn = getattr(nat.lib, name)
    st, msg = _call(nat, fn, None, 2, 8, [5, 5], [0.5, 0.5], outs=False)
    assert st == nat.RBK_EINVAL and "null" in msg
    st, msg = _call(nat, fn, None, 2, 8, [5, 5], [0.5, 0.5])
    assert st == nat.RBK_EINVAL and "null" in msg
    st, msg = _call(nat, fn, None, 0, 8, [], [])
    assert st == nat.RBK_EINVAL          # a null handle is refused whatever B is


def test_python_refuses_bad_arrays_before_the_library(nat):
    calls = []

    def fn(*args):
        calls.append(args)
        return nat.RBK_OK
    q = np.ones((2, 4))
    with pytest.raises(nat.RbkError):
        nat._search_each(fn, None, q, [5, 0], [None, None])
    with pytest.raises(ValueError):
        nat._search_each(fn, None, q, [5], [None, None])
    assert not calls


def test_python_plumbing_through_a_recording_stand_in(nat):
    """What _search_each hands the C call: f64 queries, int32 k, float64 thresholds with None as -inf, [B][K] outputs."""
    seen = {}

    def fn(h, qp, B, dim, kp, mp, sp, vp, cp, msp):
        seen.update(h=h, B=B, dim=dim)
        seen["q"] = np.ctypeslib.as_array(C.cast(qp, C.POINTER(C.c_double)), (B, dim)).copy()
        seen["k"] = np.ctypeslib.as_array(C.cast(kp, C.POINTER(C.c_int32)), (B,)).copy()
        seen["m"] = np.ctypeslib.as_array(C.cast(mp, C.POINTER(C.c_double)), (B,)).copy()
        K = int(seen["k"].max())
        slots = np.ctypeslib.as_array(C.cast(sp, C.POINTER(C.c_int64)), (B, K))
        scores = np.ctypeslib.as_array(C.cast(vp, C.POINTER(C.c_double)), (B, K))
        counts = np.ctypeslib.as_array(C.cast(cp, C.POINTER(C.c_int32)), (B,))
        for b in range(B):
            slots[b] = np.arange(K) + 100 * b
            scores[b] = b
            counts[b] = seen["k"][b]
        C.cast(msp, C.POINTER(C.c_float))[0] = 1.5
        return nat.RBK_OK
    q = np.arange(12, dtype=np.float32).reshape(3, 4)
    slots, scores, counts, ms = nat._search_each(fn, "handle", q, [2, 7, 1], [None, 0.5, -1])
    assert seen["h"] == "handle" and seen["B"] == 3 and seen["dim"] == 4
    assert (seen["q"] == q).all() and seen["k"].tolist() == [2, 7, 1]
    assert seen["m"][0] == -np.inf and seen["m"][1:].tolist() == [0.5, -1.0]
    assert slots.shape == (3, 7) and scores.shape == (3, 7) and counts.tolist() == [2, 7, 1] and ms == 1.5
    assert hasattr(nat.Index, "search_each") and hasattr(nat.Group, "search_each")


class EachOracleIndex(OracleIndex):
    """OracleIndex with search_each: each query at its own k and threshold, rows padded to the largest k."""

    def __init__(self, dim, device=0, capacity_hint=0):
        super().__init__(dim, device, capacity_hint)
        self.each_calls = []
        self.search_calls = 0

    def search(self, queries, k_fetch, min_score=0.5):
        self.search_calls += 1
        return super().search(queries, k_fetch, min_score)

    def search_each(self, queries, k_fetch, min_score):
        q = np.atleast_2d(np.asarray(queries, dtype=np.float64))
        self.each_calls.append((len(q), list(k_fetch), list(min_score)))
        K = max(k_fetch)
        slots = np.full((len(q), K), -1, np.int64)
        scores = np.full((len(q), K), np.nan)
        counts = np.zeros(len(q), np.int32)
        for b in range(len(q)):
            s, v, c, _ = super().search(q[b], k_fetch[b], min_score[b])
            slots[b, :k_fetch[b]], scores[b, :k_fetch[b]], counts[b] = s[0], v[0], c[0]
        return slots, scores, counts, 0.0


def _chunks(n, doc, typ, services, text="api latency spike"):
    return [{"chunk": {"id": f"{doc}-c{i}", "documentId": doc, "content": f"{text} {doc} part {i}"},
             "documentTitle": f"title {doc}", "type": typ, "services": list(services)} for i in range(n)]


def test_batcher_serves_mixed_callers_in_one_search_each(tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200.batcher import MicroBatcher
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    made = []

    def factory(d, dev):
        made.append(EachOracleIndex(d))
        return made[-1]
    store = VectorStore(str(tmp_path / "vectors.db"), index_factory=factory)
    try:
        store.add_chunks(_chunks(40, "doc1", "runbook", ("api",)))
        store.add_chunks(_chunks(40, "doc2", "postmortem", ("db",), text="redis connection pool exhausted failover"))
        store.add_chunks(_chunks(40, "doc3", "runbook", ("web",), text="kubernetes pod crashloop oom"))
        asks = [("redis connection pool exhausted", {"topK": 5, "minScore": 0.3}),
                ("pod crashloop oom", {"topK": 57, "minScore": 0.2, "typeFilter": ["runbook"]}),   # 2*topK > 112
                ("redis failover", {"topK": 100, "minScore": 0.1, "serviceFilter": ["db"]}),
                ("connection pool", {}),
                ("api latency", {"topK": 1000, "minScore": 0.05}),
                ("nothing matches this zzz", {"topK": 4})]
        want = [store.search(q, o) for q, o in asks]
        ix = made[0]
        ix.each_calls.clear()
        n_search = ix.search_calls
        mb = MicroBatcher(store, window_ms=300.0, max_batch=64)
        got = [None] * len(asks)
        gate = threading.Barrier(len(asks))

        def worker(i):
            gate.wait()
            got[i] = mb.search(*asks[i])
        threads = [threading.Thread(target=worker, args=(i,)) for i in range(len(asks))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        mb.close()
        assert got == want
        assert mb.batches == 1 and mb.served == len(asks)
        assert ix.search_calls == n_search, "no caller took a search() of its own"
        assert len(ix.each_calls) == 1
        B, ks, mins = ix.each_calls[0]
        assert B == len(asks)
        order = {q: (2 * (o.get("topK") or 10), o.get("minScore") or 0.5) for q, o in asks}
        assert sorted(zip(ks, mins)) == sorted(order.values())
    finally:
        store.close()
        embedder.reset()


# --------------------------------------------------------------------------- the N-API addon's searchEach
@pytest.fixture(scope="module")
def shim_each_harness(tmp_path_factory, oracle_mod):
    from test_unbounded_host import _shim_harness
    return _shim_harness(tmp_path_factory.mktemp("shim_each"), "rbk_shim_each")


@pytest.fixture(scope="module")
def shim_without_each_harness(tmp_path_factory, oracle_mod):
    from test_unbounded_host import _shim_harness
    return _shim_harness(tmp_path_factory.mktemp("shim_without_each"), "rbk_shim_unbounded")


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_each_against_the_oracle_backed_stand_in(tmp_path, oracle_mod, shim_each_harness, devices):
    """searchEach under the mock N-API runtime, as async work on one device and on a device list: row b is the oracle's
    answer at kFetch[b] and minScore[b], -1 / NaN to K = max kFetch; a kFetch of 0 rejects with the library's message
    and a short kFetch throws."""
    from test_napi_addon import _write_inputs
    w = _write_inputs(tmp_path, devices, n=3000, min_score=0.05)
    nq = w["nq"]
    ks = [[1, 5, 24, 112, 113, 1000, 3][b % 7] for b in range(nq)]
    mins = [[0.05, "-inf", 0.1, -0.5][b % 4] for b in range(nq)]
    (tmp_path / "each.txt").write_text("".join(f"{k} {m}\n" for k, m in zip(ks, mins)))
    r = subprocess.run([str(shim_each_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "has_search_each.txt").read_text() == "1"
    K = max(ks)
    slots = np.fromfile(tmp_path / "each_slots.i64", dtype=np.int64).reshape(nq, K)
    scores = np.fromfile(tmp_path / "each_scores.f64", dtype=np.float64).reshape(nq, K)
    counts = np.fromfile(tmp_path / "each_counts.i32", dtype=np.int32)
    for b in range(nq):
        m = None if mins[b] == "-inf" else float(mins[b])
        es, ev = oracle_mod.search(w["corpus"], w["q"][b], ks[b], m, live=w["live"])
        n = len(es)
        assert counts[b] == n and (slots[b, :n] == es).all(), b
        assert scores[b, :n].tobytes() == np.asarray(ev).tobytes(), b
        assert (slots[b, n:] == -1).all() and np.isnan(scores[b, n:]).all(), b
    log = dict(line.split(" ", 1) for line in (tmp_path / "log.txt").read_text().strip().splitlines())
    assert log["err_each"].startswith("k_fetch[0] must be >= 1")
    assert "one entry per query" in log["err_each_len"]


def test_addon_search_each_throws_against_a_library_without_it(tmp_path, oracle_mod, shim_without_each_harness):
    """A library without the per-query search still loads the addon: hasSearchEach is false and searchEach throws,
    after every method before it ran."""
    from test_napi_addon import _write_inputs
    w = _write_inputs(tmp_path, [])
    (tmp_path / "each.txt").write_text("".join(f"{5 + b} 0.1\n" for b in range(w["nq"])))
    r = subprocess.run([str(shim_without_each_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr
    assert (tmp_path / "has_search_each.txt").read_text() == "0"
    err = (tmp_path / "error.txt").read_text()
    assert "searchEach rejected" in err and "no per-query search" in err
    assert (tmp_path / "slots.i64").exists()     # search() before it ran against the same handle


def test_batcher_serves_unshareable_callers_alone(tmp_path):
    """A caller whose 2*topK no shared search_each can carry - below 1, or above 4096 (every row of the shared result
    would be that wide) - goes through VectorStore.search on its own: its error reaches it alone, and the others still
    share one call."""
    from runbookai_b200 import embedder
    from runbookai_b200.batcher import MicroBatcher
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    made = []

    def factory(d, dev):
        made.append(EachOracleIndex(d))
        return made[-1]
    store = VectorStore(str(tmp_path / "vectors.db"), index_factory=factory)
    try:
        store.add_chunks(_chunks(60, "doc1", "runbook", ("api",)))
        store.add_chunks(_chunks(60, "doc2", "postmortem", ("db",), text="redis connection pool exhausted failover"))
        good = [("redis connection pool", {"topK": 5, "minScore": 0.2}), ("api latency", {"topK": 30, "minScore": 0.1}),
                ("failover", {"topK": 3000, "minScore": 0.0})]
        want = [store.search(q, o) for q, o in good]
        ix = made[0]
        ix.each_calls.clear()
        mb = MicroBatcher(store, window_ms=300.0, max_batch=64)
        try:
            futs = [mb.submit(q, o) for q, o in good] + [mb.submit("pool", {"topK": -4})]
            got = [f.result(timeout=60) for f in futs[:3]]
            with pytest.raises(Exception):
                futs[3].result(timeout=60)
        finally:
            mb.close()
        assert got == want
        assert len(ix.each_calls) == 1 and ix.each_calls[0][1] == [10, 60]   # the two shareable callers, one call
        assert mb.batches == 1 and mb.served == 4
    finally:
        store.close()
        embedder.reset()
