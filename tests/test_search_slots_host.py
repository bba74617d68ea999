"""CPU suite for stored rows as queries (rbk_index_search_slots_f64 / rbk_group_search_slots_f64): the header and the
library's exports, the null-handle refusal, the Python plumbing, and VectorStore.search_similar on a CPU stand-in
index against search() with an embedder that hands back the stored embedding."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from common import HashEmbedder, OracleIndex

ROOT = Path(__file__).resolve().parents[1]
SLOTS = ("rbk_index_search_slots_f64", "rbk_group_search_slots_f64")


@pytest.fixture(scope="module")
def nat(native):
    from runbookai_b200 import _native
    return _native


def test_header_declares_both_calls():
    h = (ROOT / "include" / "rbk_knn.h").read_text()
    for name, handle in zip(SLOTS, ("rbk_index* idx", "rbk_group* grp")):
        m = re.search(name + r"\(([^;]*)\);", h)
        assert m, name
        args = " ".join(m.group(1).split())
        assert args == (handle + ", const int64_t* query_slots, int32_t B, const int32_t* k_fetch, const double* "
                        "min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts, float* "
                        + ("kernel_ms_out" if "index" in name else "device_ms_out")), args
    assert "#define RBK_ABI_VERSION 2" in h


def test_library_exports_both_calls(nat):
    assert set(SLOTS) <= set(nat.SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", str(nat.LIB_PATH)], capture_output=True, text=True).stdout
    for name in SLOTS:
        assert re.search(r"\bT " + name + r"\b", out), name


@pytest.mark.parametrize("name", SLOTS)
def test_null_handle_is_refused(nat, name):
    fn = getattr(nat.lib, name)
    sl = np.zeros(2, np.int64)
    k = np.array([5, 5], np.int32)
    m = np.array([0.5, 0.5])
    slots, scores, counts = np.empty((2, 5), np.int64), np.empty((2, 5)), np.empty(2, np.int32)
    ms = C.c_float(0)
    for B in (2, 0):
        st = fn(None, nat.ptr(sl), B, nat.ptr(k), nat.ptr(m), nat.ptr(slots), nat.ptr(scores), nat.ptr(counts),
                C.byref(ms))
        assert st == nat.RBK_EINVAL and "null" in (nat.lib.rbk_last_error() or b"").decode()


def test_python_plumbing_through_a_recording_stand_in(nat):
    """What _search_slots hands the C call: int64 slots, int32 k (a scalar broadcast), float64 thresholds with None as
    -inf, [B][K] outputs."""
    seen = {}

    def fn(h, sp, B, kp, mp, op, vp, cp, msp):
        seen.update(h=h, B=B)
        seen["s"] = np.ctypeslib.as_array(C.cast(sp, C.POINTER(C.c_int64)), (B,)).copy()
        seen["k"] = np.ctypeslib.as_array(C.cast(kp, C.POINTER(C.c_int32)), (B,)).copy()
        seen["m"] = np.ctypeslib.as_array(C.cast(mp, C.POINTER(C.c_double)), (B,)).copy()
        K = int(seen["k"].max())
        np.ctypeslib.as_array(C.cast(op, C.POINTER(C.c_int64)), (B, K))[:] = 7
        np.ctypeslib.as_array(C.cast(vp, C.POINTER(C.c_double)), (B, K))[:] = 0.25
        np.ctypeslib.as_array(C.cast(cp, C.POINTER(C.c_int32)), (B,))[:] = K
        C.cast(msp, C.POINTER(C.c_float))[0] = 2.5
        return nat.RBK_OK
    slots, scores, counts, ms = nat._search_slots(fn, "h", [4, 9, 2**40], 6, None)
    assert seen["h"] == "h" and seen["B"] == 3 and seen["s"].tolist() == [4, 9, 2**40]
    assert seen["k"].tolist() == [6, 6, 6] and (seen["m"] == -np.inf).all()
    assert slots.shape == (3, 6) and (slots == 7).all() and (scores == 0.25).all() and ms == 2.5
    nat._search_slots(fn, "h", [1, 2], [3, 8], [0.5, None])
    assert seen["k"].tolist() == [3, 8] and seen["m"][0] == 0.5 and seen["m"][1] == -np.inf
    with pytest.raises(nat.RbkError):
        nat._search_slots(fn, "h", [1, 2], [3, 0], None)
    with pytest.raises(ValueError):
        nat._search_slots(fn, "h", [1, 2], [3], None)
    assert hasattr(nat.Index, "search_slots") and hasattr(nat.Group, "search_slots")


class SlotsOracleIndex(OracleIndex):
    """OracleIndex with search_slots (the stored bf16 row widened is the query) and compact."""

    def search_slots(self, slots, k_fetch, min_score):
        slots = np.asarray(slots, np.int64).reshape(-1)
        ks = np.broadcast_to(np.asarray(k_fetch), slots.shape)
        for s in slots:
            if not (0 <= s - self.slot_base < self.size()) or not self.live[s - self.slot_base]:
                from runbookai_b200._native import RBK_EINVAL, RbkError
                raise RbkError(RBK_EINVAL, "query slot not held or tombstoned")
        q = (self.rows[slots - self.slot_base].astype(np.uint32) << 16).view(np.float32).astype(np.float64)
        K = int(ks.max())
        out_s = np.full((len(slots), K), -1, np.int64)
        out_v = np.full((len(slots), K), np.nan)
        out_c = np.zeros(len(slots), np.int32)
        for b in range(len(slots)):
            s, v, c, _ = self.search(q[b], int(ks[b]), min_score)
            out_s[b, :ks[b]], out_v[b, :ks[b]], out_c[b] = s[0], v[0], c[0]
        return out_s, out_v, out_c, 0.0

    def compact(self):
        keep = self.live.astype(bool)
        old_to_new = np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int64)
        self.rows, self.live = self.rows[keep], self.live[keep]
        return old_to_new


def _chunks(n, doc, typ, services, text):
    return [{"chunk": {"id": f"{doc}-c{i}", "documentId": doc, "content": f"{text} {doc} part {i}"},
             "documentTitle": f"title {doc}", "type": typ, "services": list(services)} for i in range(n)]


ALL = (_chunks(30, "doc1", "runbook", ("api",), "api latency spike")
       + _chunks(30, "doc2", "postmortem", ("db",), "redis connection pool exhausted failover")
       + _chunks(30, "doc3", "runbook", ("web", "db"), "kubernetes pod crashloop oom"))
OPTIONS = [{}, {"topK": 3, "minScore": 0.2}, {"topK": 8, "minScore": 0.1, "typeFilter": ["runbook"]},
           {"topK": 70, "minScore": 0.05, "serviceFilter": ["db"]},
           {"topK": 5, "minScore": 0.0, "typeFilter": ["postmortem"], "serviceFilter": ["db"]}]


class StoredEmbedder:
    """search(f"vec_{chunk id}") through this embedder queries with that chunk's stored embedding."""

    def __init__(self, store):
        self.store = store

    def embed_text(self, text):
        from runbookai_b200.vector_store import buffer_to_float_array
        row = self.store.db.execute("SELECT embedding FROM vector_embeddings WHERE id = ?", (text,)).fetchone()
        return buffer_to_float_array(row["embedding"])

    def embed_texts(self, texts):
        return [self.embed_text(t) for t in texts]


def _store(tmp_path, name, chunks):
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    store = VectorStore(str(tmp_path / f"{name}.db"), index_factory=lambda d, dev: SlotsOracleIndex(d))
    store.add_chunks(chunks)
    return store


def _view(results):
    return [r.to_dict() for r in results]


def test_search_similar_equals_search_with_the_stored_embedding(tmp_path):
    from runbookai_b200 import embedder
    store = _store(tmp_path, "a", ALL)
    try:
        embedder.configure(StoredEmbedder(store))
        for cid in ("doc1-c0", "doc2-c7", "doc3-c29"):
            for o in OPTIONS:
                got = store.search_similar(cid, {**o, "excludeSelf": False})
                assert _view(got) == _view(store.search(f"vec_{cid}", o)), (cid, o)
        batch = store.search_similar_batch(["doc1-c1", "doc3-c2"], {"topK": 4, "excludeSelf": False})
        assert [_view(x) for x in batch] == [_view(store.search(f"vec_{c}", {"topK": 4})) for c in ("doc1-c1", "doc3-c2")]
    finally:
        store.close()
        embedder.reset()


def test_exclude_self_equals_search_on_a_store_without_the_chunk(tmp_path):
    from runbookai_b200 import embedder
    store = _store(tmp_path, "a", ALL)
    try:
        for cid in ("doc1-c0", "doc2-c7", "doc3-c29"):
            embedder.configure(HashEmbedder(64))
            other = _store(tmp_path, f"without-{cid}", [c for c in ALL if c["chunk"]["id"] != cid])
            try:
                q = StoredEmbedder(store).embed_text(f"vec_{cid}")

                class Fixed:
                    def embed_text(self, t):
                        return q

                    def embed_texts(self, ts):
                        return [q for _ in ts]
                embedder.configure(Fixed())
                for o in OPTIONS:
                    got = store.search_similar(cid, o)
                    assert all(r.id != cid for r in got)
                    assert _view(got) == _view(other.search("x", o)), (cid, o)
            finally:
                other.close()
    finally:
        store.close()
        embedder.reset()


def test_unknown_deleted_and_ragged(tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200._native import DimensionError
    store = _store(tmp_path, "a", ALL)
    try:
        embedder.reset()     # no embedder: search_similar never embeds
        with pytest.raises(KeyError):
            store.search_similar("nope")
        store.delete_document("doc2")
        with pytest.raises(KeyError):
            store.search_similar("doc2-c3")
        assert store.search_similar("doc1-c3", {"topK": 2})
        assert store.search_similar_batch([]) == []
        store._set("vec_odd", np.ones(5))     # another length in the Map: the reference's search throws
        with pytest.raises(DimensionError):
            store.search_similar("doc1-c3")
    finally:
        store.close()


def test_slots_follow_compaction(tmp_path):
    from runbookai_b200 import embedder
    store = _store(tmp_path, "a", ALL)
    try:
        embedder.configure(StoredEmbedder(store))
        store.delete_document("doc1")
        want = {cid: _view(store.search_similar(cid, {"topK": 6})) for cid in ("doc2-c0", "doc3-c5")}
        assert store.compact() == 30
        for cid, w in want.items():
            assert _view(store.search_similar(cid, {"topK": 6})) == w
            assert _view(store.search_similar(cid, {"topK": 6, "excludeSelf": False})) == \
                _view(store.search(f"vec_{cid}", {"topK": 6}))
    finally:
        store.close()
        embedder.reset()


# --------------------------------------------------------------------------- the N-API addon's searchSlots
@pytest.fixture(scope="module")
def shim_slots_harness(tmp_path_factory, oracle_mod):
    from test_unbounded_host import _shim_harness
    return _shim_harness(tmp_path_factory.mktemp("shim_slots"), "rbk_shim_slots")


@pytest.fixture(scope="module")
def shim_without_slots_harness(tmp_path_factory, oracle_mod):
    from test_unbounded_host import _shim_harness
    return _shim_harness(tmp_path_factory.mktemp("shim_without_slots"), "rbk_shim_each")


def slot_queries(w):
    """Live slots (one of them overwritten, one a tie group's first row) at a mix of k and thresholds."""
    live = np.flatnonzero(w["live"])
    qs = [5, int(live[1]), int(live[-1]), int(live[len(live) // 2]), 17 if w["live"][17] else 5, int(live[100])]
    ks = [1, 5, 24, 112, 113, 1000]
    mins = [0.05, "-inf", 0.1, -0.5, "-inf", 0.2]
    return qs, ks, mins


def check_slot_answers(d, w, oracle_mod):
    qs, ks, mins = slot_queries(w)
    K = max(ks)
    slots = np.fromfile(d / "slots_slots.i64", dtype=np.int64).reshape(len(qs), K)
    scores = np.fromfile(d / "slots_scores.f64", dtype=np.float64).reshape(len(qs), K)
    counts = np.fromfile(d / "slots_counts.i32", dtype=np.int32)
    for b, s in enumerate(qs):
        m = None if mins[b] == "-inf" else float(mins[b])
        es, ev = oracle_mod.search(w["corpus"], w["corpus"][s], ks[b], m, live=w["live"])
        n = len(es)
        assert counts[b] == n and (slots[b, :n] == es).all(), b
        assert scores[b, :n].tobytes() == np.asarray(ev).tobytes(), b
        assert (slots[b, n:] == -1).all() and np.isnan(scores[b, n:]).all(), b
    log = dict(line.split(" ", 1) for line in (d / "log.txt").read_text().strip().splitlines())
    assert log["err_slots"].startswith("k_fetch[0] must be >= 1")
    assert "is not a slot of this" in log["err_slots_range"]


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_slots_against_the_oracle_backed_stand_in(tmp_path, oracle_mod, shim_slots_harness, devices):
    """searchSlots under the mock N-API runtime, as async work on one device and on a device list: row b is the
    oracle's answer for the stored row of slots[b] at kFetch[b] and minScore[b]; a kFetch of 0 and a slot past the end
    reject with the library's message."""
    from test_napi_addon import _write_inputs
    w = _write_inputs(tmp_path, devices, n=3000, min_score=0.05)
    qs, ks, mins = slot_queries(w)
    (tmp_path / "slots.txt").write_text("".join(f"{s} {k} {m}\n" for s, k, m in zip(qs, ks, mins)))
    r = subprocess.run([str(shim_slots_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "has_search_slots.txt").read_text() == "1"
    check_slot_answers(tmp_path, w, oracle_mod)


def test_addon_search_slots_throws_against_a_library_without_it(tmp_path, oracle_mod, shim_without_slots_harness):
    """A library without search by slot still loads the addon: hasSearchSlots is false and searchSlots throws, after
    every method before it ran."""
    from test_napi_addon import _write_inputs
    w = _write_inputs(tmp_path, [])
    qs, ks, mins = slot_queries(w)
    (tmp_path / "slots.txt").write_text("".join(f"{s} {k} {m}\n" for s, k, m in zip(qs, ks, mins)))
    r = subprocess.run([str(shim_without_slots_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr
    assert (tmp_path / "has_search_slots.txt").read_text() == "0"
    err = (tmp_path / "error.txt").read_text()
    assert "searchSlots rejected" in err and "no search by slot" in err
    assert (tmp_path / "slots.i64").exists()     # search() before it ran against the same handle
