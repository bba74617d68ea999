"""CPU suite for every pair of stored rows at or above a threshold (rbk_index_similar_pairs_f64 /
rbk_group_similar_pairs_f64): the header and the library's exports, the null-handle refusal, the Python page loop
against an oracle-backed stand-in of the C call, and VectorStore.similar_pairs on a CPU stand-in index."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from common import HashEmbedder
from test_search_slots_host import ALL, SlotsOracleIndex

ROOT = Path(__file__).resolve().parents[1]
PAIRS = ("rbk_index_similar_pairs_f64", "rbk_group_similar_pairs_f64")


@pytest.fixture(scope="module")
def nat(native):
    from runbookai_b200 import _native
    return _native


def test_header_declares_both_calls():
    h = (ROOT / "include" / "rbk_knn.h").read_text()
    for name, handle in zip(PAIRS, ("rbk_index* idx", "rbk_group* grp")):
        m = re.search(name + r"\(([^;]*)\);", h)
        assert m, name
        args = " ".join(m.group(1).split())
        assert args == (handle + ", double min_score, int64_t first_slot, int64_t max_pairs, int64_t* out_a, int64_t* "
                        "out_b, double* out_scores, int64_t* n_out, int64_t* next_slot, float* "
                        + ("kernel_ms_out" if "index" in name else "device_ms_out")), args
    assert "#define RBK_ABI_VERSION 2" in h


def test_library_exports_both_calls(nat):
    assert set(PAIRS) <= set(nat.SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", str(nat.LIB_PATH)], capture_output=True, text=True).stdout
    for name in PAIRS:
        assert re.search(r"\bT " + name + r"\b", out), name


@pytest.mark.parametrize("name", PAIRS)
def test_null_handle_is_refused(nat, name):
    fn = getattr(nat.lib, name)
    a, b, s = np.empty(4, np.int64), np.empty(4, np.int64), np.empty(4)
    n, nxt, ms = C.c_int64(0), C.c_int64(0), C.c_float(0)
    st = fn(None, 0.5, 0, 4, nat.ptr(a), nat.ptr(b), nat.ptr(s), C.byref(n), C.byref(nxt), C.byref(ms))
    assert st == nat.RBK_EINVAL and "null" in (nat.lib.rbk_last_error() or b"").decode()


class PairsOracleIndex(SlotsOracleIndex):
    """SlotsOracleIndex with similar_pairs: a stand-in for the C call, from the oracle's pairwise cosines, paged by the
    contract (whole rows from first_slot on while they fit in max_pairs), under the library's Python plumbing."""

    def c_call(self, h, min_score, first, max_pairs, pa, pb, ps, pn, pnext, pms):
        from runbookai_b200._native import RBK_EINVAL, RBK_OK
        end = self.slot_base + self.size()
        if min_score != min_score or not (self.slot_base <= first <= end) or max_pairs < max(self.size(), 1):
            return RBK_EINVAL
        out_a = np.ctypeslib.as_array(C.cast(pa, C.POINTER(C.c_int64)), (max_pairs,))
        out_b = np.ctypeslib.as_array(C.cast(pb, C.POINTER(C.c_int64)), (max_pairs,))
        out_s = np.ctypeslib.as_array(C.cast(ps, C.POINTER(C.c_double)), (max_pairs,))
        n, a = 0, first
        m = None if min_score == -np.inf else min_score
        for a in range(first, end):
            if self.live[a - self.slot_base]:
                s, v, c, _ = self.search_slots([a], max(self.count(), 1), m)
                keep = s[0, :c[0]] > a
                k = int(keep.sum())
                if n + k > max_pairs:
                    break
                out_a[n:n + k], out_b[n:n + k], out_s[n:n + k] = a, s[0, :c[0]][keep], v[0, :c[0]][keep]
                n += k
        else:
            a = end
        C.cast(pn, C.POINTER(C.c_int64))[0] = n
        C.cast(pnext, C.POINTER(C.c_int64))[0] = a
        return RBK_OK

    def similar_pairs(self, min_score, first_slot=None, max_pairs=None):
        from runbookai_b200._native import _similar_pairs
        return _similar_pairs(self.c_call, None, self.slot_base, self.size(), min_score, first_slot, max_pairs)


def _brute(ix, min_score):
    """Every pair from the oracle's pairwise cosines, in the contract's order."""
    import oracle
    out = []
    for a in np.flatnonzero(ix.live):
        q = (ix.rows[a].astype(np.uint32) << 16).view(np.float32).astype(np.float64)
        s, v = oracle.search(ix.rows, q, ix.size(), min_score, live=ix.live)
        out += [(ix.slot_base + a, ix.slot_base + int(b), float(x)) for b, x in zip(s, v) if b > a]
    return out


def _pages(ix, min_score, max_pairs):
    got, nxt = [], None
    while True:
        a, b, s, n2 = ix.similar_pairs(min_score, nxt, max_pairs)
        assert nxt is None or n2 > nxt
        got += list(zip(a.tolist(), b.tolist(), s.tolist()))
        nxt = n2
        if nxt >= ix.slot_base + ix.size():
            return got


def test_python_page_loop_against_the_oracle_stand_in(nat):
    rng = np.random.default_rng(4)
    ix = PairsOracleIndex(24)
    rows = rng.standard_normal((90, 24))
    rows[40] = rows[3]
    rows[41:45] = rows[5] + 0.1 * rng.standard_normal((4, 24))
    ix.append_f64(rows)
    ix.set_slot_base(1000)
    ix.tombstone([7, 42])
    for m in (None, 0.2, 0.9):
        want = _brute(ix, m)
        big = ix.similar_pairs(m, None, 90 * 90)
        assert big[3] == 1090 and list(zip(big[0].tolist(), big[1].tolist(), big[2].tolist())) == want
        assert _pages(ix, m, 90) == want            # the smallest buffer
        assert _pages(ix, m, 200) == want
        a, b, s, nxt = ix.similar_pairs(m, 1050, 90 * 90)
        assert list(zip(a.tolist(), b.tolist(), s.tolist())) == [p for p in want if p[0] >= 1050]
    assert ix.similar_pairs(0.5, 1090, 90)[3] == 1090
    with pytest.raises(nat.RbkError):
        ix.similar_pairs(0.5, None, 89)
    with pytest.raises(nat.RbkError):
        ix.similar_pairs(float("nan"))
    with pytest.raises(nat.RbkError):
        ix.similar_pairs(0.5, 999)
    assert hasattr(nat.Index, "similar_pairs") and hasattr(nat.Group, "similar_pairs")


def _store(tmp_path, name, chunks):
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    store = VectorStore(str(tmp_path / f"{name}.db"), index_factory=lambda d, dev: PairsOracleIndex(d))
    store.add_chunks(chunks)
    return store


def _ids_of(store, pairs):
    return [(store._ids[a][4:], store._ids[b][4:], s) for a, b, s in pairs]


def test_vector_store_similar_pairs(tmp_path):
    from runbookai_b200 import embedder
    from runbookai_b200._native import DimensionError
    dup = [{**c, "chunk": {**c["chunk"], "id": c["chunk"]["id"] + "-copy"}} for c in ALL[:10]]
    store = _store(tmp_path, "a", ALL + dup)
    try:
        embedder.reset()     # no embedder needed
        for m in (0.9, 0.3):
            got = store.similar_pairs(m)
            assert got == _ids_of(store, _brute(store._index, m))
        got = store.similar_pairs(0.999)
        assert {(a, b) for a, b, _ in got} >= {(c["chunk"]["id"], c["chunk"]["id"] + "-copy") for c in ALL[:10]}
        store.delete_document("doc2")
        got = store.similar_pairs(0.3)
        assert got and not any(x.startswith("doc2-") for p in got for x in p[:2])
        want = {(a, b, s) for a, b, s in got}
        assert store.compact() == 30
        assert set(store.similar_pairs(0.3)) == want      # the same pairs under the new slots
        with pytest.raises(ValueError):
            store.similar_pairs(float("nan"))
        store._set("vec_odd", np.ones(5))
        with pytest.raises(DimensionError):
            store.similar_pairs(0.5)
    finally:
        store.close()
    empty = _store(tmp_path, "empty", [])
    try:
        assert empty.similar_pairs(0.5) == []
    finally:
        empty.close()


# --------------------------------------------------------------------------- the N-API addon's similarPairs
@pytest.fixture(scope="module")
def shim_pairs_harness(tmp_path_factory, oracle_mod):
    from test_unbounded_host import _shim_harness
    return _shim_harness(tmp_path_factory.mktemp("shim_pairs"), "rbk_shim_pairs")


@pytest.fixture(scope="module")
def shim_without_pairs_harness(tmp_path_factory, oracle_mod):
    from test_unbounded_host import _shim_harness
    return _shim_harness(tmp_path_factory.mktemp("shim_without_pairs"), "rbk_shim_slots")


PAIRS_MIN, PAIRS_PAGE = 0.2, 1500


def check_pair_answers(d, w, oracle_mod, min_score=PAIRS_MIN):
    """The harness's concatenated pages against the oracle: for every live a, its hits at k = n above a."""
    corpus, live = w["corpus"], w["live"]
    n = len(live)
    a = np.fromfile(d / "pairs_a.i64", dtype=np.int64)
    b = np.fromfile(d / "pairs_b.i64", dtype=np.int64)
    s = np.fromfile(d / "pairs_scores.f64", dtype=np.float64)
    ea, eb, ev = [], [], []
    for q in np.flatnonzero(live):
        es, vs = oracle_mod.search(corpus, corpus[q], n, min_score, live=live)
        es, vs = np.asarray(es), np.asarray(vs)
        keep = es > q
        ea.append(np.full(int(keep.sum()), q, np.int64))
        eb.append(es[keep])
        ev.append(vs[keep])
    ea, eb, ev = np.concatenate(ea), np.concatenate(eb), np.concatenate(ev)
    assert len(a) == len(ea) and (a == ea).all() and (b == eb).all()
    assert s.tobytes() == ev.tobytes()
    assert int((d / "pairs_pages.txt").read_text()) > 1
    log = dict(line.split(" ", 1) for line in (d / "log.txt").read_text().strip().splitlines())
    assert log["err_pairs"].startswith("max_pairs must be >=")


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_similar_pairs_against_the_oracle_backed_stand_in(tmp_path, oracle_mod, shim_pairs_harness, devices):
    """similarPairs under the mock N-API runtime, as async work on one device and on a device list: the pages from
    slot 0 on, concatenated, are the oracle's pairs; a maxPairs of 0 rejects with the library's message."""
    from test_napi_addon import _write_inputs
    w = _write_inputs(tmp_path, devices, n=1200)
    (tmp_path / "pairs.txt").write_text(f"{PAIRS_MIN} {PAIRS_PAGE}\n")
    r = subprocess.run([str(shim_pairs_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "has_similar_pairs.txt").read_text() == "1"
    check_pair_answers(tmp_path, w, oracle_mod)


def test_addon_similar_pairs_throws_against_a_library_without_it(tmp_path, oracle_mod, shim_without_pairs_harness):
    """A library without similar pairs still loads the addon: hasSimilarPairs is false and similarPairs throws, after
    every method before it ran."""
    from test_napi_addon import _write_inputs
    _write_inputs(tmp_path, [], n=1200)
    (tmp_path / "pairs.txt").write_text(f"{PAIRS_MIN} {PAIRS_PAGE}\n")
    r = subprocess.run([str(shim_without_pairs_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr
    assert (tmp_path / "has_similar_pairs.txt").read_text() == "0"
    err = (tmp_path / "error.txt").read_text()
    assert "similarPairs rejected" in err and "no similar pairs" in err
    assert (tmp_path / "slots.i64").exists()     # search() before it ran against the same handle
