"""Compaction (rbk_index_compact) without a GPU: the declared symbol, `VectorStore.compact()` and the compaction that
`KnowledgeRetriever.sync()` triggers over a CPU stand-in index with `compact`, the N-API addon's compact() against the
oracle-backed stand-in of the C ABI (tests/napi_shim/rbk_shim_compact.cc), and the addon against a library without
compaction."""
import importlib.util
import subprocess

import numpy as np
import pytest

from common import HashEmbedder, OracleIndex
from conftest import ROOT
from test_napi_addon import _build_shim, _write_inputs


class CompactOracleIndex(OracleIndex):
    """OracleIndex plus rbk_index_compact's contract: live rows keep their order and move to slots 0 .. count()-1."""

    def compact(self):
        live = self.live.astype(bool)
        old_to_new = np.where(live, np.cumsum(live) - 1, -1).astype(np.int64)
        self.rows = self.rows[live]
        self.live = np.ones(self.rows.shape[0], dtype=np.uint8)
        self.compactions = getattr(self, "compactions", 0) + 1
        return old_to_new


def test_compact_symbol_is_declared(native):
    assert "rbk_index_compact" in native.SYMBOLS
    header = (ROOT / "include" / "rbk_knn.h").read_text()
    assert "rbk_status rbk_index_compact(rbk_index* idx, int64_t* old_to_new, int64_t old_to_new_len);" in header


def _chunks(doc, n, words):
    return [{"chunk": {"id": f"{doc}_{i}", "documentId": doc, "content": " ".join(words[i % len(words):][:4]) + f" {i}",
                       "sectionTitle": "S"}, "documentTitle": doc.upper(), "type": "runbook", "services": ["api"]}
            for i in range(n)]


WORDS = ["redis", "pool", "exhausted", "postgres", "replication", "lag", "failover", "kubernetes", "pod", "crashloop",
         "oom", "latency", "gateway", "tls", "certificate"]
QUERIES = ["redis pool exhausted", "postgres failover lag", "kubernetes pod oom", "gateway tls latency"]


@pytest.fixture
def hash_embedder():
    from runbookai_b200 import embedder
    embedder.configure(HashEmbedder(64))
    yield
    embedder.reset()


def _answers(vs, top_k=8):
    return [[(c.id, c.score, c.documentId) for c in vs.search(q, {"topK": top_k, "minScore": 0.1})] for q in QUERIES]


def test_vector_store_compact_keeps_every_answer(tmp_path, hash_embedder):
    from runbookai_b200.vector_store import VectorStore
    vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: CompactOracleIndex(d))
    for j in range(12):
        vs.add_chunks(_chunks(f"d{j}", 5 + j, WORDS[j:] + WORDS[:j]))
    for j in (0, 3, 4, 7, 11):
        vs.delete_document(f"d{j}")
    ix = vs._index
    before = _answers(vs) + [_answers(vs, 60)]
    live_ids = [i for i in vs._ids if i is not None]
    size, count = ix.size(), ix.count()
    assert size > count
    assert vs.compact() == size - count
    assert ix.size() == ix.count() == count and len(vs._ids) == count
    assert vs._ids == live_ids                                   # Map order survives
    assert all(vs._slot_of[v] == s for s, v in enumerate(vs._ids))
    assert _answers(vs) + [_answers(vs, 60)] == before
    assert vs.compact() == 0                                     # nothing left to reclaim
    # appends land behind the survivors, deletes and a second compaction work as before
    vs.add_chunks(_chunks("d99", 3, WORDS))
    assert vs._slot_of["vec_d99_0"] == count
    vs.delete_document("d1")
    assert vs.compact() == 6 and None not in vs._ids and ix.size() == ix.count()
    vs.close()


def test_vector_store_compact_skips_an_index_without_compact(tmp_path, hash_embedder):
    from runbookai_b200.vector_store import VectorStore
    vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: OracleIndex(d))
    vs.add_chunks(_chunks("d0", 6, WORDS))
    vs.delete_document("d0")
    assert vs.compact() == 0 and vs._index.size() == 6
    vs.close()


def _docs(round_, n_docs=40):
    """Every document comes back each round; a third of them with changed text (and so new chunk vectors)."""
    return [{"id": f"doc{j}", "type": "runbook", "title": f"DOC{j}", "services": ["api"],
             "chunks": [{"id": f"doc{j}_{i}", "sectionTitle": "S",
                         "content": " ".join(WORDS[(i + j + (round_ if j % 3 == 0 else 0)) % len(WORDS):][:5])}
                        for i in range(8 + j % 5)]} for j in range(n_docs)]


def test_sync_compacts_and_bounds_the_index_through_churn(tmp_path, hash_embedder, monkeypatch):
    from runbookai_b200 import retriever
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    monkeypatch.setattr(retriever, "_COMPACT_MIN_DEAD", 64)      # a small store stands in for a large one
    rnd = [0]
    vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: CompactOracleIndex(d))
    r = KnowledgeRetriever({"storePath": str(tmp_path / "knowledge.db"), "sources": [lambda since: _docs(rnd[0])]},
                           vector_store=vs)
    # the same documents in a store that never compacts: every answer must agree
    ref = VectorStore(str(tmp_path / "ref.db"), index_factory=lambda d, dev: OracleIndex(d))
    rr = KnowledgeRetriever({"storePath": str(tmp_path / "ref_knowledge.db"), "sources": [lambda since: _docs(rnd[0])]},
                            vector_store=ref)
    sizes = []
    for rnd[0] in range(10):
        r.sync()
        rr.sync()
        ix = vs._index
        dead = ix.size() - ix.count()
        assert dead < max(64, ix.size() / 4)                     # sync() left no more dead slots than its threshold
        assert ix.count() == ref._index.count()
        sizes.append(ix.size())
        assert _answers(vs) == _answers(ref)
    live = ref._index.count()
    assert max(sizes) < 2 * live and ref._index.size() > 5 * live   # bounded here, growing without compaction
    assert vs._index.compactions >= 3
    vs.compact()
    assert None not in vs._ids and _answers(vs, 40) == _answers(ref, 40)
    r.close()
    rr.close()


def test_sync_leaves_small_stores_alone(tmp_path, hash_embedder):
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    rnd = [0]
    vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: CompactOracleIndex(d))
    r = KnowledgeRetriever({"storePath": str(tmp_path / "knowledge.db"), "sources": [lambda since: _docs(rnd[0])]},
                           vector_store=vs)
    for rnd[0] in range(3):
        r.sync()
    assert getattr(vs._index, "compactions", 0) == 0 and vs._index.size() > 2 * vs._index.count()
    r.close()


@pytest.fixture(scope="module")
def shim_compact_harness(tmp_path_factory, oracle_mod):
    """The addon harness linked against rbk_shim_compact.cc (built in a temporary directory)."""
    spec = importlib.util.spec_from_file_location("rbk_napi_mock_build", ROOT / "napi" / "mock" / "build.py")
    mb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mb)
    objs = mb.build_objects()
    olib = ROOT / "oracle" / "librbk_oracle.so"
    out = tmp_path_factory.mktemp("shim_compact")
    shim = out / "librbk_knn_shim_compact.so"
    mb.run(mb.CXX + ["-fPIC", "-shared", ROOT / "tests" / "napi_shim" / "rbk_shim_compact.cc", "-o", shim,
                     "-L", olib.parent, "-l:librbk_oracle.so", f"-Wl,-rpath,{olib.parent}"])
    exe = out / "harness_shim_compact"
    mb.run(["g++"] + objs + ["-o", exe, "-L", out, "-l:librbk_knn_shim_compact.so", f"-Wl,-rpath,{out}",
                             f"-Wl,-rpath,{olib.parent}", "-L", olib.parent, "-l:librbk_oracle.so", "-lpthread"])
    return exe


def write_compact_input(d, w, seed=3):
    """compact.txt: more slots to tombstone before compact() - whole runs of slots, like a deleted document."""
    rng = np.random.default_rng(seed)
    n = w["n"]
    more = np.concatenate([np.arange(s, min(n, s + rng.integers(8, 41))) for s in rng.choice(n, 12, replace=False)])
    more = np.unique(np.concatenate([more, [0, n - 1]]))
    (d / "compact.txt").write_text(" ".join(map(str, more)) + "\n")
    live = w["live"].copy()
    live[more] = 0
    return live


def check_compact_outputs(d, w, oracle_mod, live):
    n, nq, k = w["n"], w["nq"], w["k"]
    keep = live.astype(bool)
    old_to_new = np.fromfile(d / "compact_map.i64", dtype=np.int64)
    assert (old_to_new == np.where(keep, np.cumsum(keep) - 1, -1)).all()
    log = dict(line.split(" ", 1) for line in (d / "log.txt").read_text().strip().splitlines())
    assert float(log["count_after_compact"]) == keep.sum()
    slots = np.fromfile(d / "compact_slots.i64", dtype=np.int64).reshape(nq, k)
    scores = np.fromfile(d / "compact_scores.f64", dtype=np.float64).reshape(nq, k)
    counts = np.fromfile(d / "compact_counts.i32", dtype=np.int32)
    survivors = w["corpus"][keep]
    for b in range(nq):
        es, ev = oracle_mod.search(survivors, w["q"][b], k, w["min_score"])
        assert counts[b] == len(es) and (slots[b, :len(es)] == es).all(), b
        assert scores[b, :len(es)].tobytes() == ev.tobytes()
        old, ov = oracle_mod.search(w["corpus"], w["q"][b], k, w["min_score"], live=live)   # the same answer, renumbered
        assert (old_to_new[old] == es).all() and ov.tobytes() == ev.tobytes()
    assert float(log["count_after_clear"]) == 0 and log["finalized"] == "1"


def test_addon_compact_against_the_oracle_backed_stand_in(tmp_path, oracle_mod, shim_compact_harness):
    w = _write_inputs(tmp_path, [])
    live = write_compact_input(tmp_path, w)
    r = subprocess.run([str(shim_compact_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    check_compact_outputs(tmp_path, w, oracle_mod, live)


def test_addon_compact_throws_for_a_device_group(tmp_path, oracle_mod, shim_compact_harness):
    w = _write_inputs(tmp_path, [0])
    write_compact_input(tmp_path, w)
    r = subprocess.run([str(shim_compact_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    log = dict(line.split(" ", 1) for line in (tmp_path / "log.txt").read_text().strip().splitlines())
    assert log["err_compact"] == "compaction is not available for a device group"
    assert not (tmp_path / "compact_map.i64").exists()


def test_addon_compact_throws_against_a_library_without_it(tmp_path, oracle_mod):
    """An ABI-2 library built before compaction (here: the stand-in without it) still loads the addon and runs every
    other method; compact() throws instead of the module failing to load."""
    exe = _build_shim()
    w = _write_inputs(tmp_path, [])
    write_compact_input(tmp_path, w)
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr          # the harness stops at the compact() that threw
    err = (tmp_path / "error.txt").read_text()
    assert "compact threw" in err and "no compaction" in err
    assert (tmp_path / "slots.i64").exists()     # search() before it ran against the same handle
