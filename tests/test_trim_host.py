"""Giving memory back (rbk_index_trim / rbk_group_trim) without a GPU: the declared and exported symbols,
`VectorStore.trim()` and the trim that `KnowledgeRetriever` runs after a compaction over a recording CPU stand-in index,
the N-API addon's trim() against a stand-in library that has it (tests/napi_shim/rbk_shim_trim.cc), and the addon
against a library without it."""
import importlib.util
import subprocess

import numpy as np
import pytest

from common import OracleIndex
from conftest import ROOT
from test_compact_host import QUERIES, WORDS, CompactOracleIndex, _answers, _chunks, _docs, hash_embedder  # noqa: F401
from test_napi_addon import _build_shim, _write_inputs


class TrimOracleIndex(CompactOracleIndex):
    """CompactOracleIndex that records every trim() and what the index held at the time."""

    def trim(self):
        self.trims = getattr(self, "trims", []) + [(self.size(), self.count())]


def test_trim_symbols_are_declared_and_exported(native):
    header = (ROOT / "include" / "rbk_knn.h").read_text()
    for name, decl in (("rbk_index_trim", "rbk_status rbk_index_trim(rbk_index* idx);"),
                       ("rbk_group_trim", "rbk_status rbk_group_trim(rbk_group* grp);")):
        assert name in native.SYMBOLS and decl in header
        assert getattr(native.lib, name) is not None          # ctypes raises AttributeError for a missing export
    out = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True).stdout
    assert " T rbk_index_trim\n" in out and " T rbk_group_trim\n" in out


def test_vector_store_trim_calls_the_index_and_keeps_every_answer(tmp_path, hash_embedder):  # noqa: F811
    from runbookai_b200.vector_store import VectorStore
    vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: TrimOracleIndex(d))
    for j in range(6):
        vs.add_chunks(_chunks(f"d{j}", 10, WORDS))
    vs.delete_document("d1")
    vs.compact()
    before = _answers(vs)
    vs.trim()
    assert vs._index.trims == [(50, 50)] and _answers(vs) == before
    vs.clear()
    vs.trim()
    assert vs._index.trims[-1] == (0, 0)
    vs.close()


def test_vector_store_trim_skips_an_index_without_trim(tmp_path, hash_embedder):  # noqa: F811
    from runbookai_b200.vector_store import VectorStore
    vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: OracleIndex(d))
    vs.add_chunks(_chunks("d0", 6, WORDS))
    vs.trim()
    assert vs._index.size() == 6
    vs.close()


def test_reclaim_trims_right_after_each_compaction(tmp_path, hash_embedder, monkeypatch):  # noqa: F811
    from runbookai_b200 import retriever
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    monkeypatch.setattr(retriever, "_COMPACT_MIN_DEAD", 64)
    rnd = [0]
    vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: TrimOracleIndex(d))
    r = KnowledgeRetriever({"storePath": str(tmp_path / "knowledge.db"), "sources": [lambda since: _docs(rnd[0])]},
                           vector_store=vs)
    ref = VectorStore(str(tmp_path / "ref.db"), index_factory=lambda d, dev: OracleIndex(d))
    rr = KnowledgeRetriever({"storePath": str(tmp_path / "ref_knowledge.db"), "sources": [lambda since: _docs(rnd[0])]},
                            vector_store=ref)
    for rnd[0] in range(8):
        r.sync()
        rr.sync()
        assert _answers(vs) == _answers(ref)
    ix = vs._index
    assert ix.compactions >= 3 and len(ix.trims) == ix.compactions
    assert all(size == count for size, count in ix.trims)      # each trim saw a freshly compacted index
    r.close()
    rr.close()


def test_reclaim_skips_trim_for_an_index_without_it(tmp_path, hash_embedder, monkeypatch):  # noqa: F811
    from runbookai_b200 import retriever
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    monkeypatch.setattr(retriever, "_COMPACT_MIN_DEAD", 64)
    rnd = [0]
    vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: CompactOracleIndex(d))
    r = KnowledgeRetriever({"storePath": str(tmp_path / "knowledge.db"), "sources": [lambda since: _docs(rnd[0])]},
                           vector_store=vs)
    for rnd[0] in range(6):
        r.sync()
    assert vs._index.compactions >= 2
    r.close()


@pytest.fixture(scope="module")
def shim_trim_harness(tmp_path_factory, oracle_mod):
    """The addon harness linked against rbk_shim_trim.cc (built in a temporary directory)."""
    spec = importlib.util.spec_from_file_location("rbk_napi_mock_build", ROOT / "napi" / "mock" / "build.py")
    mb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mb)
    objs = mb.build_objects()
    olib = ROOT / "oracle" / "librbk_oracle.so"
    out = tmp_path_factory.mktemp("shim_trim")
    shim = out / "librbk_knn_shim_trim.so"
    mb.run(mb.CXX + ["-fPIC", "-shared", ROOT / "tests" / "napi_shim" / "rbk_shim_trim.cc", "-o", shim,
                     "-L", olib.parent, "-l:librbk_oracle.so", f"-Wl,-rpath,{olib.parent}"])
    exe = out / "harness_shim_trim"
    mb.run(["g++"] + objs + ["-o", exe, "-L", out, "-l:librbk_knn_shim_trim.so", f"-Wl,-rpath,{out}",
                             f"-Wl,-rpath,{olib.parent}", "-L", olib.parent, "-l:librbk_oracle.so", "-lpthread"])
    return exe


def check_trim_outputs(d, w, oracle_mod):
    """trim_* must be the oracle's answer over the rows the scenario left live, bit for bit."""
    nq, k = w["nq"], w["k"]
    log = dict(line.split(" ", 1) for line in (d / "log.txt").read_text().strip().splitlines())
    assert log["trim_identical"] == "1" and log["finalized"] == "1"
    slots = np.fromfile(d / "trim_slots.i64", dtype=np.int64).reshape(nq, k)
    scores = np.fromfile(d / "trim_scores.f64", dtype=np.float64).reshape(nq, k)
    counts = np.fromfile(d / "trim_counts.i32", dtype=np.int32)
    for b in range(nq):
        es, ev = oracle_mod.search(w["corpus"], w["q"][b], k, w["min_score"], live=w["live"])
        assert counts[b] == len(es) and (slots[b, :len(es)] == es).all(), b
        assert scores[b, :len(es)].tobytes() == ev.tobytes(), b


@pytest.mark.parametrize("devices,entry", [([], "rbk_index_trim"), ([0], "rbk_group_trim")])
def test_addon_trim_against_the_stand_in(tmp_path, oracle_mod, shim_trim_harness, devices, entry):
    w = _write_inputs(tmp_path, devices)
    (tmp_path / "trim.txt").write_text("1\n")
    r = subprocess.run([str(shim_trim_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stderr.count(f"rbk_shim: {entry}\n") == 1 and r.stderr.count("rbk_shim: rbk_") == 1
    check_trim_outputs(tmp_path, w, oracle_mod)


def test_addon_trim_throws_against_a_library_without_it(tmp_path, oracle_mod):
    """An ABI-2 library built before trim (here: the stand-in without it) still loads the addon and runs every other
    method; trim() throws instead of the module failing to load."""
    exe = _build_shim()
    _write_inputs(tmp_path, [])
    (tmp_path / "trim.txt").write_text("1\n")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr          # the harness stops at the trim() that threw
    err = (tmp_path / "error.txt").read_text()
    assert "trim threw" in err and "no trim" in err
    assert (tmp_path / "slots.i64").exists()     # search() before it ran against the same handle
