"""Unbounded search (any k_fetch) without a GPU: the host mirror's routing of k_fetch > 4096 to the device search, the
N-API addon's searchUnbounded against the oracle-backed stand-in of the C ABI (tests/napi_shim/rbk_shim_unbounded.cc),
and the addon against a library without the unbounded entry points."""
import importlib.util
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from test_napi_addon import _write_inputs


def _shim_harness(out, source):
    """The addon harness linked against one oracle-backed stand-in of the C ABI (built in `out`)."""
    spec = importlib.util.spec_from_file_location("rbk_napi_mock_build", ROOT / "napi" / "mock" / "build.py")
    mb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mb)
    objs = mb.build_objects()
    olib = ROOT / "oracle" / "librbk_oracle.so"
    shim = out / f"lib{source}.so"
    mb.run(mb.CXX + ["-fPIC", "-shared", ROOT / "tests" / "napi_shim" / f"{source}.cc", "-o", shim,
                     "-L", olib.parent, "-l:librbk_oracle.so", f"-Wl,-rpath,{olib.parent}"])
    exe = out / f"harness_{source}"
    mb.run(["g++"] + objs + ["-o", exe, "-L", out, f"-l:lib{source}.so", f"-Wl,-rpath,{out}",
                             f"-Wl,-rpath,{olib.parent}", "-L", olib.parent, "-l:librbk_oracle.so", "-lpthread"])
    return exe


@pytest.fixture(scope="module")
def shim_unbounded_harness(tmp_path_factory, oracle_mod):
    return _shim_harness(tmp_path_factory.mktemp("shim_unbounded"), "rbk_shim_unbounded")


@pytest.fixture(scope="module")
def shim_large_only_harness(tmp_path_factory, oracle_mod):
    return _shim_harness(tmp_path_factory.mktemp("shim_large_only"), "rbk_shim_large")


class _Recorder:
    """Stand-in index that records which search the mirror's search_any_k calls."""

    def __init__(self):
        self.calls = []

    def _result(self, B, k):
        return (np.full((B, k), -1, np.int64), np.full((B, k), np.nan), np.zeros(B, np.int32), 0.0)

    def search(self, q, k, ms):
        self.calls.append(("search", k))
        return self._result(len(q), k)

    def search_large(self, q, k, ms):
        self.calls.append(("search_large", k))
        return self._result(len(q), k)

    def search_unbounded(self, q, k, ms):
        self.calls.append(("search_unbounded", k))
        return self._result(len(q), k)

    def exact_scores(self, q):
        raise AssertionError("search_any_k must not copy every row's score to the host")


@pytest.mark.parametrize("cls", ["Index", "Group"])
def test_search_any_k_routes_large_k_to_the_unbounded_search(native, cls):
    from runbookai_b200 import _native
    method = getattr(_native, cls).search_any_k
    q = np.zeros((2, 8))
    for k, path in ((1, "search"), (112, "search"), (113, "search_large"), (4096, "search_large"),
                    (4097, "search_unbounded"), (250_000, "search_unbounded")):
        ix = _Recorder()
        slots, scores, counts, _ = method(ix, q, k, 0.1)
        assert [c[0] for c in ix.calls] == [path], (cls, k, ix.calls)
        assert slots.shape == (2, k)


def test_unbounded_symbols_are_declared(native):
    from runbookai_b200 import _native
    for name in ("rbk_index_search_unbounded_f64", "rbk_group_search_unbounded_f64"):
        assert name in _native.SYMBOLS
        assert hasattr(_native.lib, name)
    assert _native.lib.rbk_abi_version() == 2


def check_unbounded_outputs(d, w, oracle_mod, ks):
    nq = w["nq"]
    for i, k in enumerate(ks):
        slots = np.fromfile(d / f"unbounded{i}_slots.i64", dtype=np.int64).reshape(nq, k)
        scores = np.fromfile(d / f"unbounded{i}_scores.f64", dtype=np.float64).reshape(nq, k)
        counts = np.fromfile(d / f"unbounded{i}_counts.i32", dtype=np.int32)
        for b in range(nq):
            es, ev = oracle_mod.search(w["corpus"], w["q"][b], k, w["min_score"], live=w["live"])
            assert counts[b] == len(es) and (slots[b, :len(es)] == es).all(), (k, b)
            assert scores[b, :len(es)].tobytes() == ev.tobytes()
            assert (slots[b, len(es):] == -1).all() and np.isnan(scores[b, len(es):]).all()
    log = dict(line.split(" ", 1) for line in (d / "log.txt").read_text().strip().splitlines())
    assert log["err_unbounded"].startswith("k_fetch must be in [1, ")


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_unbounded_against_the_oracle_backed_stand_in(tmp_path, oracle_mod, shim_unbounded_harness,
                                                                   devices):
    w = _write_inputs(tmp_path, devices, n=6000, min_score=-1.0)
    live = int(w["live"].sum())
    ks = [5000, 9000]                    # above 4096; 9000 > the live rows: every live row, then -1 / NaN
    assert ks[0] < live < ks[1]
    (tmp_path / "unbounded.txt").write_text(" ".join(map(str, ks)) + "\n")
    r = subprocess.run([str(shim_unbounded_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    check_unbounded_outputs(tmp_path, w, oracle_mod, ks)


def test_addon_search_unbounded_throws_against_a_library_without_it(tmp_path, oracle_mod, shim_large_only_harness):
    """A library with the large-k search but without the unbounded one still loads the addon; searchUnbounded throws
    instead of the module failing to load, and the methods before it ran."""
    _write_inputs(tmp_path, [])
    (tmp_path / "unbounded.txt").write_text("5000\n")
    r = subprocess.run([str(shim_large_only_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr          # the harness stops at the rejected searchUnbounded
    err = (tmp_path / "error.txt").read_text()
    assert "searchUnbounded rejected" in err and "no unbounded search" in err
    assert (tmp_path / "slots.i64").exists()     # search() before it ran against the same handle
