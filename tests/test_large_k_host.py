"""Large-k search (k_fetch up to 4096) without a GPU: the host mirror's routing between the three search paths, and
the N-API addon's searchLarge against the oracle-backed stand-in of the C ABI (tests/napi_shim/rbk_shim_large.cc), and
the addon against a library without the large-k entry points."""
import importlib.util
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from test_napi_addon import _build_shim, _write_inputs


@pytest.fixture(scope="module")
def shim_large_harness(tmp_path_factory, oracle_mod):
    """The addon harness linked against rbk_shim_large.cc (built in a temporary directory)."""
    spec = importlib.util.spec_from_file_location("rbk_napi_mock_build", ROOT / "napi" / "mock" / "build.py")
    mb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mb)
    objs = mb.build_objects()
    olib = ROOT / "oracle" / "librbk_oracle.so"
    out = tmp_path_factory.mktemp("shim_large")
    shim = out / "librbk_knn_shim_large.so"
    mb.run(mb.CXX + ["-fPIC", "-shared", ROOT / "tests" / "napi_shim" / "rbk_shim_large.cc", "-o", shim,
                     "-L", olib.parent, "-l:librbk_oracle.so", f"-Wl,-rpath,{olib.parent}"])
    exe = out / "harness_shim_large"
    mb.run(["g++"] + objs + ["-o", exe, "-L", out, "-l:librbk_knn_shim_large.so", f"-Wl,-rpath,{out}",
                             f"-Wl,-rpath,{olib.parent}", "-L", olib.parent, "-l:librbk_oracle.so", "-lpthread"])
    return exe


class _Recorder:
    """Stand-in index that records which path _search_any_k takes."""

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

    def exact_scores(self, q):
        self.calls.append(("exact_scores", None))
        return np.full((len(q), 5), 0.25)


def test_search_any_k_routes_by_k_fetch(native):
    from runbookai_b200 import _native
    assert _native.RBK_MAX_K_FETCH == 112 and _native.RBK_MAX_K_FETCH_LARGE == 4096
    q = np.zeros((2, 8))
    for k, path in ((1, "search"), (112, "search"), (113, "search_large"), (1000, "search_large"),
                    (4096, "search_large"), (4097, "exact_scores"), (5000, "exact_scores")):
        ix = _Recorder()
        slots, scores, counts, _ = _native._search_any_k(ix, q, k, 0.1)
        assert [c[0] for c in ix.calls] == [path], (k, ix.calls)
        assert slots.shape == (2, k)
        if path == "exact_scores":
            assert (counts == 5).all() and (slots[:, :5] == np.arange(5)).all()


def test_large_k_symbols_are_declared(native):
    from runbookai_b200 import _native
    assert "rbk_index_search_large_f64" in _native.SYMBOLS and "rbk_group_search_large_f64" in _native.SYMBOLS
    assert _native.lib.rbk_abi_version() == 2


def check_large_outputs(d, w, oracle_mod, ks):
    nq = w["nq"]
    for i, k in enumerate(ks):
        slots = np.fromfile(d / f"large{i}_slots.i64", dtype=np.int64).reshape(nq, k)
        scores = np.fromfile(d / f"large{i}_scores.f64", dtype=np.float64).reshape(nq, k)
        counts = np.fromfile(d / f"large{i}_counts.i32", dtype=np.int32)
        for b in range(nq):
            es, ev = oracle_mod.search(w["corpus"], w["q"][b], k, w["min_score"], live=w["live"])
            assert counts[b] == len(es) and (slots[b, :len(es)] == es).all(), (k, b)
            assert scores[b, :len(es)].tobytes() == ev.tobytes()
            assert (slots[b, len(es):] == -1).all() and np.isnan(scores[b, len(es):]).all()
    log = dict(line.split(" ", 1) for line in (d / "log.txt").read_text().strip().splitlines())
    assert log["err_large"] == "k_fetch must be in [1, 4096]"


@pytest.mark.parametrize("devices", [[], [0]], ids=["index", "group"])
def test_addon_search_large_against_the_oracle_backed_stand_in(tmp_path, oracle_mod, shim_large_harness, devices):
    exe = shim_large_harness
    w = _write_inputs(tmp_path, devices, n=1500, min_score=-1.0)
    ks = [300, 4000]                     # 4000 > the 1300-odd live rows: every live row, then -1 / NaN
    (tmp_path / "large.txt").write_text(" ".join(map(str, ks)) + "\n")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    check_large_outputs(tmp_path, w, oracle_mod, ks)


def test_addon_search_large_throws_against_a_library_without_it(tmp_path, oracle_mod):
    """An ABI-2 library built before the large-k search (here: the stand-in without it) still loads the addon and runs
    every other method; searchLarge throws instead of the module failing to load."""
    exe = _build_shim()
    _write_inputs(tmp_path, [])
    (tmp_path / "large.txt").write_text("300\n")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr          # the harness stops at the rejected searchLarge
    err = (tmp_path / "error.txt").read_text()
    assert "searchLarge rejected" in err and "no large-k search" in err
    assert (tmp_path / "slots.i64").exists()     # search() before it ran against the same handle
