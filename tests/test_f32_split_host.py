"""CPU suite for split float32 exact rows (RBK_INDEX_KEEP_F32_SPLIT): the header, docs and binding agree, the flag
rules refuse what they must, the Python helpers and the vector store handle the new width, the N-API addon takes
exactRows 'f32_split' and widens it, the split rule restores every float32 (numpy and the library's own header agree),
and the new kernel instantiations spill no more than their float32 twins."""
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from test_f32_rows_host import ADDON_STUB, Float32Stub, _drive, _ptxas

ROOT = Path(__file__).resolve().parents[1]
HEADER = ROOT / "include" / "rbk_knn.h"
CSRC = ROOT / "runbookai_b200" / "csrc"
NVCC = "/usr/local/cuda/bin/nvcc"
SPLIT, KEEP64, KEEP32, HOST, F16 = 128, 1, 64, 2, 16


def test_header_and_docs():
    from runbookai_b200 import _native as n
    h = HEADER.read_text()
    assert re.search(r"#define RBK_INDEX_KEEP_F32_SPLIT 128u", h)
    assert n.RBK_INDEX_KEEP_F32_SPLIT == SPLIT
    for doc in ("README.md", "DESIGN.md", "INTEGRATION.md"):
        assert "f32_split" in (ROOT / doc).read_text() or "KEEP_F32_SPLIT" in (ROOT / doc).read_text(), doc
    assert "'f32_split'" in (ROOT / "ts" / "gpu-embedding-index.ts").read_text()


def test_flag_refusals_without_a_device():
    """check_flags runs before the device is looked at: refused sets are RBK_EINVAL even here."""
    import ctypes as C
    from runbookai_b200._native import RBK_EINVAL, lib
    refused = [SPLIT | KEEP64, SPLIT | KEEP32, SPLIT | KEEP64 | KEEP32, SPLIT | F16, SPLIT | F16 | HOST,
               SPLIT | KEEP32 | HOST, SPLIT | 4, SPLIT | 8, SPLIT | 32, 4, 8, 32, 256]
    for flags in refused:
        h = C.c_void_p()
        assert lib.rbk_index_create_ex(16, 0, 0, flags, C.byref(h)) == RBK_EINVAL, flags
        assert lib.rbk_group_create(16, (C.c_int32 * 1)(0), 1, 0, flags, C.byref(h)) == RBK_EINVAL, flags
    for flags in (SPLIT, SPLIT | HOST):
        h = C.c_void_p()
        assert lib.rbk_index_create_ex(16, 0, 0, flags, C.byref(h)) != RBK_EINVAL, flags
        lib.rbk_index_destroy(h)


def test_flag_helpers():
    from runbookai_b200._native import _index_flags, _tier_flags, exact_rows_of
    assert _index_flags(False, False, keep_f32_split=True) == SPLIT
    assert _index_flags(False, True, keep_f32_split=True) == SPLIT | HOST
    assert _index_flags(False, False, True, False, True) == SPLIT | F16          # passed through: the library refuses
    assert _tier_flags(KEEP64 | HOST, None, None, "f32_split") == SPLIT | HOST
    assert _tier_flags(KEEP32 | F16, None, False, "f32_split") == SPLIT
    assert _tier_flags(SPLIT | HOST, False, None, "f64") == KEEP64              # the widen clears the split bit
    assert _tier_flags(SPLIT, None, True, "f32") == KEEP32 | F16
    assert _tier_flags(SPLIT, None, None, None) == SPLIT
    with pytest.raises(ValueError):
        _tier_flags(SPLIT, None, None, "split")
    assert (exact_rows_of(SPLIT), exact_rows_of(SPLIT | HOST), exact_rows_of(KEEP32)) == ("f32_split", "f32_split", "f32")


class SplitStub(Float32Stub):
    """A keep_f32_split stand-in: refuses non-float32 values until set_tier(exact_rows='f64')."""

    def __init__(self, dim, device=0, capacity_hint=0):
        super().__init__(dim, device, capacity_hint)
        self.flags = SPLIT

    def _guard(self, rows):
        if self.flags & SPLIT:
            self.flags |= KEEP32       # the parent refuses while the float32 bit is set
            try:
                super()._guard(rows)
            finally:
                self.flags &= ~KEEP32
        else:
            super()._guard(rows)


def test_vector_store_widens_a_split_index(monkeypatch):
    from runbookai_b200.vector_store import VectorStore
    made = []

    def factory(dim, dev):
        made.append(SplitStub(dim))
        return made[-1]

    vs = VectorStore(":memory:", index_factory=factory, exact_rows="f32_split")
    try:
        assert vs.exact_rows == "f32_split"
        e = np.float32(np.random.default_rng(1).standard_normal(8)).astype(np.float64)
        vs._set("vec_a", e)
        assert made[0].flags == SPLIT and vs.exact_rows == "f32_split"
        odd = e.copy()
        odd[2] = 0.1
        vs._set("vec_b", odd)                                    # an append the split index refuses
        assert made[0].widened == 1 and made[0].flags == KEEP64 and vs.exact_rows == "f64"
        assert vs._index.size() == 2
    finally:
        vs.close()
    monkeypatch.setenv("RUNBOOK_KNN_EXACT_ROWS", "f32_split")
    vs = VectorStore(":memory:", index_factory=factory)
    try:
        assert vs.exact_rows == "f32_split"
    finally:
        vs.close()


def test_vector_store_asks_for_a_split_index(tmp_path, monkeypatch):
    """The default factory passes keep_f32_split=True, and retrievers pass exact_rows through."""
    from runbookai_b200 import vector_store
    seen = []

    class Recorder(SplitStub):
        def __init__(self, dim, device=0, capacity_hint=0, **kw):
            seen.append(kw)
            super().__init__(dim, device, capacity_hint)

    monkeypatch.setattr(vector_store, "Index", Recorder)
    for var in ("RUNBOOK_KNN_F64_ON_HOST", "RUNBOOK_KNN_SCAN_F16"):
        monkeypatch.delenv(var, raising=False)
    vs = vector_store.create_vector_store(str(tmp_path), shared=False, exact_rows="f32_split")
    try:
        vs._set("vec_a", np.ones(8))
        assert seen == [{"keep_f32_split": True, "f64_on_host": False, "scan_f16": False}]
    finally:
        vs.close()


# --------------------------------------------------------------------------- the N-API addon's exactRows 'f32_split'
SPLIT_STUB = ADDON_STUB.replace("if (!(g_flags & RBK_INDEX_KEEP_F32)) return true;",
                                "if (!(g_flags & (RBK_INDEX_KEEP_F32 | RBK_INDEX_KEEP_F32_SPLIT))) return true;")

SPLIT_DRIVER = r'''
#include <cstdio>
#include <string>
#include "mock_napi.h"
static napi_value str(napi_env env, const char* s) {
  napi_value v;
  napi_create_string_utf8(env, s, NAPI_AUTO_LENGTH, &v);
  return v;
}
int main(int argc, char** argv) {
  napi_env env = mock::new_env();
  napi_value exports;
  napi_create_object(env, &exports);
  rbk_mock_module_init(env, exports);
  napi_value cls = mock::get_property(env, exports, "RbkIndex"), ix, r, t;
  std::string err;
  std::vector<napi_value> args = {mock::number(env, 4), mock::number(env, 0), mock::number(env, 0), mock::number(env, 0),
                                  mock::number(env, 0)};
  if (argc > 1) args.push_back(str(env, argv[1]));
  if (!mock::construct(env, cls, args, &ix, &err)) { fprintf(stderr, "construct threw: %s\n", err.c_str()); return 0; }
  auto tier = [&]() {
    mock::get_accessor(env, ix, "tier", &t, &err);
    napi_value e = mock::get_property(env, t, "exactRows");
    char buf[16] = {0};
    size_t n = 0;
    napi_get_value_string_utf8(env, e, buf, sizeof buf, &n);
    fprintf(stderr, "tier %s\n", buf);
  };
  tier();
  const double ok[4] = {0.5, -2, 0.25, 1e30f}, odd[4] = {0.5, 0.1, 0, 0};
  const long long slot = 0;
  for (const double* row : {ok, odd, ok}) {
    napi_value a = mock::typed_array(env, napi_float64_array, row, 4);
    if (!mock::call_method(env, ix, "appendF64", {a}, &r, &err)) fprintf(stderr, "appendF64 threw: %s\n", err.c_str());
  }
  mock::call_method(env, ix, "setTier", {mock::object(env, {{"exactRows", str(env, "f32_split")}})}, &r, &err);
  tier();
  napi_value s = mock::typed_array(env, napi_bigint64_array, &slot, 1);
  napi_value o = mock::typed_array(env, napi_float64_array, odd, 4);
  if (!mock::call_method(env, ix, "overwriteF64Batch", {s, o}, &r, &err)) fprintf(stderr, "overwrite threw\n");
  tier();
  mock::delete_env(env);
  return 0;
}
'''


@pytest.fixture(scope="module")
def split_driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("addon_split")
    (d / "stub.cc").write_text(SPLIT_STUB)
    (d / "driver.cc").write_text(SPLIT_DRIVER)
    exe = d / "driver"
    r = subprocess.run([cxx, "-std=c++17", "-O0", "-Wall", "-Werror", "-I", str(ROOT / "napi" / "mock"),
                        "-I", str(ROOT / "include"), str(ROOT / "napi" / "rbk_napi.cc"),
                        str(ROOT / "napi" / "mock" / "mock_napi.cc"), str(d / "stub.cc"), str(d / "driver.cc"),
                        "-o", str(exe), "-lpthread"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return exe


def test_addon_split_rows_and_widen_and_retry(split_driver):
    assert _drive(split_driver, "f32_split") == [
        "create_ex flags 128", "tier f32_split",
        "append 1",
        "append refused", "set_tier flags 1", "append 1",        # refused, widened (split bit cleared), repeated once
        "append 1",
        "set_tier flags 128", "tier f32_split",                  # setTier({ exactRows: 'f32_split' })
        "overwrite refused", "set_tier flags 1", "overwrite 1", "tier f64"]
    assert _drive(split_driver, env={"RUNBOOK_KNN_EXACT_ROWS": "f32_split"})[:2] == ["create_ex flags 128",
                                                                                    "tier f32_split"]


# --------------------------------------------------------------------------- the split rule
HI_CLASSES = {
    "zero": [0x0000, 0x8000],
    "subnormal": [0x0001, 0x0040, 0x007F, 0x8001, 0x807F],
    "normal": [0x0080, 0x3F80, 0x4049, 0xC2F7, 0x7F00, 0x8080],
    "max_finite": [0x7F7F, 0xFF7F],
    "inf": [0x7F80, 0xFF80],
    "nan": [0x7F81, 0x7FC0, 0x7FFF, 0xFF81, 0xFFC0, 0xFFFF],
}


def all_patterns():
    hi = np.array([h for v in HI_CLASSES.values() for h in v], np.uint32)
    lo = np.arange(65536, dtype=np.uint32)
    return ((hi[:, None] << 16) | lo[None, :]).ravel()


def split_rule(u):
    """The split rule of rbk_internal.h, restated: the scan copy s and the low half r of float32 bits u."""
    u = np.asarray(u, np.uint32)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    s = np.where(nan, np.uint32(0x7FFF), (u + np.uint32(0x8000)) >> 16).astype(np.uint16)
    return s, (u & 0xFFFF).astype(np.uint16)


def join(s, r):
    s, r = s.astype(np.uint32), r.astype(np.uint32)
    return ((s - (r >> 15)) << 16) | r


def rne_bf16(u):
    u = np.asarray(u, np.uint32)
    return ((u + np.uint32(0x7FFF) + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def test_split_rule_restores_every_float32():
    u = all_patterns()
    s, r = split_rule(u)
    back = join(s, r)
    f = u.view(np.float32)
    nan = np.isnan(f)
    assert (back[~nan] == u[~nan]).all()
    assert np.isnan(back[nan].view(np.float32)).all()
    assert (s[nan] == 0x7FFF).all()                               # canonical: no carry into the sign bit
    # the scan copy is bf16 rounded to nearest, ties away from zero: it is RNE's except on an exact tie
    fin = ~nan
    tie = (r == 0x8000) & fin
    assert (s[fin & ~tie] == rne_bf16(u[fin & ~tie])).all()
    away = (u[tie] >> 16) + 1
    assert (s[tie] == away).all()
    # the sign is never touched for a non-NaN value; values from 0x7F7F8000 up round to +-inf, as under RNE
    assert ((s[fin] >> 15) == (u[fin] >> 31)).all()
    big = fin & ((u & 0x7FFFFFFF) >= 0x7F7F8000)
    assert ((s[big] & 0x7FFF) == 0x7F80).all()
    # bf16 sources: s = the bits themselves, r = 0
    b = np.arange(65536, dtype=np.uint32) << 16
    sb, rb = split_rule(b)
    okb = ~np.isnan(b.view(np.float32))
    assert (rb == 0).all() and (sb[okb] == (b[okb] >> 16)).all()


HOST_PROBE = r'''
#include <cstdio>
#include "rbk_internal.h"
int main() {
  unsigned u;
  while (fread(&u, 4, 1, stdin) == 1) {
    const unsigned short s = rbk::split_hi(u), r = static_cast<unsigned short>(u & 0xFFFF);
    const unsigned back = rbk::split_join(s, r);
    fwrite(&s, 2, 1, stdout);
    fwrite(&back, 4, 1, stdout);
  }
  return 0;
}
'''


@pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")
def test_library_split_rule_matches_the_restatement(tmp_path):
    """The header's split_hi / split_join, compiled for the host, agree with the numpy rule on every pattern."""
    (tmp_path / "probe.cu").write_text(HOST_PROBE)
    exe = tmp_path / "probe"
    r = subprocess.run([NVCC, "-std=c++17", "-I", str(CSRC), str(tmp_path / "probe.cu"), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    u = all_patterns()
    out = subprocess.run([str(exe)], input=u.tobytes(), capture_output=True, timeout=120).stdout
    rec = np.frombuffer(out, dtype=np.dtype([("s", "<u2"), ("back", "<u4")]))
    s, _ = split_rule(u)
    assert (rec["s"] == s).all()
    assert (rec["back"] == join(*split_rule(u))).all()


@pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")
def test_split_kernels_spill_no_more_than_float32_twins(tmp_path):
    def twin(spills, name, prefix):
        t = [v for n, v in spills.items() if n.startswith(prefix)]
        assert len(t) == 1, (name, t)
        return int(t[0])

    spills = _ptxas(tmp_path, "rbk_finalize.cu")
    split = {n: s for n, s in spills.items() if "split_kernel" in n or "5F32Lo" in n}
    assert len(split) == 6, list(split)                          # finalize x2, large_score x2, exact_scan, exact_scores
    for name, s in split.items():
        m = re.search(r"\d+(finalize|large_score)_split_kernel(ILb[01]E)", name)
        if m:
            k = f"{m.group(1)}_f32_kernel"
            t = twin(spills, name, name[:m.start()] + f"{len(k)}{k}{m.group(2)}")
        else:
            t = twin(spills, name, name.split("NS_5F32LoE")[0] + "f")
        assert int(s) <= t, (name, s, t)
    spills = _ptxas(tmp_path, "rbk_ingest.cu")
    split = {n: s for n, s in spills.items() if "5F32Lo" in n}
    assert len(split) == 6, list(split)                          # convert x3, row_norms, join x2
    for name, s in split.items():
        if "join_exact" in name:
            assert s == "0", name
        else:
            assert int(s) <= twin(spills, name, name.split("NS_5F32LoE")[0] + "f"), name
    spills = _ptxas(tmp_path, "rbk_compact.cu")
    assert any("5F32Lo" in n for n in spills) and all(s == "0" for s in spills.values())
