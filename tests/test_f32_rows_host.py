"""CPU suite for float32 exact rows (RBK_INDEX_KEEP_F32): the header and the binding agree, the flag helpers build the
right sets, the vector store widens its index and repeats a refused call, and the new kernel instantiations compile
without spills."""
import importlib.util
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from common import OracleIndex

ROOT = Path(__file__).resolve().parents[1]
HEADER = ROOT / "include" / "rbk_knn.h"
CSRC = ROOT / "runbookai_b200" / "csrc"
NVCC = "/usr/local/cuda/bin/nvcc"


def test_header_defines_match_the_binding():
    from runbookai_b200 import _native as n
    h = HEADER.read_text()
    assert re.search(r"#define RBK_INDEX_KEEP_F32 64u", h)
    assert re.search(r"#define RBK_INDEX_ROWS_ON_HOST RBK_INDEX_F64_ON_HOST", h)
    assert re.search(r"RBK_ENOTF32 = 6", h)
    assert (n.RBK_INDEX_KEEP_F32, n.RBK_ENOTF32, n.RBK_INDEX_ROWS_ON_HOST) == (64, 6, n.RBK_INDEX_F64_ON_HOST)
    assert issubclass(n.NotFloat32Error, n.RbkError)
    for sym in n.SYMBOLS:
        assert getattr(n.lib, sym) is not None


def test_flag_helpers():
    from runbookai_b200._native import _index_flags, _tier_flags, exact_rows_of
    assert _index_flags(False, False, False, True) == 64
    assert _index_flags(False, True, True, True) == 64 | 2 | 16
    assert _index_flags(True, False, False, True) == 65         # passed through: the library refuses it
    assert _tier_flags(1 | 2, None, None, "f32") == 64 | 2
    assert _tier_flags(64 | 16, False, None, "f64") == 1 | 16
    assert _tier_flags(64, None, None, None) == 64
    assert _tier_flags(0, None, None, "f32") == 64              # no exact rows: the library refuses the change
    with pytest.raises(ValueError):
        _tier_flags(1, None, None, "f16")
    assert (exact_rows_of(1), exact_rows_of(64 | 2), exact_rows_of(0)) == ("f64", "f32", None)


def test_check_flags_without_a_device():
    """check_flags runs before the device is looked at: refused sets are RBK_EINVAL even here."""
    import ctypes as C
    from runbookai_b200._native import RBK_EINVAL, lib
    h = C.c_void_p()
    for flags in (1 | 64, 1 | 64 | 2, 2, 16, 2 | 16, 4, 8, 32):
        assert lib.rbk_index_create_ex(16, 0, 0, flags, C.byref(h)) == RBK_EINVAL, flags
    for flags in (64, 64 | 2, 64 | 16, 64 | 2 | 16, 1 | 2 | 16):
        h = C.c_void_p()
        assert lib.rbk_index_create_ex(16, 0, 0, flags, C.byref(h)) != RBK_EINVAL, flags
        lib.rbk_index_destroy(h)


class Float32Stub(OracleIndex):
    """OracleIndex that behaves like a keep_f32 index: float64 values no float32 holds are refused with RBK_ENOTF32
    (nothing written) until set_tier(exact_rows='f64')."""

    def __init__(self, dim, device=0, capacity_hint=0):
        super().__init__(dim, device, capacity_hint)
        self.flags = 64
        self.widened = 0

    def _guard(self, rows):
        from runbookai_b200._native import RBK_ENOTF32, NotFloat32Error
        r = np.asarray(rows, dtype=np.float64)
        if self.flags & 64 and not np.array_equal(r.astype(np.float32).astype(np.float64), r, equal_nan=True):
            raise NotFloat32Error(RBK_ENOTF32, "a value is not exactly a float32")

    def set_tier(self, *, f64_on_host=None, scan_f16=None, exact_rows=None):
        assert exact_rows == "f64" and f64_on_host is None and scan_f16 is None
        self.flags = 1
        self.widened += 1

    def append_f64(self, rows):
        self._guard(rows)
        return super().append_f64(rows)

    def overwrite_f64(self, slot, row):
        self._guard(row)
        return super().overwrite_f64(slot, row)

    def overwrite_f64_batch(self, slots, rows):
        self._guard(rows)
        return super().overwrite_f64_batch(slots, rows)


def test_vector_store_widens_and_repeats(tmp_path, monkeypatch):
    from runbookai_b200.vector_store import VectorStore
    made = []

    def factory(dim, dev):
        made.append(Float32Stub(dim))
        return made[-1]

    vs = VectorStore(":memory:", index_factory=factory, exact_rows="f32")
    try:
        assert vs.exact_rows == "f32"
        e = np.float32(np.random.default_rng(0).standard_normal(8)).astype(np.float64)
        vs._set("vec_a", e)
        vs._set("vec_b", e * 2)
        assert vs.exact_rows == "f32" and made[0].widened == 0
        odd = e.copy()
        odd[3] = 0.1
        vs._set("vec_a", odd)                                    # an overwrite the float32 index refuses
        assert made[0].widened == 1 and vs.exact_rows == "f64"
        vs._set("vec_c", odd)                                    # the widened index takes it directly
        assert made[0].widened == 1
        assert vs._index.size() == 3
    finally:
        vs.close()
    monkeypatch.setenv("RUNBOOK_KNN_EXACT_ROWS", "f32")
    vs = VectorStore(":memory:", index_factory=factory)
    try:
        assert vs.exact_rows == "f32"
    finally:
        vs.close()
    with pytest.raises(ValueError):
        VectorStore(":memory:", index_factory=factory, exact_rows="f16")


def _ptxas(tmp_path, source):
    spec = importlib.util.spec_from_file_location("rbk_build", ROOT / "runbookai_b200" / "build.py")
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    res = subprocess.run([NVCC, "-Xptxas=-v", *flags, "-c", str(CSRC / source), "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    report, current = {}, None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            report[current] = ""
        elif current is not None:
            report[current] += line + "\n"
    return {n: re.search(r"(\d+) bytes spill stores", t).group(1) for n, t in report.items()}


@pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")
def test_float32_row_kernels_have_no_spills(tmp_path):
    spills = _ptxas(tmp_path, "rbk_finalize.cu")
    f32 = {n: s for n, s in spills.items() if "f32_kernel" in n or "IfEEv" in n}
    assert len(f32) == 6, list(f32)                              # finalize x2, large_score x2, exact_scan, exact_scores
    for name, s in f32.items():
        if "finalize_f32_kernelILb0" in name:                    # spills exactly what its float64 twin does
            twin = [v for n, v in spills.items() if "15finalize_kernelILb0" in n]
            assert [s] == twin, (name, s, twin)
        else:
            assert s == "0", name
    # ingest: each float32-row instantiation spills exactly what its float64 twin does (the fp16 conversion of a float64
    # source keeps a few bytes on the stack either way)
    spills = _ptxas(tmp_path, "rbk_ingest.cu")
    pat = r"(kernelI(?:[dft]|Lb[01]E))f"
    f32 = {n: s for n, s in spills.items() if re.search(pat, n) and "convert_exact" not in n}
    assert len(f32) == 8, list(f32)                              # convert x3, convert_f16 x3, row_norms x2
    assert all(s == "0" for n, s in spills.items() if "convert_exact" in n or "find_not_f32" in n)
    for name, s in f32.items():
        assert s == spills[re.sub(pat, r"\1d", name)], name
    spills = _ptxas(tmp_path, "rbk_compact.cu")
    assert any("IfEEv" in n for n in spills) and all(s == "0" for s in spills.values())


# --------------------------------------------------------------------------- the N-API addon's exactRows
# A stand-in of librbk_knn.so for the addon alone: one index whose flags the calls record; a float32-row index refuses
# any float64 value no float32 holds with RBK_ENOTF32, as the library does.
ADDON_STUB = r'''
#include <cmath>
#include <cstdio>
#include "rbk_knn.h"
static uint32_t g_flags = 0;
static int64_t g_rows = 0;
static rbk_index* const kIx = reinterpret_cast<rbk_index*>(0x10);
extern "C" {
const char* rbk_last_error(void) { return "stand-in refusal"; }
rbk_status rbk_index_create_ex(int32_t, int32_t, int64_t, uint32_t flags, rbk_index** out) {
  fprintf(stderr, "create_ex flags %u\n", flags);
  g_flags = flags;
  *out = kIx;
  return RBK_OK;
}
void rbk_index_destroy(rbk_index*) {}
uint32_t rbk_index_flags(const rbk_index*) { return g_flags; }
rbk_status rbk_index_set_tier(rbk_index*, uint32_t flags) {
  fprintf(stderr, "set_tier flags %u\n", flags);
  g_flags = flags;
  return RBK_OK;
}
static bool fits(const double* v, int64_t n) {
  if (!(g_flags & RBK_INDEX_KEEP_F32)) return true;
  for (int64_t i = 0; i < n; ++i)
    if (v[i] == v[i] && (double)(float)v[i] != v[i]) return false;
  return true;
}
rbk_status rbk_index_append_f64(rbk_index*, const double* rows, int64_t n, int64_t* first) {
  if (!fits(rows, n * 4)) { fprintf(stderr, "append refused\n"); return RBK_ENOTF32; }
  fprintf(stderr, "append %lld\n", (long long)n);
  *first = g_rows;
  g_rows += n;
  return RBK_OK;
}
rbk_status rbk_index_overwrite_f64_batch(rbk_index*, const int64_t*, int64_t n, const double* rows) {
  if (!fits(rows, n * 4)) { fprintf(stderr, "overwrite refused\n"); return RBK_ENOTF32; }
  fprintf(stderr, "overwrite %lld\n", (long long)n);
  return RBK_OK;
}
#define NOPE { return RBK_EINVAL; }
rbk_status rbk_index_tombstone(rbk_index*, const int64_t*, int64_t) NOPE
rbk_status rbk_index_clear(rbk_index*) NOPE
rbk_status rbk_index_compact(rbk_index*, int64_t*, int64_t) NOPE
rbk_status rbk_index_trim(rbk_index*) NOPE
int64_t rbk_index_count(const rbk_index*) { return g_rows; }
int64_t rbk_index_size(const rbk_index*) { return g_rows; }
rbk_status rbk_index_search_f64(rbk_index*, const double*, int32_t, int32_t, int32_t, double, int64_t*, double*,
                                int32_t*, float*) NOPE
rbk_status rbk_index_search_large_f64(rbk_index*, const double*, int32_t, int32_t, int32_t, double, int64_t*, double*,
                                      int32_t*, float*) NOPE
rbk_status rbk_index_search_unbounded_f64(rbk_index*, const double*, int32_t, int32_t, int32_t, double, int64_t*,
                                          double*, int32_t*, float*) NOPE
rbk_status rbk_group_create(int32_t, const int32_t*, int32_t, int64_t, uint32_t, rbk_group**) NOPE
void rbk_group_destroy(rbk_group*) {}
rbk_status rbk_group_append_f64(rbk_group*, const double*, int64_t, int64_t*) NOPE
rbk_status rbk_group_overwrite_f64_batch(rbk_group*, const int64_t*, int64_t, const double*) NOPE
rbk_status rbk_group_tombstone(rbk_group*, const int64_t*, int64_t) NOPE
rbk_status rbk_group_clear(rbk_group*) NOPE
rbk_status rbk_group_compact(rbk_group*, int64_t*, int64_t) NOPE
rbk_status rbk_group_trim(rbk_group*) NOPE
int64_t rbk_group_count(const rbk_group*) { return 0; }
int64_t rbk_group_size(const rbk_group*) { return 0; }
rbk_index* rbk_group_member(rbk_group*, int32_t) { return kIx; }
rbk_status rbk_group_set_tier(rbk_group*, uint32_t) NOPE
rbk_status rbk_group_search_f64(rbk_group*, const double*, int32_t, int32_t, int32_t, double, int64_t*, double*,
                                int32_t*, float*) NOPE
rbk_status rbk_group_search_large_f64(rbk_group*, const double*, int32_t, int32_t, int32_t, double, int64_t*, double*,
                                      int32_t*, float*) NOPE
rbk_status rbk_group_search_unbounded_f64(rbk_group*, const double*, int32_t, int32_t, int32_t, double, int64_t*,
                                          double*, int32_t*, float*) NOPE
}
'''

ADDON_DRIVER = r'''
#include <cstdio>
#include <cstdlib>
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
    char buf[8] = {0};
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
  mock::call_method(env, ix, "setTier", {mock::object(env, {{"exactRows", str(env, "f32")}})}, &r, &err);
  tier();
  napi_value s = mock::typed_array(env, napi_bigint64_array, &slot, 1);
  napi_value o = mock::typed_array(env, napi_float64_array, odd, 4);
  if (!mock::call_method(env, ix, "overwriteF64Batch", {s, o}, &r, &err)) fprintf(stderr, "overwrite threw\n");
  tier();
  if (mock::call_method(env, ix, "setTier", {mock::object(env, {{"exactRows", str(env, "f16")}})}, &r, &err))
    fprintf(stderr, "setTier f16 did not throw\n");
  else
    fprintf(stderr, "setTier threw: %s\n", err.c_str());
  mock::delete_env(env);
  return 0;
}
'''


@pytest.fixture(scope="module")
def addon_driver(tmp_path_factory):
    import shutil
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("addon_f32")
    (d / "stub.cc").write_text(ADDON_STUB)
    (d / "driver.cc").write_text(ADDON_DRIVER)
    exe = d / "driver"
    r = subprocess.run([cxx, "-std=c++17", "-O0", "-Wall", "-Werror", "-I", str(ROOT / "napi" / "mock"),
                        "-I", str(ROOT / "include"), str(ROOT / "napi" / "rbk_napi.cc"),
                        str(ROOT / "napi" / "mock" / "mock_napi.cc"), str(d / "stub.cc"), str(d / "driver.cc"),
                        "-o", str(exe), "-lpthread"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return exe


def _drive(exe, *args, env=None):
    import os
    e = dict(os.environ)
    e.pop("RUNBOOK_KNN_EXACT_ROWS", None)
    e.update(env or {})
    r = subprocess.run([str(exe), *args], capture_output=True, text=True, env=e, timeout=60)
    assert r.returncode == 0, r.stderr
    return r.stderr.splitlines()


def test_addon_exact_rows_and_widen_and_retry(addon_driver):
    log = _drive(addon_driver, "f32")
    assert log == ["create_ex flags 64", "tier f32",
                   "append 1",                                   # float32-exact: taken as it is
                   "append refused", "set_tier flags 1", "append 1",   # refused, widened in place, repeated once
                   "append 1",                                   # the index is float64 now
                   "set_tier flags 64", "tier f32",              # setTier({ exactRows: 'f32' })
                   "overwrite refused", "set_tier flags 1", "overwrite 1", "tier f64",
                   "setTier threw: setTier: exactRows must be 'f64' or 'f32'"]


def test_addon_exact_rows_default_and_environment(addon_driver):
    assert _drive(addon_driver)[:2] == ["create_ex flags 1", "tier f64"]
    assert _drive(addon_driver, env={"RUNBOOK_KNN_EXACT_ROWS": "f32"})[:2] == ["create_ex flags 64", "tier f32"]
    assert _drive(addon_driver, "f64", env={"RUNBOOK_KNN_EXACT_ROWS": "f32"})[:2] == ["create_ex flags 1", "tier f64"]
    assert _drive(addon_driver, "f16") == ["construct threw: exactRows must be 'f64' or 'f32'"]
