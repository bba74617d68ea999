"""The fp16 scan of float64-backed indexes (RBK_INDEX_SCAN_F16) without a GPU: the declared flag and
`rbk_index_read_rows_f16`, the library's flag checks, the plumbing of `Index` / `Group` / `VectorStore` (and its
environment variable) down to `rbk_index_create_ex` / `rbk_group_create` through a recording stand-in of the library,
the N-API addon's `scanF16` argument against an oracle-backed stand-in of the C ABI
(tests/napi_shim/rbk_shim_scan_f16.cc), and the compiled fp16 scan: three instantiations in their own translation unit,
no spills, fp16 HGMMA only, and the bf16 scan's HGMMA unchanged."""
import ctypes as C
import importlib.util
import re
import shutil
import subprocess
from collections import Counter
from pathlib import Path

import pytest

from conftest import ROOT
from test_napi_addon import _check_outputs, _write_inputs

CSRC = ROOT / "runbookai_b200" / "csrc"
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).parent / "cuobjdump")


def test_header_declares_the_flag_and_the_read_call(native):
    header = (ROOT / "include" / "rbk_knn.h").read_text()
    assert "#define RBK_INDEX_SCAN_F16 16u" in header
    assert ("rbk_status rbk_index_read_rows_f16(rbk_index* idx, int64_t first_local_slot, int64_t n_rows, "
            "uint16_t* out);") in header
    assert "#define RBK_ABI_VERSION 2" in header
    assert "rbk_index_read_rows_f16" in native.SYMBOLS
    assert native.RBK_INDEX_SCAN_F16 == 16
    assert hasattr(C.CDLL(str(native.LIB_PATH)), "rbk_index_read_rows_f16")   # the built library exports it


def test_library_checks_the_flag_before_looking_for_a_device(native):
    """Flag errors come before the device lookup, so they are the same with or without a GPU."""
    for flags, msg in ((16, "RBK_INDEX_SCAN_F16 requires RBK_INDEX_KEEP_F64"),
                       (16 | 2, "RBK_INDEX_F64_ON_HOST requires RBK_INDEX_KEEP_F64"),
                       (16 | 4, "unknown flag"), (32 | 1, "unknown flag")):
        h = C.c_void_p()
        assert native.lib.rbk_index_create_ex(64, 0, 0, flags, C.byref(h)) == native.RBK_EINVAL
        assert native.lib.rbk_last_error().decode() == msg
        assert not h.value
    with pytest.raises(native.RbkError, match="RBK_INDEX_SCAN_F16 requires RBK_INDEX_KEEP_F64"):
        native.Index(64, scan_f16=True)


class RecordingLib:
    """Stands in for librbk_knn.so: records the flags of every create call and checks them as the library does."""

    def __init__(self):
        self.calls = []
        self.err = b""

    def _create(self, kind, flags, out):
        self.calls.append((kind, flags))
        if flags & ~(1 | 2 | 16):
            self.err = b"unknown flag"
            return 1
        for bit, name in ((2, b"RBK_INDEX_F64_ON_HOST"), (16, b"RBK_INDEX_SCAN_F16")):
            if flags & bit and not flags & 1:
                self.err = name + b" requires RBK_INDEX_KEEP_F64"
                return 1
        out._obj.value = 0x1000 + len(self.calls)   # out = ctypes.byref(handle)
        return 0

    def rbk_index_create_ex(self, dim, device, hint, flags, out):
        return self._create("index", flags, out)

    def rbk_group_create(self, dim, devs, n, hint, flags, out):
        return self._create("group", flags, out)

    def rbk_last_error(self):
        return self.err

    def rbk_index_destroy(self, h):
        pass

    rbk_group_destroy = rbk_index_destroy


@pytest.fixture
def recording(native, monkeypatch):
    rec = RecordingLib()
    monkeypatch.setattr(native, "lib", rec)
    return rec


def test_index_and_group_pass_the_flag(native, recording):
    native.Index(64, keep_f64=True, scan_f16=True).close()
    native.Index(64, keep_f64=True, f64_on_host=True, scan_f16=True).close()
    native.Index(64, keep_f64=True).close()
    native.Group(64, [0], keep_f64=True, scan_f16=True).close()
    native.Group(64, [0], keep_f64=True, f64_on_host=True, scan_f16=True).close()
    native.Group(64, [0], keep_f64=True).close()
    assert recording.calls == [("index", 17), ("index", 19), ("index", 1), ("group", 17), ("group", 19), ("group", 1)]
    with pytest.raises(native.RbkError, match="RBK_INDEX_SCAN_F16 requires RBK_INDEX_KEEP_F64"):
        native.Group(64, [0], scan_f16=True)


@pytest.mark.parametrize("env, arg, host, want", [(None, None, None, 1), ("0", None, None, 1), ("1", None, None, 17),
                                                  ("1", False, None, 1), (None, True, None, 17), ("1", None, "1", 19)])
def test_vector_store_scan_from_argument_and_environment(tmp_path, native, recording, monkeypatch, env, arg, host,
                                                         want):
    from runbookai_b200.vector_store import VectorStore
    monkeypatch.setenv("RUNBOOK_KNN_SIDECAR", "0")
    for var, val in (("RUNBOOK_KNN_SCAN_F16", env), ("RUNBOOK_KNN_F64_ON_HOST", host)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)
    vs = VectorStore(str(tmp_path / "vectors.db"), scan_f16=arg)
    assert vs.scan_f16 == bool(want & 16)
    vs._ensure_index(64)
    vs.close()
    assert recording.calls == [("index", want)]


def test_create_vector_store_and_retriever_pass_it_through(tmp_path, native, recording, monkeypatch):
    from runbookai_b200 import embedder
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import create_vector_store
    monkeypatch.setenv("RUNBOOK_KNN_SIDECAR", "0")
    monkeypatch.delenv("RUNBOOK_KNN_SCAN_F16", raising=False)
    (tmp_path / "a").mkdir()
    vs = create_vector_store(str(tmp_path / "a"), shared=False, scan_f16=True)
    vs._ensure_index(64)
    vs.close()
    monkeypatch.setattr(embedder, "is_embedder_configured", lambda: True)
    kr = KnowledgeRetriever({"storePath": str(tmp_path / "b" / "knowledge.db")}, scan_f16=True)
    assert kr.vector_store.scan_f16
    kr.vector_store._ensure_index(64)
    kr.vector_store.close()
    assert recording.calls == [("index", 17), ("index", 17)]


@pytest.fixture(scope="module")
def shim_scan_f16_harness(tmp_path_factory, oracle_mod):
    """The addon harness linked against rbk_shim_scan_f16.cc (built in a temporary directory)."""
    spec = importlib.util.spec_from_file_location("rbk_napi_mock_build", ROOT / "napi" / "mock" / "build.py")
    mb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mb)
    objs = mb.build_objects()
    olib = ROOT / "oracle" / "librbk_oracle.so"
    out = tmp_path_factory.mktemp("shim_scan_f16")
    shim = out / "librbk_knn_shim_scan_f16.so"
    mb.run(mb.CXX + ["-fPIC", "-shared", ROOT / "tests" / "napi_shim" / "rbk_shim_scan_f16.cc", "-o", shim,
                     "-L", olib.parent, "-l:librbk_oracle.so", f"-Wl,-rpath,{olib.parent}"])
    exe = out / "harness_shim_scan_f16"
    mb.run(["g++"] + objs + ["-o", exe, "-L", out, "-l:librbk_knn_shim_scan_f16.so", f"-Wl,-rpath,{out}",
                             f"-Wl,-rpath,{olib.parent}", "-L", olib.parent, "-l:librbk_oracle.so", "-lpthread"])
    return exe


@pytest.mark.parametrize("devices, kind", [([], "create_ex"), ([0], "group_create")], ids=["index", "group"])
@pytest.mark.parametrize("host_rows, scan_f16, want", [(None, None, 1), (None, 0, 1), (None, 1, 17), (1, 1, 19),
                                                       (1, None, 3)],
                         ids=["absent", "zero", "one", "with-host-rows", "host-rows-only"])
def test_addon_scan_f16_argument(tmp_path, oracle_mod, shim_scan_f16_harness, devices, kind, host_rows, scan_f16,
                                 want):
    w = _write_inputs(tmp_path, devices)
    if host_rows is not None:
        (tmp_path / "host_rows.txt").write_text(f"{host_rows}\n")
    if scan_f16 is not None:
        (tmp_path / "scan_f16.txt").write_text(f"{scan_f16}\n")
    r = subprocess.run([str(shim_scan_f16_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert re.findall(r"(create_ex|group_create) flags (\d+)", r.stderr) == [(kind, str(want))]
    _check_outputs(tmp_path, w, oracle_mod)


def test_typescript_wrapper_reads_the_environment_variable():
    ts = (ROOT / "ts" / "gpu-embedding-index.ts").read_text()
    assert "process.env.RUNBOOK_KNN_SCAN_F16 === '1'" in ts
    assert ts.count("hostRowsFromEnv(), scanF16FromEnv())") == 2


# --------------------------------------------------------------------------- the compiled kernels
def _compile(tmp_path: Path, src: str, *defines: str) -> tuple[Path, str]:
    spec = importlib.util.spec_from_file_location("rbk_build", ROOT / "runbookai_b200" / "build.py")
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    assert src in build.SOURCES and "rbk_scan_kernel.cuh" in build.HEADERS
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    out = tmp_path / f"{src}{len(defines)}.cubin"
    res = subprocess.run([NVCC, "-Xptxas=-v", *defines, *flags, "-cubin", str(CSRC / src), "-o", str(out)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return out, res.stdout + res.stderr


def _report(log: str) -> dict[str, str]:
    report: dict[str, str] = {}
    current = None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            report[current] = ""
        elif current is not None:
            report[current] += line + "\n"
    return report


def _hgmma(cubin: Path) -> dict[str, Counter]:
    sass = subprocess.run([CUOBJDUMP, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    shape: dict[str, Counter] = {}
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : \S*scan_kernelILi(\d)", line)
        if m:
            cur = shape.setdefault(m.group(1), Counter())
            continue
        if "Function :" in line:
            cur = None
        m = re.search(r"(HGMMA\.\S+)", line)
        if cur is not None and m:
            op = m.group(1).rstrip(",")
            cur[op] += 1
    return shape


needs_nvcc = pytest.mark.skipif(not (Path(NVCC).exists() and Path(CUOBJDUMP).exists()),
                                reason="nvcc / cuobjdump not available")


@needs_nvcc
def test_f16_scan_compiles_with_three_instantiations_and_no_spills(tmp_path):
    cubin, log = _compile(tmp_path, "rbk_scan_f16.cu")
    scans = {n: t for n, t in _report(log).items() if "scan_kernel" in n}
    assert sorted(re.search(r"scan_kernelILi(\d)", n).group(1) for n in scans) == ["0", "1", "2"], list(scans)
    assert all("rbk_scan_f16_cu" in n for n in scans)
    for name, text in scans.items():
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
        assert m, (name, text)
        stack, stores, loads = map(int, m.groups())
        assert stores == 0 and loads == 0 and stack <= 64, (name, text)
        assert int(re.search(r"Used (\d+) registers", text).group(1)) <= 168, (name, text)
    shape = _hgmma(cubin)
    assert sorted(shape) == ["0", "1", "2"], shape
    for mode, ops in shape.items():
        assert sum(ops.values()) >= 4, (mode, ops)
        assert not any("BF16" in op for op in ops), (mode, ops)        # sm_90 SASS prints fp16 HGMMA without a type
        assert all(op.startswith("HGMMA.64x256x16.F32") for op in ops), (mode, ops)
    # the probe stays in the bf16 translation unit
    probe, _ = _compile(tmp_path, "rbk_scan_f16.cu", "-DRBK_SCAN_CYCLE_STATS")
    assert b"g_cycle_stats" not in cubin.read_bytes() and b"g_cycle_stats" not in probe.read_bytes()


@needs_nvcc
def test_bf16_scan_keeps_its_bf16_hgmma(tmp_path):
    shape = _hgmma(_compile(tmp_path, "rbk_scan.cu")[0])
    assert sorted(shape) == ["0", "1", "2"], shape
    for mode, ops in shape.items():
        assert ops and all(op.startswith("HGMMA.64x256x16.F32.BF16") for op in ops), (mode, ops)
    f16 = _hgmma(_compile(tmp_path, "rbk_scan_f16.cu")[0])
    assert {m: sum(o.values()) for m, o in f16.items()} == {m: sum(o.values()) for m, o in shape.items()}
