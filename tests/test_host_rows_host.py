"""Float64 rows in pinned host memory (RBK_INDEX_F64_ON_HOST) without a GPU: the declared flag and
`rbk_index_storage_bytes`, the plumbing of `Index` / `Group` / `VectorStore` (and its environment variable) down to
`rbk_index_create_ex` / `rbk_group_create` through a recording stand-in of the library, the N-API addon's `hostRows`
argument against an oracle-backed stand-in of the C ABI (tests/napi_shim/rbk_shim_flags.cc), and the register budget
of the host-row instantiations of the re-rank kernels."""
import ctypes as C
import importlib.util
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from conftest import ROOT
from test_napi_addon import _check_outputs, _write_inputs

CSRC = ROOT / "runbookai_b200" / "csrc"
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def test_header_declares_the_flag_and_storage_bytes(native):
    header = (ROOT / "include" / "rbk_knn.h").read_text()
    assert "#define RBK_INDEX_F64_ON_HOST 2u" in header
    assert ("rbk_status rbk_index_storage_bytes(const rbk_index* idx, int64_t* device_bytes, "
            "int64_t* pinned_host_bytes);") in header
    assert "rbk_index_storage_bytes" in native.SYMBOLS
    assert native.RBK_INDEX_F64_ON_HOST == 2 and native.RBK_INDEX_KEEP_F64 == 1
    assert hasattr(C.CDLL(str(native.LIB_PATH)), "rbk_index_storage_bytes")   # the built library exports it


class RecordingLib:
    """Stands in for librbk_knn.so: records the flags of every create call and checks them as the library does."""

    def __init__(self):
        self.calls = []
        self.err = b""

    def _create(self, kind, flags, out):
        self.calls.append((kind, flags))
        if flags & ~3:
            self.err = b"unknown flag"
            return 1
        if flags & 2 and not flags & 1:
            self.err = b"RBK_INDEX_F64_ON_HOST requires RBK_INDEX_KEEP_F64"
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


def test_index_and_group_pass_the_flags(native, recording):
    native.Index(64, keep_f64=True, f64_on_host=True).close()
    native.Index(64, keep_f64=True).close()
    native.Index(64).close()
    native.Group(64, [0], keep_f64=True, f64_on_host=True).close()
    native.Group(64, [0], keep_f64=True).close()
    assert recording.calls == [("index", 3), ("index", 1), ("index", 0), ("group", 3), ("group", 1)]


def test_f64_on_host_without_keep_f64_raises_the_library_error(native, recording):
    with pytest.raises(native.RbkError, match="RBK_INDEX_F64_ON_HOST requires RBK_INDEX_KEEP_F64") as e:
        native.Index(64, f64_on_host=True)
    assert e.value.status == native.RBK_EINVAL
    with pytest.raises(native.RbkError, match="requires RBK_INDEX_KEEP_F64"):
        native.Group(64, [0], f64_on_host=True)
    assert recording.calls == [("index", 2), ("group", 2)]


@pytest.mark.parametrize("env, arg, want", [(None, None, 1), ("0", None, 1), ("1", None, 3), ("1", False, 1),
                                            (None, True, 3)])
def test_vector_store_placement_from_argument_and_environment(tmp_path, native, recording, monkeypatch, env, arg, want):
    from runbookai_b200.vector_store import VectorStore
    monkeypatch.setenv("RUNBOOK_KNN_SIDECAR", "0")
    if env is None:
        monkeypatch.delenv("RUNBOOK_KNN_F64_ON_HOST", raising=False)
    else:
        monkeypatch.setenv("RUNBOOK_KNN_F64_ON_HOST", env)
    vs = VectorStore(str(tmp_path / "vectors.db"), f64_on_host=arg)
    assert vs.f64_on_host == (want == 3)
    vs._ensure_index(64)
    vs.close()
    assert recording.calls == [("index", want)]


@pytest.fixture(scope="module")
def shim_flags_harness(tmp_path_factory, oracle_mod):
    """The addon harness linked against rbk_shim_flags.cc (built in a temporary directory)."""
    spec = importlib.util.spec_from_file_location("rbk_napi_mock_build", ROOT / "napi" / "mock" / "build.py")
    mb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mb)
    objs = mb.build_objects()
    olib = ROOT / "oracle" / "librbk_oracle.so"
    out = tmp_path_factory.mktemp("shim_flags")
    shim = out / "librbk_knn_shim_flags.so"
    mb.run(mb.CXX + ["-fPIC", "-shared", ROOT / "tests" / "napi_shim" / "rbk_shim_flags.cc", "-o", shim,
                     "-L", olib.parent, "-l:librbk_oracle.so", f"-Wl,-rpath,{olib.parent}"])
    exe = out / "harness_shim_flags"
    mb.run(["g++"] + objs + ["-o", exe, "-L", out, "-l:librbk_knn_shim_flags.so", f"-Wl,-rpath,{out}",
                             f"-Wl,-rpath,{olib.parent}", "-L", olib.parent, "-l:librbk_oracle.so", "-lpthread"])
    return exe


@pytest.mark.parametrize("devices, kind", [([], "create_ex"), ([0], "group_create")], ids=["index", "group"])
@pytest.mark.parametrize("host_rows, want", [(None, 1), (0, 1), (1, 3)], ids=["absent", "zero", "one"])
def test_addon_host_rows_argument(tmp_path, oracle_mod, shim_flags_harness, devices, kind, host_rows, want):
    w = _write_inputs(tmp_path, devices)
    if host_rows is not None:
        (tmp_path / "host_rows.txt").write_text(f"{host_rows}\n")
    r = subprocess.run([str(shim_flags_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert re.findall(r"(create_ex|group_create) flags (\d+)", r.stderr) == [(kind, str(want))]
    _check_outputs(tmp_path, w, oracle_mod)


def _ptxas_report(tmp_path: Path) -> dict[str, str]:
    spec = importlib.util.spec_from_file_location("rbk_build", ROOT / "runbookai_b200" / "build.py")
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    cmd = [NVCC, "-Xptxas=-v", *flags, "-c", str(CSRC / "rbk_finalize.cu"), "-o", str(tmp_path / "rbk_finalize.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    report: dict[str, str] = {}
    current = None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            report[current] = ""
        elif current is not None:
            report[current] += line + "\n"
    return report


@pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")
def test_host_row_rerank_kernels_have_no_spills(tmp_path):
    report = _ptxas_report(tmp_path)
    for kernel in ("finalize_kernel", "large_score_kernel"):
        inst = {n: t for n, t in report.items() if kernel in n}
        assert sorted(re.search(kernel + r"ILb(\d)", n).group(1) for n in inst) == ["0", "1"], list(inst)
        (name, text), = [(n, t) for n, t in inst.items() if kernel + "ILb1" in n]
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
        assert m and m.groups() == ("0", "0", "0"), (name, text)
