"""The RBK_SCAN_CYCLE_STATS cycle probe of the fused scan times the same wgmma pipeline as the default build, and
leaves no trace in the default build.

The probe adds clock reads and register pressure to the scan's main loop; a default library carrying any of it would be
a slower library.  A probe build whose wgmma pipeline ptxas had serialized (it does so around any call in the kernel,
a printf for one) would time another kernel, so both builds must issue the same HGMMA groups with the same waits.
Runs without a GPU; skips when nvcc is absent.
"""
from __future__ import annotations

import importlib.util
import re
import shutil
import subprocess
from collections import Counter
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "runbookai_b200" / "csrc"
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).parent / "cuobjdump")

pytestmark = pytest.mark.skipif(not (Path(NVCC).exists() and Path(CUOBJDUMP).exists()),
                                reason="nvcc / cuobjdump not available")


def _cubin(tmp_path: Path, *defines: str) -> tuple[Path, str]:
    """(cubin, ptxas report) of rbk_scan.cu."""
    spec = importlib.util.spec_from_file_location("rbk_build", ROOT / "runbookai_b200" / "build.py")
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    out = tmp_path / f"scan{len(defines)}.cubin"
    res = subprocess.run([NVCC, "-Xptxas=-v", *defines, *flags, "-cubin", str(CSRC / "rbk_scan.cu"), "-o", str(out)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return out, res.stdout + res.stderr


def _wgmma_shape(cubin: Path) -> dict[str, Counter]:
    """Per scan_kernel instantiation: counts of HGMMA, wgmma fences and each wait_group depth."""
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
        if cur is None:
            continue
        m = re.search(r"(HGMMA\.\S+|WARPGROUP\.ARRIVE|WARPGROUP\.DEPBAR\.LE gsb0, 0x[0-9a-f]+)", line)
        if m:
            cur[m.group(1)] += 1
    return shape


def test_probe_build_keeps_the_wgmma_pipeline(tmp_path):
    default, default_log = _cubin(tmp_path)
    probe, probe_log = _cubin(tmp_path, "-DRBK_SCAN_CYCLE_STATS")
    for log in (default_log, probe_log):
        assert "C7510" not in log and "serialized" not in log, log
    shape = _wgmma_shape(default)
    assert sorted(shape) == ["0", "1", "2"], shape
    assert all(s["WARPGROUP.DEPBAR.LE gsb0, 0x1"] >= 1 for s in shape.values()), shape
    assert _wgmma_shape(probe) == shape


def test_default_build_has_no_cycle_probe(tmp_path):
    default = _cubin(tmp_path)[0].read_bytes()
    probe = _cubin(tmp_path, "-DRBK_SCAN_CYCLE_STATS")[0].read_bytes()
    for marker in (b"g_cycle_stats",):
        assert marker in probe, marker   # the marker does identify the probe
        assert marker not in default, marker
