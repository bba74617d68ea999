"""The fused scan kernel compiles for sm_90a without register spills in any of its three instantiations.

The wgmma warpgroups hold 128 fp32 accumulators per thread next to the score prefilter; a spill there would put
local-memory traffic on every tile.  Runs without a GPU; skips when nvcc is absent.
"""
from __future__ import annotations

import re
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "runbookai_b200" / "csrc"
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

pytestmark = pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")


def _ptxas_report(tmp_path: Path) -> dict[str, str]:
    import importlib.util
    spec = importlib.util.spec_from_file_location("rbk_build", ROOT / "runbookai_b200" / "build.py")
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    cmd = [NVCC, "-Xptxas=-v", *flags, "-c", str(CSRC / "rbk_scan.cu"), "-o", str(tmp_path / "rbk_scan.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    # ptxas prints, per entry: "Compiling entry function '<name>'", "Function properties for <name>",
    # "<n> bytes stack frame, <n> bytes spill stores, <n> bytes spill loads", "Used <n> registers ..."
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


def test_scan_kernel_has_no_spills(tmp_path):
    report = _ptxas_report(tmp_path)
    scans = {name: text for name, text in report.items() if "scan_kernel" in name}
    # top-k' (mode 0), large-k count (mode 1) and emit (mode 2)
    assert sorted(re.search(r"scan_kernelILi(\d)", n).group(1) for n in scans) == ["0", "1", "2"], list(scans)
    for name, text in scans.items():
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
        assert m, (name, text)
        stack, stores, loads = map(int, m.groups())
        assert stores == 0 and loads == 0, (name, text)
        # what may stay on the stack is the compaction's dynamically indexed key array (8 x 8 bytes, rare path)
        assert stack <= 64, (name, text)
        regs = int(re.search(r"Used (\d+) registers", text).group(1))
        assert regs <= 168, (name, text)   # 384 threads, one CTA per SM
