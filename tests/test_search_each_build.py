"""Build check of the per-query kernels of rbk_index_search_each_f64 (no GPU needed): every one of them compiles for
sm_90a and spills no more than the scalar kernel it was made from."""
import importlib.util
import re
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
NVCC = "/usr/local/cuda/bin/nvcc"


def _ptxas_spills(tmp_path, source):
    """{mangled kernel name: (spill store bytes, spill load bytes)} from -Xptxas -v with the library's flags."""
    spec = importlib.util.spec_from_file_location("rbk_build", ROOT / "runbookai_b200" / "build.py")
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    res = subprocess.run([NVCC, "-Xptxas=-v", *flags, "-c", str(ROOT / "runbookai_b200" / "csrc" / source), "-o",
                          str(tmp_path / "k.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    out, current = {}, None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current is not None:
            out[current] = (int(m.group(1)), int(m.group(2)))
            current = None
    return out


def _one(spills, pattern):
    hit = [v for n, v in spills.items() if re.search(pattern, n)]
    assert len(hit) == 1, (pattern, [n for n in spills if re.search(pattern, n)])
    return hit[0]


@pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")
def test_per_query_kernels_spill_no_more_than_their_scalar_twins(tmp_path):
    s = _ptxas_spills(tmp_path, "rbk_finalize.cu")
    pairs = []
    for host in (0, 1):
        for width, twin in ((8, r"15finalize_kernel"), (4, r"19finalize_f32_kernel"), (2, r"21finalize_split_kernel")):
            pairs.append((rf"20finalize_each_kernelILb{host}ELi{width}E", rf"{twin}ILb{host}E"))
    for width, xt in ((8, "d"), (4, "f"), (2, "NS_5F32LoE")):
        pairs.append((rf"22exact_scan_each_kernelILi{width}E", rf"17exact_scan_kernelI{xt}E"))
    for norm2 in (0, 1):
        for f16 in (0, 1):
            pairs.append((rf"19prep_queries_kernelIdLb{norm2}ELb{f16}ELb1E", rf"19prep_queries_kernelIdLb{norm2}ELb{f16}ELb0E"))
    pairs.append((r"16seg_merge_kernelILb1E", r"16seg_merge_kernelILb0E"))
    for each, scalar in pairs:
        e, t = _one(s, each), _one(s, scalar)
        assert e[0] <= t[0] and e[1] <= t[1], (each, e, scalar, t)
