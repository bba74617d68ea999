"""Build check of the gather kernel of rbk_index_search_slots_f64 (no GPU needed): each of its four instantiations -
float64, float32 and split exact rows, and bf16 rows alone - compiles for sm_90a without spills."""
from pathlib import Path

import pytest

from test_search_each_build import NVCC, _one, _ptxas_spills


@pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")
def test_gather_kernel_compiles_without_spills(tmp_path):
    s = _ptxas_spills(tmp_path, "rbk_gather.cu")
    for xt in ("d", "f", "NS_5F32LoE", "t"):
        assert _one(s, rf"18gather_rows_kernelI{xt}E") == (0, 0), xt
