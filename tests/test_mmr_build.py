"""Build check of the MMR selection kernel of rbk_index_search_mmr_f64 (no GPU needed): it compiles for sm_90a without
spills."""
from pathlib import Path

import pytest

from test_search_each_build import NVCC, _one, _ptxas_spills


@pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")
def test_mmr_select_kernel_compiles_without_spills(tmp_path):
    s = _ptxas_spills(tmp_path, "rbk_mmr.cu")
    assert _one(s, r"17mmr_select_kernel") == (0, 0)
