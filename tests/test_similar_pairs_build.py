"""Build check of the similar-pairs kernels (no GPU needed): the mask, offsets and writer kernels, and the re-score
instantiations they run after (each exact-row type, rows on the device and in host memory), compile for sm_90a
without spills."""
from pathlib import Path

import pytest

from test_search_each_build import NVCC, _one, _ptxas_spills


@pytest.mark.skipif(not Path(NVCC).exists(), reason="nvcc not available")
def test_pairs_kernels_compile_without_spills(tmp_path):
    s = _ptxas_spills(tmp_path, "rbk_finalize.cu")
    for k in ("17pairs_mask_kernel", "20pairs_offsets_kernel", "18pairs_write_kernel"):
        assert _one(s, k) == (0, 0), k
    for k in ("18large_score_kernel", "22large_score_f32_kernel", "24large_score_split_kernel"):
        for host in ("Lb1E", "Lb0E"):
            assert _one(s, k + "I" + host) == (0, 0), (k, host)
