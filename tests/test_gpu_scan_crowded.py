"""GPU suite (-m gpu): the fused scan when many queries have rows above their running threshold in many tiles at
once, in all three epilogue modes (top-k' candidate lists, large-k count, large-k emit), and the scan's raw scores
pinned bit for bit.  Bar, against the oracle: ids identical, fp64 scores bit-identical.
"""
from pathlib import Path

import numpy as np
import pytest

from test_gpu_large_k import check, oracle_bf16
from test_gpu_parity import check_against_oracle

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


@pytest.mark.parametrize("n,d,b,k", [
    (1500, 128, 130, 56),     # 6 tiles: every unit starts without a threshold and has one or two tiles
    (9000, 256, 256, 112),    # two full query blocks, k' = 128 keeps the thresholds low for many tiles
])
def test_no_threshold_small_units(rb, oracle_mod, n, d, b, k):
    """min_score = -inf (findMostSimilar) and few tiles per unit: almost every row of every query passes the filter."""
    from runbookai_b200 import synth
    corpus = synth.random_corpus(n, d, 40 + d)
    q = synth.random_queries(b, d, 41 + d)
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        check_against_oracle(oracle_mod, ix, corpus, q, k, None, nq=b)
        check(ix.search_large(q, 300, None), *oracle_bf16(oracle_mod, corpus, q, 300, None))


def test_all_positive_corpus_d1536(rb, oracle_mod):
    """Cosines crowded in 0.64 .. 1: thresholds stay close to most rows, so most (query, tile) pairs have survivors."""
    from runbookai_b200 import synth
    n, b, d = 6000, 140, 1536
    rng = np.random.Generator(np.random.Philox(4242))
    corpus = synth.f32_to_bf16_bits(np.abs(rng.standard_normal((n, d), dtype=np.float32)) + 0.05)
    corpus[:500] = synth.f32_to_bf16_bits(np.full((500, d), 1.0, np.float32) +
                                          rng.uniform(0, 2 ** -6, (500, d)).astype(np.float32))
    q = synth.bf16_round(np.abs(rng.standard_normal((b, d), dtype=np.float32)) + 0.05)
    q[0] = 1.0
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        for ms in (None, 0.5):
            check_against_oracle(oracle_mod, ix, corpus, q, 32, ms, nq=b)
            check(ix.search_large(q, 1000, ms), *oracle_bf16(oracle_mod, corpus, q, 1000, ms))


def test_tie_group_of_300_rows(rb, oracle_mod):
    """300 identical rows near every query of the batch: each tile holding one of them has survivors for all queries."""
    from runbookai_b200 import synth
    n, d, b = 40_000, 128, 128
    corpus = synth.random_corpus(n, d, 51)
    q = synth.random_queries(b, d, 52)
    centre = q.mean(axis=0)
    q = synth.bf16_round((q * 0.05 + centre).astype(np.float32))
    dup = np.sort(np.random.default_rng(53).choice(n, 300, replace=False))
    corpus[dup] = synth.f32_to_bf16_bits(centre.astype(np.float32))
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        s, _, _ = check_against_oracle(oracle_mod, ix, corpus, q, 20, None, nq=b)
        assert np.isin(s[:, 0], dup).all()
        for k, ms in ((200, None), (500, 0.5)):
            check(ix.search_large(q, k, ms), *oracle_bf16(oracle_mod, corpus, q, k, ms))


def test_debug_scores_bit_identical_to_stored(rb):
    """rbk_index_debug_scores_f32 returns the scan's fp32 scores (accumulator * 1/||c||).  A change to the scan's
    pipeline must not change them by a bit: the fixture holds queries 0-3 and 126-129 (both query blocks) of this
    seeded case as the scan computed them on an H100."""
    from runbookai_b200 import synth
    n, d, b = 3000, 384, 130
    corpus = synth.random_corpus(n, d, 61)
    corpus[17] = 0                                  # zero row -> NaN
    q = synth.random_queries(b, d, 62)
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        got = ix.debug_scores(q)[np.r_[0:4, 126:130]]
    want = np.load(GOLDEN / "scan_debug_scores_f32.npy")
    assert got.shape == want.shape
    assert got.view(np.uint32).tobytes() == want.view(np.uint32).tobytes()
