"""CPU suite for the float32 matrix (tests/test_gpu_f32_matrix.py): its float32 exponent ladder against the C oracle
and oracle/pyref.py, as tests/test_float_range_host.py checks float_range_cases for float64, and every corpus builder of
the GPU file against the rules its tiers need - float32-exact rows, no low half of 0x8000 on split and splithost, planted
ones on splitdirty, duplicates that stay duplicates."""
import numpy as np
import pytest

import threshold_cases as tc
from float_range_cases import matches
from oracle import pyref
from test_gpu_f32_matrix import (F32_LADDER, F32_SCALES, F32_SPECIAL, HI_IS_INF, TIERS, all_ties, bound_corpus,
                                 f32_ladder_row, ladder_corpus, prep, rerank_corpus, staging_rows, width_corpus)
from test_gpu_f32_split_rows import low_halves, split_hi
from test_gpu_float_range import in_band
from test_float_range_host import bits

D = 24
TINY = 2.0 ** -126          # the smallest float32 normal


def f32_exact(x):
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        y = x.astype(np.float32).astype(np.float64)
    return bool(((y == x) | (np.isnan(x) & np.isnan(y))).all())


def split_join(s, r):
    """rbk_internal.h split_join, in numpy: the float32 bits joined from a scan copy s and a low half r."""
    s, r = np.asarray(s, dtype=np.uint32), np.asarray(r, dtype=np.uint32)
    return (((s - (r >> 15)) << 16) | r).astype(np.uint32)


@pytest.mark.parametrize("e", sorted(F32_SCALES))
def test_each_rung_is_the_stated_float32_class(oracle_mod, e):
    rng = np.random.default_rng(3000 + e)
    base = rng.standard_normal((40, D))
    x = f32_ladder_row(base[0], e)
    assert f32_exact(x)
    a = np.abs(x[x != 0])
    assert len(a) >= D // 4                    # at 2^-149 about half the elements round to zero
    cls = F32_SCALES[e]
    if cls == "subnormal":
        assert (a < TINY).all()
        assert (np.ldexp(a, 149) == np.round(np.ldexp(a, 149))).all()     # multiples of 2^-149
    elif cls == "mixed":
        assert (a < TINY).any() and (a >= TINY).any()
    else:
        assert (a >= TINY).all() and np.isfinite(x).all() and (a <= np.finfo(np.float32).max).all()
    assert bool(in_band(x)) == (e == 0)
    for partner in base[1:]:
        for u, v in ((x, partner), (partner, x)):
            c = oracle_mod.cosine(u, v)
            assert bits(c) == bits(pyref.cosine_similarity(u.tolist(), v.tolist()))
            assert matches("finite", c), (e, c)


@pytest.mark.parametrize("name", sorted(F32_SPECIAL))
def test_special_rows(oracle_mod, name):
    rng = np.random.default_rng(11)
    x = f32_ladder_row(rng.standard_normal(D), name)
    assert f32_exact(x)
    for p in rng.standard_normal((10, D)):
        for u, v in ((x, p), (p, x)):
            c = oracle_mod.cosine(u, v)
            assert bits(c) == bits(pyref.cosine_similarity(u.tolist(), v.tolist()))
            assert matches(F32_SPECIAL[name], c), (name, c)
    hi = split_hi(x[None, :])[0]
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    finite = ~np.isnan(x)
    assert (split_join(hi, u & 0xFFFF)[finite] == u[finite]).all()     # the split gives every non-NaN value back
    if name in ("f32_max", "hi_is_inf"):
        assert not in_band(x)
        big = np.flatnonzero(np.abs(x) >= HI_IS_INF)
        assert len(big) and ((hi[big] & 0x7FFF) == 0x7F80).all()       # the scan copy is infinite, the value is not


def test_ladder_table_is_the_gpu_ladder():
    assert F32_LADDER == sorted(F32_SCALES) + sorted(F32_SPECIAL)
    assert {-149, -126, 0, 125} <= set(F32_SCALES)


def check_rows(rows, tier, what):
    assert f32_exact(rows), what
    fin = np.isfinite(rows) & (rows != 0)
    ties = (low_halves(rows) == 0x8000) & fin
    if tier == "splitdirty":
        assert ties.sum() > 0.08 * fin.sum(), what
    elif tier.startswith("split"):
        assert not ties.any(), what
    return rows


@pytest.mark.parametrize("tier", list(TIERS))
def test_corpus_builders_store_float32_rows(tier):
    for d in (1, 3, 9, 100):
        _, rows, _, _, wide, _ = width_corpus(d, tier)
        check_rows(rows, tier, f"width d={d}")
        dup = wide[3][0]
        assert (rows[dup] == rows[dup[0]]).all(), f"width d={d}: the tie group stays a tie group"
    for d in (15, 512):
        rows, _ = rerank_corpus(d, tier)
        check_rows(rows, tier, f"rerank d={d}")
    _, rows, _ = ladder_corpus(16, tier, 76)
    n_plain = len(rows) - len(F32_LADDER)
    check_rows(rows[:n_plain], tier, "ladder plain")
    hi = rows[n_plain + F32_LADDER.index("hi_is_inf")]
    assert np.ascontiguousarray(hi[:1], dtype=np.float32).view(np.uint32)[0] == 0x7F7F8000
    assert f32_exact(rows)
    for d in (100,):
        c = tc.tie_corpus(d, False, seed=d)
        rows = check_rows(prep(c["rows"], tier), tier, f"threshold ties d={d}")
        for g in c["dup"]:
            assert (rows[g] == rows[g[0]]).all()
        check_rows(prep(tc.ends_corpus(d, False, seed=d)["rows"], tier), tier, f"ends d={d}")


def test_staging_and_bound_corpora():
    _, rows, over = staging_rows("split")
    assert rows.size > (64 << 20) // 8 and f32_exact(rows) and f32_exact(over)
    assert not (low_halves(rows) == 0x8000).any()
    for kind in ("gaussian", "positive"):
        corpus, q = bound_corpus(768, kind)
        assert f32_exact(corpus) and f32_exact(q)
        assert (low_halves(corpus) == 0x8000).all()
    x = all_ties(np.array([[1.0, -0.0, 0.0, np.inf, 3.0]]))
    assert np.isinf(x[0, 3]) and x[0, 1] == 0 and np.signbit(x[0, 1])
