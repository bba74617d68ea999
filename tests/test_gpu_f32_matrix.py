"""GPU suite (-m gpu): float32 exact rows (RBK_INDEX_KEEP_F32, x_elem 4) and split float32 exact rows
(RBK_INDEX_KEEP_F32_SPLIT, x_elem 2) through the oracle matrices the float64 tiers run: widths from 1 to 65536, the
host-staged and large-k re-rank chunks, the float32 exponent range, the scan bound under the split's rounding, min_score
cuts, the exhaustive kernel and the retry, chunked host staging and unaligned device sources, tier changes where the
scan pitch dpad differs from d, growth and groups.

Tiers (TIERS): f32, f32host, f32f16, split, splithost, and splitdirty - split rows with a low half of 0x8000 in one
element in eight, which the split's scan copy rounds away from zero where a float64 twin's rounds to even.  Every corpus
is float32-exact (prep) and the oracle scores those float32 rows.  Where a KEEP_F64 twin with the same placement and
scan is cheap, every output and stats counter must equal the twin's (the answers only, for splitdirty).

Bar: ids, counts and float64 score bytes equal to the oracle's; every case built to reach the retry or the exhaustive
kernel asserts through stats() that it did.  Run with -s to see, per width and tier, the largest ratio of scan error to
its bound, which path answered at d = 65536, and the module's wall time."""
import time

import numpy as np
import pytest

import threshold_cases as tc
from common import group_devices
from float_range_cases import SCALES, scaled
from test_gpu_compact import assert_same_through_map, expected_map
from test_gpu_exact_paths import (CASES, WIDE_ABOVE, check, counters, group_scores, mismatches, oracle_answers,
                                  sweep_corpus, tie_corpus, tie_queries)
from test_gpu_f32_rows import answers, assert_same_answers, f32x, same
from test_gpu_f32_split_rows import assert_same_answers_only, low_halves, retie, split_hi
from test_gpu_float_range import all_routes, in_band
from test_gpu_group_compact import bit_equal, member_rows, routes, runs_dead
from test_gpu_group_members import append_in_pieces, check_members, member_slots
from test_gpu_scan_f16 import acc_eps, bf16_angle, bits_to_f64, f16_angle
from test_gpu_thresholds import Oracle, band_thresholds, check_exact_scores, compare, every_route, stats_line
from test_gpu_widths import BATCHES, K, batch_pool, extreme_routes, route_corpus

pytestmark = pytest.mark.gpu

KEEP64, HOST, F16, KEEP32, SPLIT = 1, 2, 16, 64, 128
TIERS = {"f32": KEEP32, "f32host": KEEP32 | HOST, "f32f16": KEEP32 | F16, "split": SPLIT, "splithost": SPLIT | HOST,
         "splitdirty": SPLIT}
WIDTHS = [1, 3, 7, 9, 100, 511, 513, 1025, 2049, 4095, 4096, 16384]
FLT_MAX = float(np.finfo(np.float32).max)
HI_IS_INF = float(np.uint32(0x7F7F8000).view(np.float32))     # finite; its split scan copy (and its RNE bf16) is +inf

# The float32 exponent ladder: exponent -> what rounding a standard-normal row scaled by 2^e to float32 leaves.  Against
# an ordinary float64 partner every rung scores a finite cosine (float64 squares neither underflow nor overflow here);
# only the e = 0 rung lies inside the scan's band [2^-40, 2^40), so the others send every query to the exhaustive kernel.
F32_SCALES = {
    -149: "subnormal",      # multiples of 2^-149, the smallest float32 subnormal: most elements become 0 or +-2^-149
    -140: "subnormal",
    -134: "subnormal",
    -133: "subnormal",      # every element below 2^-126 as long as |z| < 2^7
    -127: "mixed",          # elements on both sides of 2^-126, the smallest float32 normal
    -126: "mixed",
    -100: "normal",
    -60: "normal",
    0: "normal",
    60: "normal",
    100: "normal",
    125: "normal",          # below float32 max as long as |z| < 8
}
# special rows -> the kind of cosine an ordinary partner gives them
F32_SPECIAL = {"f32_max": "finite", "hi_is_inf": "finite", "one_nan": "nan", "one_inf": "nan", "one_neg_inf": "nan",
               "neg_zero": "nan"}
F32_LADDER = sorted(F32_SCALES) + sorted(F32_SPECIAL)

RATIOS = {}                # (what, tier, d) -> largest |scan - exact| / eps_q
PATHS = {}                 # (d, tier) -> (retry batches, fallback queries) of one top-k search


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


@pytest.fixture(scope="module", autouse=True)
def report(rb):
    t0 = time.perf_counter()
    yield
    print("\nscan error / eps_q, largest seen:")
    for key in sorted(RATIOS, key=str):
        print(f"  {key}: {RATIOS[key]:.4f}")
    print("paths at d = 65536 (retry batches, fallback queries of one 3-query search):")
    for key in sorted(PATHS):
        print(f"  {key}: {PATHS[key]}")
    print(f"module wall time: {time.perf_counter() - t0:.1f} s")


def make(rb, d, flags, cls=None, devices=None, cap=0):
    kw = dict(capacity_hint=cap, keep_f64=bool(flags & KEEP64), keep_f32=bool(flags & KEEP32),
              keep_f32_split=bool(flags & SPLIT), f64_on_host=bool(flags & HOST), scan_f16=bool(flags & F16))
    return rb.Group(d, devices, **kw) if cls is rb.Group else rb.Index(d, **kw)


def twin_flags(flags):
    """The KEEP_F64 tier with the same placement and scan."""
    return (flags & (HOST | F16)) | KEEP64


def exact_name(flags):
    return "f64" if flags & KEEP64 else ("f32" if flags & KEEP32 else "f32_split")


def plant_ties(rows):
    """float32-exact rows with a low half of 0x8000 in every element of columns 3 mod 8 (column 0 when d <= 3), zeros
    and non-finite values left alone.  retie(..., True) plants by flat position; planting by column keeps exact
    duplicate rows duplicates at every d."""
    u = np.ascontiguousarray(rows, dtype=np.float32).view(np.uint32).copy()
    first = 3 if u.shape[-1] > 3 else 0
    pick = np.zeros(u.shape, bool)
    pick[..., first::8] = True
    pick &= np.isfinite(rows) & (rows != 0)
    u[pick] = (u[pick] & 0xFFFF0000) | 0x8000
    return u.view(np.float32).astype(np.float64)


def prep(rows, tier):
    """The float32-exact rows a tier stores: for split and splithost with no low half of exactly 0x8000 (so that the
    scan copy equals the float64 twin's and every counter must match), for splitdirty with planted ones."""
    rows = f32x(rows)
    if not tier.startswith("split"):
        return rows
    keep = ~np.isfinite(rows) | (rows == 0)
    out = retie(rows, False)
    out[keep] = rows[keep]
    return plant_ties(out) if tier == "splitdirty" else out


def all_ties(rows):
    """Every nonzero finite element's low half set to 0x8000: the split's scan copy rounds each one away from zero."""
    u = np.ascontiguousarray(rows, dtype=np.float32).view(np.uint32).copy()
    pick = np.isfinite(rows) & (rows != 0)
    u[pick] = (u[pick] & 0xFFFF0000) | 0x8000
    return u.view(np.float32).astype(np.float64)


def rne_hi(rows):
    """The bf16 scan copy of a float32 or float64 tier: round to nearest, ties to even."""
    from runbookai_b200 import synth
    with np.errstate(over="ignore"):
        return synth.f32_to_bf16_bits(np.asarray(rows, dtype=np.float64).astype(np.float32))


def scan_angle(rows, hi):
    """asin(||x - scan copy|| / ||x||) per row, from the scan copy the index holds (0 for a zero row)."""
    x = np.atleast_2d(rows)
    n = np.linalg.norm(x, axis=1)
    r = np.linalg.norm(x - bits_to_f64(hi), axis=1) / np.where(n > 0, n, 1.0)
    return np.arcsin(np.minimum(r, 1.0))


def scan_eps(ix, rows, q, flags, mask=None):
    """eps_q as the proof computes it, with the corpus angle of the index's own scan copy over the rows mask keeps."""
    d = rows.shape[1]
    mask = np.ones(len(rows), bool) if mask is None else mask
    if flags & F16:
        return acc_eps(d) + f16_angle(q) + f16_angle(rows[mask]).max()
    return acc_eps(d) + bf16_angle(q) + scan_angle(rows[mask], ix.read_rows_bf16(0, ix.size())[mask]).max()


def bound_ratio(ix, rows, live, q, flags, key):
    """debug_scores within eps_q over the live nonzero rows; records the largest error / bound ratio under key."""
    q = f32x(q)
    live_rows = (np.asarray(live) != 0) & (np.linalg.norm(rows, axis=1) > 0)
    if not live_rows.any():
        return
    eps = scan_eps(ix, rows, q, flags, live_rows)
    got = ix.debug_scores(q.astype(np.float32)).astype(np.float64)[:, live_rows]
    ref = (q @ rows[live_rows].T) / (np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(rows[live_rows], axis=1))
    ratio = np.abs(got - ref) / eps[:, None]
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(ratio.max()))
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert (ratio <= 1.0).all(), (key, worst, ratio[worst])


def twins_agree(ix, twin, q, tier, skip=()):
    """Every output and counter of answers() equal to the twin's; for splitdirty, whose scan copy differs from the
    twin's, only the slots, scores and counts of each route (not the scan's debug scores, exactness flags or counters)."""
    a, b = answers(ix, q), answers(twin, q)
    dirty = tier == "splitdirty"
    for key in a:
        if key in skip or (dirty and key in ("debug", "async")):   # async: the first pass's own answers
            continue
        x, y = (a[key][:-1][:3], b[key][:-1][:3]) if dirty else (a[key], b[key])
        assert len(x) == len(y) and all((u == v) if isinstance(u, tuple) else same(u, v) for u, v in zip(x, y)), key


# --------------------------------------------------------------------------- 1. every route at every width
def width_corpus(d, tier):
    rng, rows, live, q, wide, narrow = route_corpus(d, d)
    return rng, prep(rows, tier), live, q, wide, narrow


@pytest.mark.parametrize("tier", list(TIERS))
@pytest.mark.parametrize("d", WIDTHS)
def test_every_route_at_every_width(rb, oracle_mod, d, tier):
    flags = TIERS[tier]
    rng, rows, live, q, wide, narrow = width_corpus(d, tier)
    dead = np.flatnonzero(live == 0)
    with make(rb, d, flags) as ix, make(rb, d, twin_flags(flags)) as twin:
        for h in (ix, twin):
            h.append_f64(rows)
            h.tombstone(dead)
        if flags & SPLIT:
            assert same(ix.read_rows_bf16(0, ix.size()), split_hi(rows))
        bound_ratio(ix, rows, live, q, flags, ("width", tier, d))
        all_routes(oracle_mod, ix, rows, live, q, f"{tier} d={d}")

        # descending batches: every key_cap tier, the retry in each, and smaller batches over stale query-pad rows
        pool = batch_pool(rng, d, wide, narrow)
        want = oracle_answers(oracle_mod, rows, live, pool, K, None)
        for B, off in BATCHES:
            sl = slice(off, off + B)
            r0, f0 = counters(ix)
            got = ix.search(pool[sl], K, None)
            r1, f1 = counters(ix)
            what = f"{tier} d={d} B={B}"
            bad = mismatches(got[:3], tuple(w[sl] for w in want))
            assert not bad, f"{what}: {len(bad)} of {B} queries differ from the oracle: {bad[:10]}"
            if 1 < d < 2049:
                continue             # at d = 2..7 random rows crowd the top ranks: which path answers is not fixed
            n_wide = int((np.arange(off, off + B) % 5 == 0).sum())
            assert r1 > r0, f"{what}: every batch holds a narrow tie group's query, which needs the retry"
            assert f1 - f0 >= n_wide, f"{what}: {f1 - f0} fell back, {n_wide} queries have a tie group wider than 128"
            if B == 1 and d > 1:
                assert f1 == f0, f"{what}: the retry holds a 60-row tie group"
        if d <= 1025 or not flags & HOST:     # wider, the host twins' exhaustive re-answers cost minutes over PCIe
            twins_agree(ix, twin, pool, tier)


@pytest.mark.parametrize("tier", ["split", "f32host"])
def test_every_route_at_65536(rb, oracle_mod, tier):
    """At d = 65536 the scan's bound is wider than the spread of random top scores: record which path answered, and
    check every route."""
    d, n = 65536, 200
    rng = np.random.default_rng(65536)
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((3, d))
    rows[[5, 50, 150]] = q + 0.5 * rng.standard_normal((3, d))
    rows = prep(rows, tier)
    flags = TIERS[tier]
    with make(rb, d, flags) as ix, make(rb, d, twin_flags(flags)) as twin:
        for h in (ix, twin):
            h.append_f64(rows)
        r0, f0 = counters(ix)
        ix.search(q, 10, None)
        r1, f1 = counters(ix)
        PATHS[(d, tier)] = (r1 - r0, f1 - f0)
        extreme_routes(oracle_mod, ix, rows, q, f"{tier} d={d}")
        got = {(k, "top"): ix.search(q, k, None)[:3] for k in (10, 112)}
        got.update({(k, "large"): ix.search_large(q, k, 0.0)[:3] for k in (200, 4096)})
        got[(n + 7, "unbounded")] = ix.search_unbounded(q, n + 7, None)[:3]
        want = {(k, "top"): twin.search(q, k, None)[:3] for k in (10, 112)}
        want.update({(k, "large"): twin.search_large(q, k, 0.0)[:3] for k in (200, 4096)})
        want[(n + 7, "unbounded")] = twin.search_unbounded(q, n + 7, None)[:3]
        assert bit_equal(got, want), f"{tier} d={d}: the float64 twin answers otherwise"
        assert ix.exact_scores(q).tobytes() == twin.exact_scores(q).tobytes()


# --------------------------------------------------------------------------- 2. host-staged and large-k re-rank chunks
RERANK_WIDTHS = [15, 16, 17, 31, 33, 511, 512, 513]


def rerank_corpus(d, tier):
    """3000 random rows and two groups of 100 duplicates (held by the retry's k' = 128, so a k_fetch 112 selection is
    128 candidates wide), 3 and 20 rows above them; 8 tie queries and 1092 random ones."""
    rng = np.random.default_rng(500 + d)
    rows, tq, _, _ = tie_corpus(rng, d, 3000, above=[3, 20], group_size=100, q_per_group=4)
    q = np.concatenate([tq, rng.standard_normal((1092, d))])
    return prep(rows, tier), q


@pytest.mark.parametrize("tier", ["f32host", "splithost"])
@pytest.mark.parametrize("d", RERANK_WIDTHS)
def test_host_staged_rerank_chunks(rb, oracle_mod, d, tier):
    """k_fetch 112 at B = 8, 300 and 1100 (key_cap 16384, 8192 and 2048: host re-rank chunks of 126, 62 and 14
    elements), search_large at 700 and 4096 (16-element staged pieces) and search_unbounded: bit for bit the
    device-placement twin's, and the oracle's.  B = 500 also has key_cap 2048."""
    flags = TIERS[tier]
    rows, q = rerank_corpus(d, tier)
    with make(rb, d, flags) as ix, make(rb, d, flags & ~HOST) as dev:
        for h in (ix, dev):
            h.append_f64(rows)
        for B in (8, 300, 500, 1100):
            for ms in (None, 0.0):
                got = ix.search(q[:B], 112, ms)[:3]
                assert bit_equal({0: got}, {0: dev.search(q[:B], 112, ms)[:3]}), (tier, d, B, ms)
                check(oracle_mod, got, rows, None, q[:B], 112, ms, f"{tier} d={d} B={B} k=112 min_score={ms}")
        for k, ms in ((700, None), (4096, 0.0)):
            got = ix.search_large(q[:8], k, ms)[:3]
            assert bit_equal({0: got}, {0: dev.search_large(q[:8], k, ms)[:3]}), (tier, d, k)
            check(oracle_mod, got, rows, None, q[:8], k, ms, f"{tier} d={d} search_large {k}")
        got = ix.search_unbounded(q[:4], 5000, None)[:3]
        assert bit_equal({0: got}, {0: dev.search_unbounded(q[:4], 5000, None)[:3]}), (tier, d, "unbounded")
        check(oracle_mod, got, rows, None, q[:4], 5000, None, f"{tier} d={d} search_unbounded")
        assert ix.exact_scores(q[:3]).tobytes() == dev.exact_scores(q[:3]).tobytes()


# Most queries of a 1024-query batch at k_fetch 112 fall back to the exhaustive kernel, whose merge pushes 13 x 112
# partial hits through a 1024-entry buffer: the case that found a block-wide barrier taken by only some threads
# (DESIGN.md §7).
@pytest.mark.parametrize("flags", [KEEP64, KEEP64 | HOST, KEEP32, KEEP32 | HOST, SPLIT, SPLIT | HOST])
@pytest.mark.parametrize("d", [511, 512])
def test_large_batches_at_k112(rb, oracle_mod, d, flags):
    rows, q = rerank_corpus(d, "f32host")
    with make(rb, d, flags) as ix:
        ix.append_f64(rows)
        for B in (500, 1024, 1100):
            _, f0 = counters(ix)
            got = ix.search(q[:B], 112, None)
            assert counters(ix)[1] - f0 > B // 2, "most queries were meant to reach the exhaustive kernel"
            check(oracle_mod, got, rows, None, q[:B], 112, None, f"flags {flags} d={d} B={B}")


# --------------------------------------------------------------------------- 3. the float32 exponent range
def f32_ladder_row(v, key):
    """A float32-exact row from the standard-normal row v: scaled by 2^key and rounded to float32 (so the subnormal
    rungs really are float32 subnormals), or one of the special rows."""
    if not isinstance(key, str):
        return f32x(scaled(v, key))
    v = f32x(v)
    if key == "f32_max":
        v = np.where(v < 0, -FLT_MAX, FLT_MAX)
    elif key == "hi_is_inf":
        v[0] = HI_IS_INF
    elif key == "one_nan":
        v[len(v) // 2] = np.nan
    elif key == "one_inf":
        v[len(v) // 3] = np.inf
    elif key == "one_neg_inf":
        v[len(v) // 3] = -np.inf
    elif key == "neg_zero":
        v[:] = -0.0
    return v


def ladder_corpus(d, tier, seed, n_plain=3000):
    """Ordinary rows plus one row per rung of F32_LADDER, each near one of 8 queries.  The specials are made after
    prep, so the 0x7F7F8000 element keeps its low half on every tier."""
    rng = np.random.default_rng(seed)
    plain = rng.standard_normal((n_plain, d))
    q = plain[rng.choice(n_plain, 8)] + 0.1 * rng.standard_normal((8, d))
    near = q[np.arange(len(F32_LADDER)) % 8] + 0.05 * rng.standard_normal((len(F32_LADDER), d))
    rungs = np.stack([f32_ladder_row(near[i], e) for i, e in enumerate(sorted(F32_SCALES))])
    specials = np.stack([f32_ladder_row(near[len(F32_SCALES) + i], s) for i, s in enumerate(sorted(F32_SPECIAL))])
    rows = np.concatenate([prep(plain, tier), prep(rungs, tier), specials])
    return rng, rows, q


@pytest.mark.parametrize("d,tier", [(16, t) for t in TIERS] + [(513, "split"), (513, "splitdirty")])
def test_row_ladder(rb, oracle_mod, d, tier):
    """Rows across the float32 range and special rows: the rungs outside the scan's band send every query to the
    exhaustive kernel; every route is the oracle's and, on every tier but splitdirty, every output and counter the
    float64 twin's.  Tombstoning the ladder gives the plain corpus's answers."""
    flags = TIERS[tier]
    rng, rows, q = ladder_corpus(d, tier, 60 + d)
    n_plain = len(rows) - len(F32_LADDER)
    with make(rb, d, flags) as ix, make(rb, d, twin_flags(flags)) as twin:
        for h in (ix, twin):
            h.append_f64(rows)
        if flags & SPLIT:
            bits = ix.read_rows_bf16(0, ix.size())
            assert same(bits, split_hi(rows))
            assert bits[n_plain + F32_LADDER.index("hi_is_inf"), 0] == 0x7F80
        _, f0 = counters(ix)
        ix.search(q, 10, None)
        _, f1 = counters(ix)
        assert f1 - f0 == len(q), f"{tier}: rows outside the scan's band must send every query to the fallback"
        all_routes(oracle_mod, ix, rows, None, q, f"{tier} d={d} float32 row ladder")
        pool = np.concatenate([q, rng.standard_normal((192, d))])
        # a row holding a NaN scores NaN under a payload of its exact width: exact_scores is checked against the
        # oracle above, every NaN one value
        twins_agree(ix, twin, pool, tier, skip=("exact",) if flags & SPLIT else ())
        live = np.ones(len(rows), np.uint8)
        live[n_plain:] = 0
        ix.tombstone(np.flatnonzero(live == 0))
        for ms in (None, 0.0, 0.5):
            check(oracle_mod, ix.search(q, 10, ms), rows, live, q, 10, ms, f"{tier} d={d} ladder tombstoned")
        check(oracle_mod, ix.search_large(q, 200, None), rows, live, q, 200, None, f"{tier} d={d} tombstoned large")


@pytest.mark.parametrize("tier", list(TIERS))
def test_query_ladder(rb, oracle_mod, tier):
    """Ordinary float32 rows; each query a row plus noise scaled by one rung of float_range_cases.SCALES.  Queries past
    the scan's band reach the exhaustive kernel."""
    d = 100
    rng = np.random.default_rng(77)
    rows = prep(rng.standard_normal((3000, d)), tier)
    es = sorted(SCALES)
    base = rows[rng.choice(len(rows), len(es))] + 0.1 * rng.standard_normal((len(es), d))
    q = np.stack([scaled(base[i], e) for i, e in enumerate(es)])
    with make(rb, d, TIERS[tier]) as ix:
        ix.append_f64(rows)
        _, f0 = counters(ix)
        ix.search(q, 10, None)
        _, f1 = counters(ix)
        n_out = int((~in_band(q)).sum())
        assert f1 - f0 >= n_out, f"{tier}: {f1 - f0} queries fell back, {n_out} are outside the scan's band"
        all_routes(oracle_mod, ix, rows, None, q, f"{tier} query ladder")


# --------------------------------------------------------------------------- 4. the scan bound under the split rounding
BOUND_WIDTHS = [768, 1536, 2048, 4096, 16384]


def bound_corpus(d, kind):
    """2000 rows whose every low half is 0x8000 (gaussian, or positive, where the truncation errors of the scan's
    accumulator do not cancel) and 16 float32 queries, one of them close to a row."""
    n, b = 2000, 16
    rng = np.random.default_rng(d + (kind == "positive"))
    if kind == "gaussian":
        corpus, q = rng.standard_normal((n, d)), rng.standard_normal((b, d))
    else:
        corpus = np.abs(rng.standard_normal((n, d))) + 0.05
        q = np.abs(rng.standard_normal((b, d))) + 0.05
        q[0] = 1.0
    corpus = all_ties(corpus)
    q[1] = corpus[17] * (1.0 + 2.0 ** -12 * rng.standard_normal(d))
    return corpus, f32x(q)


@pytest.mark.parametrize("kind", ["gaussian", "positive"])
@pytest.mark.parametrize("tier", ["split", "f32"])
@pytest.mark.parametrize("d", BOUND_WIDTHS)
def test_scan_bound_under_the_split_rounding(rb, d, tier, kind):
    """debug_scores within eps_q = (d+8) 2^-22 + angle(q, bf16 q) + the largest angle between a row and the scan copy
    read_rows_bf16 returns.  The split's copy rounds every element away from zero; the f32 tier's rounds the same
    rows to even, so the two differ only in the scan copy."""
    corpus, q = bound_corpus(d, kind)
    assert (low_halves(corpus) == 0x8000).all()
    with make(rb, d, TIERS[tier]) as ix:
        ix.append_f64(corpus)
        hi = ix.read_rows_bf16(0, ix.size())
        assert same(hi, split_hi(corpus) if tier == "split" else rne_hi(corpus))
        if tier == "split":
            assert (hi != rne_hi(corpus)).mean() > 0.4    # ties to even keep about half of them where they were
        bound_ratio(ix, corpus, np.ones(len(corpus)), q, TIERS[tier], ("bound " + kind, tier, d))


# --------------------------------------------------------------------------- 5. min_score cuts
CUT_TIERS = ("f32", "split", "splithost", "splitdirty")


@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", CUT_TIERS)
def test_band_ladder(rb, oracle_mod, tier, d):
    """Four queries with rows spread over their band; the thresholds come from the oracle's scores of the stored
    float32 rows, and hundreds of live rows lie within the index's own eps_q of each band centre."""
    flags = TIERS[tier]
    c = tc.band_corpus(d, False, seed=10 + d)
    rows = prep(c["rows"], tier)
    with make(rb, d, flags) as ix:
        ix.append_f64(rows)
        eps = scan_eps(ix, rows, c["q"], flags)
        orc = Oracle(oracle_mod, rows)
        for i, q in enumerate(c["q"]):
            assert int((np.abs(orc.scores(q) - c["t"][i]) <= eps[i]).sum()) >= 100, (i, eps[i])
        ths = band_thresholds(orc, c)
        for i, ms in enumerate(ths):
            every_route(orc, ix, c["q"], ms, f"{tier} d={d} band", general=not flags & HOST or i % 5 == 0)
        check_exact_scores(orc, ix, c["q"], ths, f"{tier} d={d}")
        print(f"{tier} d={d}: {len(ths)} thresholds, {stats_line(ix)}")


@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", CUT_TIERS)
def test_tie_group_on_the_threshold(rb, oracle_mod, tier, d):
    """5, 70 and 150 duplicates whose common score (the oracle's, over the float32 rows) is min_score: a k_fetch inside
    the group takes the retry for 70 and the exhaustive kernel for 150; one ulp above drops the group."""
    c = tc.tie_corpus(d, False, seed=d)
    rows = prep(c["rows"], tier)
    with make(rb, d, TIERS[tier]) as ix:
        ix.append_f64(rows)
        orc = Oracle(oracle_mod, rows)
        for g, size in enumerate(c["sizes"]):
            dup = c["dup"][g]
            assert (rows[dup] == rows[dup[0]]).all()
            q1 = c["q"][g:g + 1]
            ms = float(orc.scores(q1[0])[dup[0]])
            what = f"{tier} d={d} group of {size}"
            k_cut = c["above"] + size // 2
            r0, f0 = counters(ix)
            compare(orc, ix.search(q1, k_cut, ms), q1, k_cut, ms, f"{what} [{stats_line(ix)}] cut inside")
            r1, f1 = counters(ix)
            if size == 150:
                assert f1 > f0, f"{what}: the group is wider than k' = 128 (retries {r1 - r0}, fallback {f1 - f0})"
            if size == 70:
                assert r1 > r0 and f1 == f0, f"{what}: k' = 128 holds the group (retries {r1 - r0}, fallback {f1 - f0})"
            k_past = c["above"] + size + 10
            got = ix.search(q1, k_past, ms) if k_past <= 112 else ix.search_large(q1, k_past, ms)
            compare(orc, got, q1, k_past, ms, f"{what} [{stats_line(ix)}] count < k_fetch")
            up = float(np.nextafter(ms, np.inf))
            got = ix.search(q1, k_cut, up)
            compare(orc, got, q1, k_cut, up, f"{what} one ulp above")
            assert not np.isin(got[0][0, :got[2][0]], dup).any(), f"{what}: one ulp above must drop the group"
            for m in (ms, up, float(np.nextafter(ms, -np.inf))):
                every_route(orc, ix, c["q"], m, what)


@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", CUT_TIERS)
def test_ends_and_extreme_thresholds(rb, oracle_mod, tier, d):
    """Multiples of each query (scores 1 / -1 or one ulp off), rows scoring +0, zero rows, tombstoned multiples on the
    thresholds; every threshold of the fixed ladder and of the ends."""
    c = tc.ends_corpus(d, False, seed=d)
    rows = prep(c["rows"], tier)
    live = np.ones(len(rows), np.uint8)
    dead = c["multiples"][::4]
    with make(rb, d, TIERS[tier]) as ix:
        ix.append_f64(rows)
        ix.tombstone(dead)
        live[dead] = 0
        orc = Oracle(oracle_mod, rows, live)
        ths = set()
        for q in c["q"]:
            ths |= {np.float64(v).tobytes() for v in tc.ends_ladder(oracle_mod.scores(rows, q))}
        ths = [float(np.frombuffer(b)[0]) for b in sorted(ths)]
        for ms in ths:
            every_route(orc, ix, c["q"], ms, f"{tier} d={d} ends")
        check_exact_scores(orc, ix, c["q"], ths, f"{tier} d={d} ends")


# --------------------------------------------------------------------------- 6. the exhaustive kernel and the retry
EXACT_TIERS = ("f32", "split", "splithost")


@pytest.mark.parametrize("d", [1001, 1024])
@pytest.mark.parametrize("tier", EXACT_TIERS)
@pytest.mark.parametrize("n_rand,above", [(60, [0]), (4853, [0, 7]), (67460, [0, 7])])
def test_fallback_block_split(rb, oracle_mod, tier, d, n_rand, above):
    """The exhaustive scan's row blocks: one block below 256 rows, and row counts that leave the last block short."""
    rng = np.random.default_rng(n_rand + d)
    rows, q, _, _ = tie_corpus(rng, d, n_rand, above=above, group_size=150, q_per_group=4)
    rows = prep(rows, tier)
    with make(rb, d, TIERS[tier]) as ix:
        ix.append_f64(rows)
        _, f0 = counters(ix)
        got = ix.search(q, 20, None)
        check(oracle_mod, got, rows, None, q, 20, None, f"{tier} d={d} n={len(rows)}")
        assert counters(ix)[1] - f0 == len(q)


@pytest.mark.parametrize("d", [1001, 1024])
@pytest.mark.parametrize("tier", EXACT_TIERS)
def test_retry_and_fallback_sweep(rb, oracle_mod, tier, d):
    """test_gpu_exact_paths's sweep (launch shapes, k_fetch, min_score in the tie band, tombstones, compaction) on
    float32 rows."""
    rng, rows, wide, narrow = sweep_corpus(d, 100 + d)
    rows = prep(rows, tier)
    live = np.ones(len(rows), np.uint8)
    with make(rb, d, TIERS[tier]) as ix:
        ix.append_f64(rows)
        for phase in ("whole", "tombstoned", "compacted"):
            if phase == "tombstoned":
                dead = np.concatenate([s[::10] for s in wide[3]] + [rng.choice(2000, 50, replace=False)])
                ix.tombstone(dead)
                live[dead] = 0
            if phase == "compacted":
                old_to_new = ix.compact()
                keep = live.astype(bool)
                assert (old_to_new[keep] == np.arange(keep.sum())).all()
                rows_now = rows[keep]
                remap = lambda src: (src[0], src[1], src[2], [old_to_new[s][old_to_new[s] >= 0] for s in src[3]])
                wide_now, narrow_now, lv = remap(wide), remap(narrow), None
            else:
                rows_now, wide_now, narrow_now, lv = rows, wide, narrow, live
            for B, k, ms in CASES:
                for kind in ("wide", "narrow") if (B, k) == (64, 20) else ("wide",):
                    src = wide_now if kind == "wide" else narrow_now
                    q, groups = tie_queries(rng, d, src, B)
                    m = float(np.median(group_scores(rows_now, src, q[B - len(groups):], groups))) if ms == "band" else ms
                    r0, f0 = counters(ix)
                    got = ix.search(q, k, m)
                    r1, f1 = counters(ix)
                    what = f"{tier} d={d} {phase} B={B} k={k} min_score={m} {kind}"
                    check(oracle_mod, got, rows_now, lv, q, k, m, what)
                    if kind == "narrow":
                        assert r1 - r0 == 1 and f1 == f0, what
                    elif ms != "band":
                        above = np.array(WIDE_ABOVE)[groups]
                        assert f1 - f0 >= int((above < k).sum()) > 0, what
                    else:
                        assert f1 - f0 >= 1, what


# --------------------------------------------------------------------------- 7. chunked host staging and alignment
STAGE_ELEMS = (64 << 20) // 8          # float64 values per 64 MB host staging chunk


def staging_rows(tier):
    """6000 x 1536 float64 values (73.7 MB: two staging chunks) to append, and as many to overwrite them with."""
    rng = np.random.default_rng(6000)
    d = 1536
    rows = prep(rng.standard_normal((6000, d)), tier)
    over = prep(rng.standard_normal((6000, d)), tier)
    return rng, rows, over


def state(ix, q):
    return (ix.size(), ix.count(), ix.storage_bytes(), ix.search(q, 20, None)[:3], ix.exact_scores(q[:2]),
            ix.read_rows_bf16(0, ix.size()))


def assert_same_state(a, b):
    assert a[:3] == b[:3]
    assert all(same(x, y) for x, y in zip(a[3], b[3]))
    assert same(a[4], b[4]) and same(a[5], b[5])


@pytest.mark.parametrize("tier", ["f32", "split"])
def test_chunked_host_staging(rb, oracle_mod, tier):
    """append_f64 and overwrite_f64_batch of float64 sources larger than one staging chunk equal the float64 twin's;
    a value that is not a float32 at the first element of the second chunk, or at the last element, is refused with
    nothing changed."""
    from runbookai_b200._native import NotFloat32Error
    rng, rows, over = staging_rows(tier)
    n, d = rows.shape
    assert rows.size > STAGE_ELEMS
    slots = rng.permutation(n)
    corpus = rows.copy()
    corpus[slots] = over
    q = corpus[rng.choice(n, 200)] + 0.1 * rng.standard_normal((200, d))
    flags = TIERS[tier]
    with make(rb, d, flags) as ix, make(rb, d, twin_flags(flags)) as twin:
        for h in (ix, twin):
            h.append_f64(rows)
        assert same(ix.read_rows_bf16(0, n), twin.read_rows_bf16(0, n))
        for h in (ix, twin):
            h.overwrite_f64_batch(slots, over)
        assert same(ix.read_rows_bf16(0, n), twin.read_rows_bf16(0, n))
        twins_agree(ix, twin, q, tier)
        check(oracle_mod, ix.search(q[:40], 20, None), corpus, None, q[:40], 20, None, f"{tier} staged")
        before = state(ix, q[:20])
        for where in (STAGE_ELEMS, over.size - 1):
            bad = over.copy()
            bad.flat[where] = 0.1
            with pytest.raises(NotFloat32Error):
                ix.append_f64(bad)
            assert_same_state(before, state(ix, q[:20]))
            with pytest.raises(NotFloat32Error):
                ix.overwrite_f64_batch(slots, bad)
            assert_same_state(before, state(ix, q[:20]))


@pytest.mark.parametrize("tier", ["f32", "split", "splitdirty"])
@pytest.mark.parametrize("d", [64, 100])
def test_unaligned_device_source(rb, oracle_mod, d, tier):
    """append_f64_device from a tensor view one float64 into its storage (8- but not 16-byte aligned) stores the rows
    an aligned source stores and gives the same answers."""
    import torch
    rng = np.random.default_rng(d)
    rows = prep(rng.standard_normal((3000, d)), tier)
    q = rows[rng.choice(3000, 200)] + 0.2 * rng.standard_normal((200, d))
    t = torch.from_numpy(np.concatenate([[0.0], rows.ravel()])).cuda()
    view = t[1:]
    ta = torch.from_numpy(rows).cuda()
    assert view.data_ptr() % 16 == 8 and ta.data_ptr() % 16 == 0
    torch.cuda.synchronize()
    with make(rb, d, TIERS[tier]) as a, make(rb, d, TIERS[tier]) as b:
        a.append_f64_device(view.data_ptr(), len(rows))
        b.append_f64_device(ta.data_ptr(), len(rows))
        assert same(a.read_rows_bf16(0, a.size()), b.read_rows_bf16(0, b.size()))
        assert_same_answers(answers(a, q), answers(b, q))
        got = a.exact_scores(q[:3])
        for i in range(3):
            assert got[i].tobytes() == oracle_mod.scores(rows, q[i]).tobytes(), i
        check(oracle_mod, a.search(q[:40], 20, None), rows, None, q[:40], 20, None, f"{tier} d={d} unaligned")


# --------------------------------------------------------------------------- 8. tier changes where dpad != d
TIER_PATH = [SPLIT, KEEP32, SPLIT | HOST, KEEP64, SPLIT, KEEP32 | F16, SPLIT]


def set_tier(h, flags):
    h.set_tier(exact_rows=exact_name(flags), f64_on_host=bool(flags & HOST), scan_f16=bool(flags & F16))
    assert h.flags == flags


def scan_bits(h, flags):
    return (h.read_rows_f16 if flags & F16 else h.read_rows_bf16)(0, h.size())


@pytest.mark.parametrize("d", [7, 100, 513, 4095])
def test_tier_changes_where_dpad_is_not_d(rb, oracle_mod, d):
    """An index and a 3-member group of split rows with planted 0x8000 low halves, along split -> f32 -> split|host ->
    f64 -> split -> f32|f16 -> split: after every step the storage bytes, the scan copy and every answer equal a new
    index built in that tier.  Then the narrowing into the split from f64|host, to the device and to the host."""
    n = 2 * 4096 + 777
    rng = np.random.default_rng(d)
    rows = prep(rng.standard_normal((n, d)), "splitdirty")
    rows[100:300] = rows[99]
    q = np.concatenate([rows[99:100], rows[rng.choice(n, 199)] + 0.3 * rng.standard_normal((199, d))])
    live = runs_dead(n, rng, 0.2)
    dead = np.flatnonzero(live == 0)
    corpus = rows[live.astype(bool)]

    def fill(h):
        h.append_f64(rows)
        h.tombstone(dead)

    with make(rb, d, TIER_PATH[0]) as ix, make(rb, d, TIER_PATH[0], rb.Group, group_devices(3)) as g:
        fill(ix), fill(g)
        for step, flags in enumerate(TIER_PATH):
            if step:
                set_tier(ix, flags)
                set_tier(g, flags)
            what = f"d={d} step {step} -> {exact_name(flags)} flags {flags}"
            with make(rb, d, flags) as fresh:
                fill(fresh)
                assert ix.storage_bytes() == fresh.storage_bytes(), what
                want_bits = scan_bits(fresh, flags)
                assert same(scan_bits(ix, flags), want_bits), what
                if flags & SPLIT:
                    assert same(want_bits, split_hi(rows)), what
                assert_same_answers_only(answers(ix, q), answers(fresh, q), skip=())
                want = routes(fresh, q[:12], n + 7)
                assert bit_equal(routes(g, q[:12], n + 7), want), what
                assert g.exact_scores(q[:3]).tobytes() == fresh.exact_scores(q[:3]).tobytes(), what
                for m in range(3):
                    assert same(member_rows(rb, g, m, "f16" if flags & F16 else "bf16"),
                                want_bits[member_slots(3, n, m)]), (what, m)
        check(oracle_mod, ix.search(q[:20], 20, None), rows, live, q[:20], 20, None, f"d={d} after the path")
        assert len(corpus) == ix.count()

    for to in (SPLIT, SPLIT | HOST):
        with make(rb, d, KEEP64 | HOST) as ix, make(rb, d, to) as fresh:
            fill(ix), fill(fresh)
            set_tier(ix, to)
            assert ix.storage_bytes() == fresh.storage_bytes()
            assert same(ix.read_rows_bf16(0, n), fresh.read_rows_bf16(0, n))
            assert_same_answers_only(answers(ix, q), answers(fresh, q), skip=())


# --------------------------------------------------------------------------- 9. growth and groups
def storage_at(cap, d, flags):
    """rbk_index_storage_bytes at capacity cap: rows | inv_norm | norm2 | tombstone bits on the device, plus the exact
    rows (4 or 2 bytes per element) wherever they are kept."""
    dpad = (d + 63) // 64 * 64
    dev = cap * dpad * 2 + (cap + 255) // 256 * 256 * 4 + 256 * 4 + cap * 8 + (cap + 31) // 32 * 4
    exact = cap * d * (4 if flags & KEEP32 else 2)
    return (dev, exact) if flags & HOST else (dev + exact, 0)


def fitted(n):
    return (max(n, 1024) + 255) // 256 * 256


GROW_STATS = ("searches", "queries", "fallback_queries", "retry_batches", "scan_launches", "kernel_launches",
              "graph_replays", "last_kprime")


@pytest.mark.parametrize("tier", EXACT_TIERS)
def test_growing_twin_matches_a_presized_one(rb, oracle_mod, tier):
    """An index that starts at 1024 rows and grows through every append route, and one sized never to grow: the same
    bits on every route, the same counters, before and after tombstones, compaction, trim and appends past the trimmed
    capacity.  Split rows carry planted 0x8000 low halves."""
    import torch
    from runbookai_b200 import synth
    d, flags = 200, TIERS[tier]
    kind = "splitdirty" if flags & SPLIT else tier
    rng = np.random.default_rng(7)
    grown, sized = make(rb, d, flags), make(rb, d, flags, cap=40000)
    twins = (grown, sized)
    corpus = np.zeros((0, d))
    live = np.zeros(0, np.uint8)
    caps = []

    def append(rows_f64, call):
        nonlocal corpus, live
        assert {call(ix) for ix in twins} == {len(corpus)}
        corpus = np.concatenate([corpus, rows_f64])
        live = np.concatenate([live, np.ones(len(rows_f64), np.uint8)])
        caps.append(grown.storage_bytes())

    def check_twins(q):
        x, y = routes(grown, q[:24], 5000), routes(sized, q[:24], 5000)
        assert bit_equal(x, y)
        sa, sb = grown.stats(), sized.stats()
        assert {k: sa[k] for k in GROW_STATS} == {k: sb[k] for k in GROW_STATS}
        assert grown.size() == sized.size() and grown.count() == sized.count()
        check(oracle_mod, grown.search(q[:24], 40, 0.2), corpus, live, q[:24], 40, 0.2, f"{tier} grown")
        sized.search(q[:24], 40, 0.2)                                  # keep the counters comparable

    try:
        assert grown.storage_bytes() == storage_at(1024, d, flags)
        r = prep(rng.standard_normal((900, d)), kind)
        append(r, lambda ix: ix.append_f64(r))
        q = corpus[rng.choice(len(corpus), 200)] + 0.5 * rng.standard_normal((200, d))
        check_twins(q)
        r32 = prep(rng.standard_normal((1500, d)), kind).astype(np.float32)
        append(r32.astype(np.float64), lambda ix: ix.append_f32(r32))
        check_twins(q)
        rbf = synth.f32_to_bf16_bits(rng.standard_normal((2100, d)).astype(np.float32))
        append(synth.bf16_bits_to_f32(rbf).astype(np.float64), lambda ix: ix.append_bf16(rbf))
        check_twins(q)
        rdv = prep(rng.standard_normal((5000, d)), kind)
        t = torch.from_numpy(rdv).cuda()
        torch.cuda.synchronize()
        append(rdv, lambda ix: ix.append_f64_device(t.data_ptr(), len(rdv)))
        check_twins(q)
        rb16 = synth.f32_to_bf16_bits(rng.standard_normal((9000, d)).astype(np.float32))
        tb = torch.from_numpy(rb16.view(np.int16)).cuda()
        torch.cuda.synchronize()
        append(synth.bf16_bits_to_f32(rb16).astype(np.float64), lambda ix: ix.append_bf16_device(tb.data_ptr(), len(rb16)))
        check_twins(q)
        assert len({c[0] for c in caps}) >= 4
        assert grown.storage_bytes() == storage_at(20480, d, flags)     # doubling, whole 256-row tiles
        assert sized.storage_bytes() == storage_at(40192, d, flags)
        if flags & SPLIT:
            assert same(grown.read_rows_bf16(0, grown.size()), split_hi(corpus))
        dead = np.setdiff1d(np.arange(len(corpus)), np.arange(0, len(corpus), 7))
        for ix in twins:
            ix.tombstone(dead)
        live[dead] = 0
        maps = [ix.compact() for ix in twins]
        assert same(maps[0], maps[1]) and same(maps[0], expected_map(live))
        corpus, live = corpus[live.astype(bool)], np.ones(int(live.sum()), np.uint8)
        for ix in twins:
            ix.trim()
            assert ix.storage_bytes() == storage_at(fitted(len(corpus)), d, flags)
        q = corpus[rng.choice(len(corpus), 200)] + 0.5 * rng.standard_normal((200, d))
        check_twins(q)
        fit = fitted(len(corpus))
        r = prep(rng.standard_normal((6000, d)), kind)
        append(r, lambda ix: ix.append_f64(r))
        check_twins(q)
        for ix in twins:
            assert ix.storage_bytes() == storage_at(fitted(max(len(corpus), 2 * fit)), d, flags)
    finally:
        for ix in twins:
            ix.close()


@pytest.mark.parametrize("tier", ["split", "splithost"])
@pytest.mark.parametrize("G", [2, 5, 8])
def test_group_members(rb, oracle_mod, G, tier):
    """A group of G co-located members and an index fed the same appends (straddling blocks and members) and
    tombstones of split rows with planted 0x8000 low halves: members hold their block-cyclic slices, every route is bit
    for bit the index's, and the same again after both compact."""
    n, d = 2 * G * 4096 + 777, 100
    flags = TIERS[tier]
    rng = np.random.default_rng(401 + G)
    corpus = prep(rng.standard_normal((n, d)), "splitdirty")
    q = corpus[rng.choice(n, 12)] + 0.2 * rng.standard_normal((12, d))
    live = runs_dead(n, rng, 0.3)
    with make(rb, d, flags, rb.Group, [0] * G) as g, make(rb, d, flags) as ix:
        append_in_pieces((g, ix), tier, corpus)
        for h in (g, ix):
            h.tombstone(np.flatnonzero(live == 0))
        check_members(rb, g, ix, tier)
        assert same(ix.read_rows_bf16(0, n), split_hi(corpus))
        before = routes(g, q, 4097)
        assert bit_equal(before, routes(ix, q, 4097))
        assert g.exact_scores(q).tobytes() == ix.exact_scores(q).tobytes()
        for key in ((20, None, "f64"), (112, 0.05, "f32"), (4096, 0.05, "large"), (4097, None, "unbounded")):
            qq = q.astype(np.float32).astype(np.float64) if key[2] == "f32" else q
            check(oracle_mod, before[key], corpus, live, qq, key[0], key[1], f"{tier} G={G} {key}")
        m_g, m_i = g.compact(), ix.compact()
        assert same(m_g, m_i) and same(m_g, expected_map(live))
        check_members(rb, g, ix, tier)
        after = routes(g, q, 4097)
        assert bit_equal(after, routes(ix, q, 4097))
        assert_same_through_map(before, after, m_g)
        survivors = corpus[live.astype(bool)]
        for key in ((20, None, "f64"), (4097, None, "unbounded")):
            check(oracle_mod, after[key], survivors, None, q, key[0], key[1], f"{tier} G={G} compacted {key}")
