"""GPU suite (-m gpu): every search route and storage tier against the oracle at embedding widths outside 8-2048.

The ABI takes any 1 <= dim <= RBK_MAX_DIM (2^20).  Width changes the scan's error bound ((d+8) 2^-22 grows linearly),
which path answers (at wide d the bound reaches the spread of the top scores, so queries retry and fall back), the
exact re-rank's chunking (chunk width from key_cap and nsel), the storage floors (1024 rows per index, 4096-row
blocks per group member, 32-row compaction staging) and, at tiny d, every search becomes one big exact tie.

Bar: ids, counts and float64 score bytes equal to the oracle's over the rows the index stores; every case built to
reach the retry or the fallback asserts through stats() that it did.  Run with -s to see, per width, the largest
ratio of scan error to its bound, which path answered at the extreme widths, and the device memory the tests used
(free memory before the module minus free memory at the sampled points, so other processes on the device count)."""
import numpy as np
import pytest

from test_gpu_compact import all_answers, assert_same_through_map, expected_map
from test_gpu_exact_paths import check, check_proven, counters, mismatches, oracle_answers, tie_corpus
from test_gpu_float_range import all_routes, bf16_f64, make_index, score_bytes, search_device
from test_gpu_group_compact import bit_equal, routes, runs_dead
from test_gpu_scan_f16 import acc_eps, bf16_angle, bits_to_f64, f16_angle, f16_store

pytestmark = pytest.mark.gpu

MAX_DIM = 1 << 20
TINY = [1, 2, 3, 5, 7]
WIDE = [2049, 3072, 4095, 4096, 8192, 16384]
TIERS = ("bf16", "device", "host", "f16")
ELEMS = 8_000_000          # n * d of a route corpus (at least 1000 rows): keeps the host oracle quick
BATCHES = [(1100, 0), (321, 500), (161, 200), (129, 900), (1, 502)]   # (B, offset into the pool), descending B
K = 20

RATIOS = {}                # (tier, kind, d) -> largest |scan - exact| / eps_q
PATHS = {}                 # (d, tier) -> (retry batches, fallback queries) of one top-k search
MEMORY = {}                # test -> largest device memory in use at a sampled point, bytes


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


@pytest.fixture(scope="module", autouse=True)
def report(rb):
    import torch
    base = torch.cuda.mem_get_info()[0]
    MEMORY["_base"] = base
    yield
    print("\nscan error / eps_q, largest seen:")
    for key in sorted(RATIOS):
        print(f"  {key}: {RATIOS[key]:.4f}")
    print("paths at d = 65536 (retry batches, fallback queries of one 3-query search):")
    for key in sorted(PATHS):
        print(f"  {key}: {PATHS[key]}")
    peaks = {k: v for k, v in MEMORY.items() if k != "_base"}
    if peaks:
        worst = max(peaks, key=peaks.get)
        print(f"device memory in use, largest sampled: {peaks[worst] / 2**30:.2f} GiB ({worst})")


def note_memory(what):
    import torch
    torch.cuda.synchronize()
    used = MEMORY["_base"] - torch.cuda.mem_get_info()[0]
    MEMORY[what] = max(MEMORY.get(what, 0), used)


def make(rb, d, tier, cls=None, **kw):
    """make_index's tiers, plus "f16host": fp16 scan over float64 rows in pinned host memory."""
    if tier == "f16host":
        return (cls or rb.Index)(d, keep_f64=True, f64_on_host=True, scan_f16=True, **kw)
    return make_index(rb, d, tier, cls, **kw)


def stored_rows(ix, rows, tier):
    return ix.read_rows_bf16(0, ix.size()) if tier == "bf16" else rows


# --------------------------------------------------------------------------- 1. every route, every tier
def route_corpus(d, seed):
    """Random rows, one tie group of 150 duplicates (wider than the retry) and one of 60 (held by the retry), each with
    5 rows above it, three planted near-duplicates of each of 4 plain queries, a zero row; 8 queries (2 per tie group,
    4 plain).  Returns (rng, rows, live, queries, wide, narrow)."""
    rng = np.random.default_rng(seed)
    n_rand = max(1000, min(6000, ELEMS // d)) - 250
    wide = tie_corpus(rng, d, n_rand, [5], group_size=150, q_per_group=2)
    narrow = tie_corpus(rng, d, 0, [5], group_size=60, q_per_group=2)
    plain = rng.standard_normal((4, d))
    planted = plain[np.repeat(np.arange(4), 3)] + 0.02 * rng.standard_normal((12, d))
    rows = np.concatenate([wide[0], narrow[0], planted])
    rows[7] = 0.0
    live = np.ones(len(rows), np.uint8)
    dead = np.setdiff1d(rng.choice(n_rand, n_rand // 30, replace=False), [7])
    live[np.concatenate([dead, wide[3][0][:5]])] = 0                      # 145 duplicates stay: still wider than 128
    q = np.concatenate([wide[1], narrow[1], plain])
    return rng, rows, live, q, wide, narrow


def batch_pool(rng, d, wide, narrow, n=1100):
    """Random queries with a wide-group query at every i = 0 mod 5 and a narrow-group one at every i = 2 mod 5."""
    pool = rng.standard_normal((n, d))
    for first, src in ((0, wide), (2, narrow)):
        idx = np.arange(first, n, 5)
        pool[idx] = src[1][idx % len(src[1])] + 0.01 * rng.standard_normal((len(idx), d))
    return pool


@pytest.mark.parametrize("d,tier", [(d, t) for d in TINY + WIDE for t in TIERS] + [(4095, "f16host")])
def test_every_route_every_tier(rb, oracle_mod, d, tier):
    rng, rows, live, q, wide, narrow = route_corpus(d, d)
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        ix.tombstone(np.flatnonzero(live == 0))
        stored = stored_rows(ix, rows, tier)
        note_memory(f"routes d={d} {tier}")
        all_routes(oracle_mod, ix, stored, live, q, f"{tier} d={d}")

        # descending batches: every key_cap tier, the retry in each, and smaller batches over stale query-pad rows
        pool = batch_pool(rng, d, wide, narrow)
        want = oracle_answers(oracle_mod, stored, live, pool, K, None)
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


# --------------------------------------------------------------------------- 2. mutations at wide widths
@pytest.mark.parametrize("tier", TIERS)
@pytest.mark.parametrize("d", [3072, 16384])
def test_mutations_at_wide_widths(rb, oracle_mod, d, tier):
    """Grow from a small capacity_hint past the 1024-row floor, overwrite a batch, tombstone document runs, compact
    (answers through the map), trim (answers unchanged), append again, then the oracle on the final state."""
    n = 1300 if d == 16384 else 3000
    rng = np.random.default_rng(d + len(tier))
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((6, d))
    near = rng.choice(n, 18, replace=False)
    rows[near] = q[np.arange(18) % 6] + 0.3 * rng.standard_normal((18, d))
    with make(rb, d, tier, capacity_hint=16) as ix:
        dev0 = ix.storage_bytes()
        for part in np.array_split(np.arange(n), 3):
            ix.append_f64(rows[part])
        assert ix.storage_bytes()[0] > dev0[0], "the index grew past its creation capacity"
        slots = rng.choice(n, 40, replace=False)
        over = rng.standard_normal((40, d))
        over[:6] = q + 0.2 * rng.standard_normal((6, d))
        ix.overwrite_f64_batch(slots, over)
        rows[slots] = over
        live = runs_dead(n, rng, 0.4)
        ix.tombstone(np.flatnonzero(live == 0))
        note_memory(f"mutations d={d} {tier}")
        before = all_answers(ix, q)
        old_to_new = ix.compact()
        assert (old_to_new == expected_map(live)).all() and ix.size() == ix.count() == live.sum()
        after = all_answers(ix, q)
        assert_same_through_map(before, after, old_to_new)
        ix.trim()
        assert bit_equal(all_answers(ix, q), after), "trim changed an answer"
        more = rng.standard_normal((500, d))
        more[:6] = q + 0.25 * rng.standard_normal((6, d))
        assert ix.append_f64(more) == live.sum()
        final = np.concatenate([rows[live.astype(bool)], more])
        stored = stored_rows(ix, final, tier)
        m = ix.size()
        for k, ms in ((1, None), (K, None), (112, 0.0)):
            check(oracle_mod, ix.search(q, k, ms), stored, None, q, k, ms, f"{tier} d={d} final k={k}")
        check(oracle_mod, ix.search_large(q, 500, None), stored, None, q, 500, None, f"{tier} d={d} final large")
        check(oracle_mod, ix.search_unbounded(q, m + 7, None), stored, None, q, m + 7, None,
              f"{tier} d={d} final unbounded")
        got = ix.exact_scores(q[:2])
        for b in range(2):
            assert score_bytes(got[b]) == score_bytes(oracle_mod.scores(stored, q[b])), (tier, d, b)


# --------------------------------------------------------------------------- 3. scan-bound soundness
@pytest.mark.parametrize("kind", ["gaussian", "positive"])
@pytest.mark.parametrize("tier", ["bf16", "device", "f16"])
@pytest.mark.parametrize("d", [3072, 4096, 8192, 16384])
def test_scan_scores_stay_within_the_bound(rb, d, tier, kind):
    """debug_scores within eps_q = (d+8) 2^-22 + the query's rounding angle + the largest row rounding angle (0 for
    bf16 rows), on gaussian data and on all-positive data, where the accumulator's truncation errors do not cancel.
    A row whose every element rounds as far as it can sets the row term."""
    n, b = 2000, 16
    rng = np.random.default_rng(d + 3 * (kind == "positive") + len(tier))
    if kind == "gaussian":
        corpus = rng.standard_normal((n, d))
        q = rng.standard_normal((b, d))
    else:
        corpus = np.abs(rng.standard_normal((n, d))) + 0.05
        q = np.abs(rng.standard_normal((b, d))) + 0.05
        q[0] = 1.0
    sign = np.sign(rng.standard_normal(d)) if kind == "gaussian" else 1.0
    half = 2.0 ** -11 if tier == "f16" else 2.0 ** -8
    corpus[17] = (1.0 + half - 2.0 ** -30) * sign
    q[1] = corpus[17] * (1.0 + half / 8 * rng.standard_normal(d))
    if tier == "bf16":
        corpus = bf16_f64(corpus)
    q = q.astype(np.float32).astype(np.float64)
    ref = (q @ corpus.T) / (np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(corpus, axis=1)[None, :])
    if tier == "f16":
        eps = acc_eps(d) + f16_angle(q) + f16_angle(corpus).max()
    else:
        eps = acc_eps(d) + bf16_angle(q) + (bf16_angle(corpus).max() if tier == "device" else 0.0)
    with make(rb, d, tier) as ix:
        ix.append_f64(corpus)
        got = ix.debug_scores(q.astype(np.float32)).astype(np.float64)
    err = np.abs(got - ref)
    ratio = err / eps[:, None]
    RATIOS[(tier, kind, d)] = float(ratio.max())
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert (err <= eps[:, None]).all(), (worst, err[worst], eps[worst[0]])


# --------------------------------------------------------------------------- 4. stored bits
@pytest.mark.parametrize("d", TINY + [4095, 16384])
def test_stored_bits_follow_the_rounding_rule(rb, d):
    """read_rows_bf16 is RNE_bf16(RNE_f32(x)) and read_rows_f16 the scaled fp16 rule, for rows from float64, float32
    and bf16 on the host and float64 and bf16 on the device."""
    import torch
    from runbookai_b200 import synth
    rng = np.random.default_rng(40 + d)
    f64 = rng.standard_normal((9, d)) * np.exp(rng.uniform(-30, 30, (9, 1)))
    f64[2] = 0.0
    f64[3] = 1.0 + 2.0 ** -8 - 2.0 ** -30            # just under a bf16 half step
    f64[4] = 1.0 + 2.0 ** -11 - 2.0 ** -30           # just under an fp16 half step
    f32 = (rng.standard_normal((5, d)) * np.exp(rng.uniform(-20, 20, (5, 1)))).astype(np.float32)
    bf = synth.f32_to_bf16_bits(rng.standard_normal((5, d)).astype(np.float32) * np.float32(7e-3))
    # slots: f64 host | f32 host | bf16 host | f64 device | bf16 device
    want = np.concatenate([f64, f32.astype(np.float64), bits_to_f64(bf), f64, bits_to_f64(bf)])
    for tier in ("bf16", "device", "f16"):
        with make(rb, d, tier) as ix:
            ix.append_f64(f64)
            ix.append_f32(f32)
            ix.append_bf16(bf)
            t = torch.from_numpy(f64).cuda()
            tb = torch.from_numpy(bf.view(np.int16)).cuda()
            torch.cuda.synchronize()
            ix.append_f64_device(t.data_ptr(), len(f64))
            ix.append_bf16_device(tb.data_ptr(), len(bf))
            if tier == "f16":
                got, exp = ix.read_rows_f16(0, ix.size()), f16_store(want)[0].view(np.uint16)
            else:
                got, exp = ix.read_rows_bf16(0, ix.size()), synth.f32_to_bf16_bits(want.astype(np.float32))
        bad = np.argwhere(got != exp)
        assert len(bad) == 0, (tier, d, bad[:5], got[tuple(bad[0])], exp[tuple(bad[0])])


# --------------------------------------------------------------------------- 5. d = 1: one big tie
@pytest.mark.parametrize("tier", TIERS)
def test_one_element_rows_are_one_tie(rb, oracle_mod, tier):
    """Every live nonzero row scores +-1 against every query: the answers are the rows of the query's sign in slot
    order, min_score = 1.0 keeps all of them, and the top-k search cannot prove anything from the scan."""
    n = 5000
    rng = np.random.default_rng(1)
    rows = rng.standard_normal((n, 1)) * np.exp(rng.uniform(-10, 10, (n, 1)))
    rows[::97] = 0.0
    if tier == "bf16":
        rows = bf16_f64(rows)
    q = np.array([[1.0], [-3.0], [0.25]])
    with make(rb, 1, tier) as ix:
        ix.append_f64(rows)
        stored = stored_rows(ix, rows, tier)
        r0, f0 = counters(ix)
        got = ix.search(q, 112, None)
        r1, f1 = counters(ix)
        check(oracle_mod, got, stored, None, q, 112, None, f"{tier} d=1")
        assert f1 - f0 == len(q), "every query of an all-tied corpus needs the exhaustive kernel"
        for b in range(len(q)):
            same_sign = np.flatnonzero(np.sign(rows[:, 0]) == np.sign(q[b, 0]))
            assert (got[0][b] == same_sign[:112]).all() and (got[1][b] == 1.0).all(), b
        for fn, k in ((ix.search, 20), (ix.search_large, 4096), (ix.search_unbounded, n + 7)):
            s, v, c, _ = fn(q, k, 1.0)
            check(oracle_mod, (s, v, c), stored, None, q, k, 1.0, f"{tier} d=1 min_score=1.0 k={k}")
            for b in range(len(q)):
                m = int((np.sign(rows[:, 0]) == np.sign(q[b, 0])).sum())
                assert c[b] == min(k, m) and (v[b, :c[b]] == 1.0).all(), (fn.__name__, b)
        for k, ms in ((4096, None), (4500, None), (5000, 0.0), (n + 7, None), (n + 7, -1.0)):
            fn = ix.search_large if k <= 4096 else ix.search_unbounded
            check(oracle_mod, fn(q, k, ms), stored, None, q, k, ms, f"{tier} d=1 k={k} min_score={ms}")


# --------------------------------------------------------------------------- 6. extreme widths
def extreme_routes(oracle_mod, ix, stored, q, what):
    """B in {1, 3} on every route (no batch above 128: the oracle reads a whole corpus per query)."""
    n = ix.count()
    for B in (1, 3):
        qq = q[:B]
        q32 = qq.astype(np.float32)
        for ms in (None, 0.0):
            w = f"{what} B={B} min_score={ms}"
            check(oracle_mod, ix.search(qq, 10, ms), stored, None, qq, 10, ms, w + " search f64")
            check(oracle_mod, ix.search(q32, 10, ms), stored, None, q32.astype(np.float64), 10, ms, w + " search f32")
            check(oracle_mod, search_device(ix, q32, 10, ms), stored, None, q32.astype(np.float64), 10, ms,
                  w + " search_device")
            check_proven(oracle_mod, ix, stored, None, q32, 10, ms)
            for k in (200, 4096):
                check(oracle_mod, ix.search_large(qq, k, ms), stored, None, qq, k, ms, f"{w} search_large {k}")
            for k in (4500, n + 7):
                check(oracle_mod, ix.search_unbounded(qq, k, ms), stored, None, qq, k, ms, f"{w} search_unbounded {k}")
    got = ix.exact_scores(q)
    for b in range(len(q)):
        assert score_bytes(got[b]) == score_bytes(oracle_mod.scores(stored, q[b])), f"{what}: exact_scores {b}"


@pytest.mark.parametrize("d", [65536, MAX_DIM])
def test_extreme_widths_bf16(rb, oracle_mod, d):
    """A few hundred bf16 rows with planted neighbours of the queries: every route, then a compaction of runs of
    deleted rows (answers through the map, then the oracle on the survivors)."""
    from runbookai_b200 import synth
    n = 300 if d == 65536 else 200
    q = synth.random_queries(3, d, d).astype(np.float64)
    corpus = synth.random_corpus(n, d, d + 1)
    synth.plant_neighbours(corpus, q.astype(np.float32), 8, d + 2)
    corpus[11] = 0
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        note_memory(f"extreme d={d}")
        extreme_routes(oracle_mod, ix, corpus, q, f"bf16 d={d}")
        live = runs_dead(n, np.random.default_rng(d), 0.4)
        ix.tombstone(np.flatnonzero(live == 0))
        before = {(k, "f64"): ix.search(q, k, None)[:3] for k in (10, 112)}
        before[(n, "large")] = ix.search_large(q, n, None)[:3]
        old_to_new = ix.compact()
        assert (old_to_new == expected_map(live)).all() and ix.size() == live.sum()
        after = {(k, "f64"): ix.search(q, k, None)[:3] for k in (10, 112)}
        after[(n, "large")] = ix.search_large(q, n, None)[:3]
        assert_same_through_map(before, after, old_to_new)
        survivors = corpus[live.astype(bool)]
        assert (ix.read_rows_bf16(0, ix.size()) == survivors).all()
        for key, got in after.items():
            check(oracle_mod, got, survivors, None, q, key[0], None, f"bf16 d={d} compacted {key}")


@pytest.mark.parametrize("tier", TIERS)
def test_every_tier_at_65536(rb, oracle_mod, tier):
    """At d = 65536 the scan's bound (0.0156) is wider than the spread of random top scores: record which path
    answered, and check every route."""
    d, n = 65536, 200
    rng = np.random.default_rng(65536)
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((3, d))
    rows[[5, 50, 150]] = q + 0.5 * rng.standard_normal((3, d))
    if tier == "bf16":
        rows = bf16_f64(rows)
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        stored = stored_rows(ix, rows, tier)
        note_memory(f"tiers d=65536 {tier}")
        r0, f0 = counters(ix)
        ix.search(q, 10, None)
        r1, f1 = counters(ix)
        PATHS[(d, tier)] = (r1 - r0, f1 - f0)
        extreme_routes(oracle_mod, ix, stored, q, f"{tier} d={d}")


def test_width_above_the_limit_is_rejected(rb):
    for dim in (MAX_DIM + 1, 0):
        with pytest.raises(rb.RbkError, match="dim out of range") as e:
            rb.Index(dim)
        assert e.value.status == rb._native.RBK_EINVAL
        with pytest.raises(rb.RbkError, match="dim out of range") as e:
            rb.Group(dim, [0])
        assert e.value.status == rb._native.RBK_EINVAL


# --------------------------------------------------------------------------- 7. groups
@pytest.mark.parametrize("n_dev", [1, 2])
@pytest.mark.parametrize("tier", ["bf16", "device"])
@pytest.mark.parametrize("d", [3072, 16384])
def test_group_answers_like_an_index(rb, oracle_mod, d, tier, n_dev):
    """A group and an index fed the same calls (more than one 4096-row block, so a second GPU holds rows): the same
    answers bit for bit on every route, the same compaction map, the same answers after trim, and the oracle's."""
    from common import group_devices
    from runbookai_b200 import synth
    n = 5000
    rng = np.random.default_rng(d + n_dev)
    q = rng.standard_normal((6, d))
    if tier == "bf16":
        corpus = synth.random_corpus(n, d, d)
        synth.plant_neighbours(corpus, q.astype(np.float32), 5, d)
        q = synth.bf16_round(q).astype(np.float64)
    else:
        corpus = rng.standard_normal((n, d))
        corpus[rng.choice(n, 30, replace=False)] = q[np.arange(30) % 6] + 0.3 * rng.standard_normal((30, d))
    live = runs_dead(n, rng, 0.4)
    live[4096:4200] = 0
    with make(rb, d, tier, rb.Group, devices=group_devices(n_dev)) as g, make(rb, d, tier) as ix:
        for h in (g, ix):
            h.append_bf16(corpus) if tier == "bf16" else h.append_f64(corpus)
            h.tombstone(np.flatnonzero(live == 0))
        note_memory(f"group d={d} {tier} x{n_dev}")
        before = routes(g, q, n + 7)
        assert bit_equal(before, routes(ix, q, n + 7))
        m_g, m_i = g.compact(), ix.compact()
        assert (m_g == m_i).all() and (m_g == expected_map(live)).all()
        after = routes(g, q, n + 7)
        assert bit_equal(after, routes(ix, q, n + 7))
        assert_same_through_map(before, after, m_g)
        g.trim()
        ix.trim()
        assert bit_equal(routes(g, q, n + 7), after) and bit_equal(routes(ix, q, n + 7), after)
        survivors = corpus[live.astype(bool)]
        for key in ((K, None, "f64"), (112, 0.05, "f64"), (n + 7, None, "unbounded")):
            check(oracle_mod, after[key], survivors, None, q, key[0], key[1], f"group {tier} d={d} {key}")
