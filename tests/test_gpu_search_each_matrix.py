"""GPU suite (-m gpu): rbk_index_search_each_f64 / rbk_group_search_each_f64 against the oracle, on every storage tier,
at per-query thresholds inside each query's own error band, at the ends of the float64 range, at widths from 1 to 65536,
through the retry and the exhaustive kernel, on groups of 2 to 8 members and after every kind of mutation.

Bar: row b of every call is the oracle's answer for query b at its own (k_b, m_b): the same ids and count, the same
float64 score bytes, the tail padded with -1 and quiet NaN.  The expected [B, K] block is built on the host from the
oracle's scores of each distinct query (threshold_cases.hits: keep `>= m_b`, stable sort by score descending, first k_b).

The batches are the point.  The per-query arrays are offset by hand at every seam of the host code (the 1,024-query
scan sub-batch, the large-k query groups, the failing-query list of the exhaustive kernel), so a query that reads a
neighbour's cut or threshold must get a visibly wrong answer:
- every position's (k, m) is drawn from a seeded permutation, never a short period;
- every query has its own threshold ladder, built at its own k (the oracle bytes of its hits k and k + 1 and their
  float64 neighbours, where the finalize proof switches between count == k and count < k), and in call c position p
  takes rung (p + c) mod L, so after L calls every (position, rung) pair has been searched while its neighbours sit at
  other rungs;
- batches straddle query 1024 on both routes, split into several large-k query groups, and fail in scattered
  positions.
Every case built to reach a path (retry, fallback, query groups, group re-answer, graph replay) asserts through stats()
that it did.  Run with -s for the module's wall time."""
import time
import zlib

import numpy as np
import pytest

import threshold_cases as tc
from float_range_cases import SCALES, SPECIAL, scaled, special
from test_gpu_exact_paths import WIDE_ABOVE, group_scores, sweep_corpus, tie_queries
from test_gpu_f32_matrix import F16, HOST, KEEP32, KEEP64, SPLIT, prep, rerank_corpus
from test_gpu_float_range import in_band, ladder_rows
from test_gpu_group_members import BLOCK, append_in_pieces, member_slots
from test_gpu_thresholds import Oracle
from test_gpu_widths import batch_pool, route_corpus

pytestmark = pytest.mark.gpu

TIERS = {"bf16": 0, "f64": KEEP64, "f64host": KEEP64 | HOST, "scan_f16": KEEP64 | F16, "f32": KEEP32,
         "f32host": KEEP32 | HOST, "f32f16": KEEP32 | F16, "split": SPLIT, "splithost": SPLIT | HOST,
         "splitdirty": SPLIT}
EXACT_TIERS = ("f64", "f64host", "f32", "f32host", "split", "splithost")
GROUP_TIERS = ("bf16", "f64", "f64host", "split", "splithost")
SEAM = 1100                         # positions of a batch that straddles query 1024 (kMaxSubBatch)
SUB_BATCH = 1024
SCAN_K = (1, 10, 56, 112)
LARGE_K = (113, 1000, 4096)
LARGE_BUDGET = 256 << 20            # rbk_index_impl.h kLargeBudget
WIDTHS = [1, 3, 7, 9, 100, 511, 513, 1025, 2049, 4095, 4096, 16384]
SEEN = {}                           # what the module reached: path -> count


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
    print(f"\n[search_each matrix] paths reached: {dict(sorted(SEEN.items()))}")
    print(f"[search_each matrix] module wall time: {time.perf_counter() - t0:.1f} s")


def make(rb, d, tier, cls=None, devices=None, cap=0):
    f = TIERS[tier]
    kw = dict(capacity_hint=cap, keep_f64=bool(f & KEEP64), keep_f32=bool(f & KEEP32), keep_f32_split=bool(f & SPLIT),
              f64_on_host=bool(f & HOST), scan_f16=bool(f & F16))
    return rb.Group(d, devices, **kw) if cls is rb.Group else rb.Index(d, **kw)


def tier_rows(rows, tier):
    """The float64 values a tier stores exactly: bf16 roundings, float32-exact rows (prep), or the rows themselves."""
    if tier == "bf16":
        return tc.bf16_f64(rows)
    if TIERS[tier] & (KEEP32 | SPLIT):
        return prep(rows, tier)
    return np.asarray(rows, dtype=np.float64)


def stored(rows, tier):
    return tc.stored(rows, tier == "bf16")


# --------------------------------------------------------------------------- the expectation and the comparison
def expected(orc, q, ks, ms):
    """The [B, K] block (K = max k): row b is the oracle's first k_b hits of q[b] at m_b (None: no threshold), then -1
    and quiet NaN."""
    B, K = len(q), int(max(ks))
    es = np.full((B, K), -1, np.int64)
    ev = np.full((B, K), np.nan)
    ec = np.zeros(B, np.int32)
    for b in range(B):
        s, v = orc.hits(q[b], ms[b])
        n = min(int(ks[b]), len(s))
        es[b, :n], ev[b, :n], ec[b] = s[:n], v[:n], n
    return es, ev, ec


def stats_line(h, st0=None):
    st = h.stats()
    keys = ("retry_batches", "fallback_queries", "scan_launches") + (("redone_batches",) if "redone_batches" in st else ())
    return ", ".join(f"{k} {st[k] - (st0[k] if st0 else 0)}" for k in keys)


def check_block(got, want, what):
    slots, scores, counts = got[:3]
    es, ev, ec = want
    assert slots.shape == es.shape and scores.shape == ev.shape, (what, slots.shape, es.shape)
    bad = np.flatnonzero((counts != ec) | (slots != es).any(axis=1)
                         | (scores.view(np.uint64) != ev.view(np.uint64)).any(axis=1))
    assert not len(bad), f"{what}: {len(bad)} of {len(es)} queries differ from the oracle (position, count, want): " \
                         f"{[(int(b), int(counts[b]), int(ec[b])) for b in bad[:8]]}"


def run(h, orc, q, ks, ms, what):
    """search_each against the oracle; returns (answer, stats delta)."""
    st0 = h.stats()
    got = h.search_each(q, ks, ms)
    st1 = h.stats()
    delta = {k: st1[k] - st0[k] for k in ("retry_batches", "fallback_queries", "scan_launches")}
    if "redone_batches" in st1:
        delta["redone_batches"] = st1["redone_batches"] - st0["redone_batches"]
        delta["per_device_scans"] = [b["scan_launches"] - a["scan_launches"]
                                     for a, b in zip(st0["per_device"], st1["per_device"])]
    for k in ("retry_batches", "fallback_queries", "redone_batches"):
        if delta.get(k):
            SEEN[k] = SEEN.get(k, 0) + delta[k]
    check_block(got, expected(orc, q, ks, ms), f"{what} [{stats_line(h, st0)}]")
    return got, delta


# --------------------------------------------------------------------------- batch builders (tests/test_search_each_matrix_host.py)
def draw(rng, B, choices):
    """Each position's pick: a seeded permutation of the choices repeated to B entries (balanced, no period)."""
    idx = rng.permutation(np.resize(np.arange(len(choices)), B))
    return [choices[i] for i in idx]


def own_ladder(scores, k, band_slots=None, t=None):
    """One query's thresholds at its own k: the bytes of its hits 1, k and k + 1 (clamped to its last hit), of the band
    row nearest t and of the band's lowest row (without a band: its median hit and its lowest live score), each with
    its float64 neighbours: 15 rungs."""
    s, v = tc.hits(scores, None)
    n = len(v)
    if band_slots is None:
        mid, low = v[n // 2], v[-1]
    else:
        mid, low = scores[band_slots[np.argmin(np.abs(scores[band_slots] - t))]], scores[band_slots].min()
    return tc.with_neighbours([v[0], v[min(k, n) - 1], v[min(k, n - 1)], mid, low])


class LadderBatch:
    """Positions over a few queries, each with its own k (drawn) and its own ladder at that k; call c gives position p
    rung (p + c) mod L."""

    def __init__(self, rng, scores, B, k_choices, band=None, t=None):
        self.qi = np.array(draw(rng, B, list(range(len(scores)))))
        self.ks = np.array(draw(rng, B, list(k_choices)), dtype=np.int64)
        self.ladders = {}
        for i, k in set(zip(self.qi.tolist(), self.ks.tolist())):
            self.ladders[(i, k)] = own_ladder(scores[i], k, None if band is None else band[i],
                                              None if t is None else t[i])
        self.L = min(len(v) for v in self.ladders.values())

    def ms(self, c):
        return [float(self.ladders[(i, k)][(p + c) % self.L]) for p, (i, k) in enumerate(zip(self.qi, self.ks))]


def budget_groups(cost):
    """rbk_capi.cu split_by_budget: contiguous query groups whose summed cost fits kLargeBudget."""
    groups, q0, used = [], 0, 0
    for b, c in enumerate(cost):
        if b > q0 and used + c > LARGE_BUDGET:
            groups.append((q0, b))
            q0, used = b, 0
        used += c
    groups.append((q0, len(cost)))
    return groups


def group_result_cost(G, K):
    """A query's cost in a group's large-k search before its candidates: its result in the local, gathered and merged
    blocks, (G + 2) (16 K + 8) bytes (rbk_group.cu group_search_large)."""
    return (G + 2) * (16 * K + 8)


BUDGET_SPLIT = dict(G=3, B=1000, K=4096)     # one count scan per member (B <= 1024), then one emit scan per group


def fallback_batch(rng, d, rows, wide, B):
    """B positions, four fifths of them queries of the wide tie groups (150 duplicates, 0 or 5 rows above) scattered
    through the batch after position 0, the rest random; k_b in [1, 112] and m_b below the group's score or None.  Returns
    (queries, ks, ms, positions that must fall back)."""
    n_tie = int(0.8 * B)
    tq, groups = tie_queries(rng, d, wide, n_tie)
    pos = np.sort(1 + rng.choice(B - 1, n_tie, replace=False))    # position 0 is a random query
    q = rng.standard_normal((B, d))
    q[pos] = tq
    ks = rng.integers(1, 113, B)
    gs = group_scores(rows, wide, tq, groups)
    ms = [None] * B
    m_tie = np.where(rng.random(n_tie) < 0.3, np.nan, gs - rng.uniform(0.02, 0.5, n_tie))
    for j, p in enumerate(pos):
        ms[p] = None if np.isnan(m_tie[j]) else float(m_tie[j])
    rest = np.setdiff1d(np.arange(B), pos)
    for p in rest:
        ms[p] = [None, -0.05, 0.0, 0.1][p % 4] if rng.random() < 0.5 else float(rng.uniform(-0.2, 0.2))
    must = pos[ks[pos] > np.array(WIDE_ABOVE)[groups]]
    return q, ks.tolist(), ms, must


# --------------------------------------------------------------------------- 1. per-query band ladder
ROUTES = {"scan": SCAN_K, "large": LARGE_K, "sorted": None}


def route_batch(route, d, tier):
    """Positions per route: the scan and large routes straddle query 1024 where the exhaustive kernel is cheap."""
    host = bool(TIERS[tier] & HOST)
    if route == "sorted":
        return 16 if host and d > 500 else 64
    if host and d > 500:
        return 40
    return SEAM if route == "scan" or d <= 500 else 300


@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", list(TIERS))
def test_band_ladder_per_query(rb, oracle_mod, tier, d):
    """band_corpus's four queries repeated over the batch, each position at its own k and at a rung of its own ladder
    at that k: kEach prep's thr_init, the finalize proof at (k_q, m_q), large_select at k_q, the re-rank and the
    segmented sort's filters at m_q."""
    c = tc.band_corpus(d, tier == "bf16", seed=10 + d)
    rows = tier_rows(c["rows"], tier)
    n = len(rows)
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        orc = Oracle(oracle_mod, stored(rows, tier))
        scores = [orc.scores(q) for q in c["q"]]
        for route, kc in ROUTES.items():
            B = route_batch(route, d, tier)
            rng = np.random.default_rng(zlib.crc32(f"{tier} {d} {route}".encode()))
            lb = LadderBatch(rng, scores, B, kc or (4097, n + 7), c["band"], c["t"])
            q = c["q"][lb.qi]
            for call in range(lb.L):
                ms = lb.ms(call)
                got, dl = run(ix, orc, q, lb.ks, ms, f"{tier} d={d} {route} B={B} call {call}")
                subs = -(-B // SUB_BATCH)
                if route == "scan":
                    assert dl["scan_launches"] in (subs, 2 * subs), dl
                else:
                    assert dl["scan_launches"] == 2 * subs and dl["fallback_queries"] == 0, dl
                if call == 0:       # the same batch shuffled: its rows come back permuted the same way
                    perm = rng.permutation(B)
                    sh = ix.search_each(q[perm], lb.ks[perm], [ms[p] for p in perm])
                    for a, b in zip(sh[:3], got[:3]):
                        assert a.tobytes() == b[perm].tobytes(), f"{tier} d={d} {route}: shuffled batch"


# --------------------------------------------------------------------------- 2. fixed ladder and the ends
@pytest.mark.parametrize("tier,huge", [(t, False) for t in TIERS] + [("f64", True), ("scan_f16", True)])
def test_fixed_ladder_and_ends(rb, oracle_mod, tier, huge):
    """ends_corpus at d = 8 with tombstoned multiples on the thresholds: every position of a batch at a different rung
    of the fixed ladder or of the ends, +-inf, +-DBL_MAX, +-0 and 1 +- ulp in one sub-batch, on both routes."""
    c = tc.ends_corpus(8, tier == "bf16", seed=8, huge=huge)
    rows = c["rows"] if tier == "bf16" else tier_rows(c["rows"], tier)
    live = np.ones(len(rows), np.uint8)
    dead = c["multiples"][::4]
    with make(rb, 8, tier) as ix:
        ix.append_f64(rows)
        ix.tombstone(dead)
        live[dead] = 0
        orc = Oracle(oracle_mod, stored(rows, tier), live)
        ths = {np.float64(v).tobytes() for q in c["q"] for v in tc.ends_ladder(oracle_mod.scores(orc.stored, q))}
        ths = [float(np.frombuffer(b)[0]) for b in sorted(ths)] + [None]
        rng = np.random.default_rng(len(ths))
        B = 3 * len(ths)
        qi = np.array(draw(rng, B, [0, 1, 2, 3]))
        for route, kc in (("scan", (1, 3, 12, 40, 112)), ("large", (113, 500, len(rows) + 7))):
            ks = draw(rng, B, list(kc))
            for call in range(3):
                ms = [ths[(p + call) % len(ths)] for p in range(B)]
                run(ix, orc, c["q"][qi], ks, ms, f"{tier} ends huge={huge} {route} call {call}")


# --------------------------------------------------------------------------- 3. tie groups on the threshold
@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", list(TIERS))
def test_tie_groups_per_query(rb, oracle_mod, tier, d):
    """tie_corpus's 5, 70 and 150 duplicates, each group's query at its own k inside its group, past it, at the group's
    score and one ulp above, among random queries: the 70 take the wide retry and nothing falls back, the 150 reach
    exact_scan_each_kernel / exact_merge_kernel at their own k."""
    if TIERS[tier] & HOST and d > 500:
        pytest.skip("covered at d = 100: each falling-back query reads every exact row over PCIe")
    c = tc.tie_corpus(d, tier == "bf16", seed=d)
    rows = tier_rows(c["rows"], tier)
    rng = np.random.default_rng(d + len(tier))
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        orc = Oracle(oracle_mod, stored(rows, tier))
        ms_g = [float(orc.scores(c["q"][g])[c["dup"][g][0]]) for g in range(3)]
        rand_q = rng.standard_normal((40, d))

        def batch(groups, kinds):
            """Tie positions (group, k, m) for every group and kind, scattered among 40 random queries."""
            ent = []
            for g in groups:
                size, above = c["sizes"][g], c["above"]
                for kind in kinds:
                    k = {"inside": above + size // 2, "past": above + size + 10}[kind[0]]
                    m = {"ms": ms_g[g], "up": float(np.nextafter(ms_g[g], np.inf)), "none": None}[kind[1]]
                    ent += [(c["q"][g], k, m, g, kind)] * 2
            ent += [(rand_q[i], int(rng.integers(1, 30)), None, -1, None) for i in range(len(rand_q))]
            order = rng.permutation(len(ent))
            ent = [ent[i] for i in order]
            return (np.array([e[0] for e in ent]), [e[1] for e in ent], [e[2] for e in ent], ent)

        what = f"{tier} d={d}"
        # (one ulp above the group, a k inside it would leave count < k with the group within the bound: unprovable)
        q, ks, ms, ent = batch([0, 1], [("inside", "ms"), ("inside", "none")])
        _, dl = run(ix, orc, q, ks, ms, f"{what} 70 inside, among random queries")
        assert dl["retry_batches"] == 1, f"{what}: the 70 take the wide retry ({dl})"
        tie = [i for i, e in enumerate(ent) if e[3] == 1]
        _, dl = run(ix, orc, q[tie], [ks[i] for i in tie], [ms[i] for i in tie], f"{what} 70 inside")
        assert dl["retry_batches"] == 1 and dl["fallback_queries"] == 0, f"{what}: k' = 128 holds the 70 ({dl})"
        q, ks, ms, ent = batch([0, 1, 2], [("inside", "ms"), ("inside", "none"), ("inside", "up")])
        _, dl = run(ix, orc, q, ks, ms, f"{what} 150 inside")
        pos150 = [i for i, e in enumerate(ent) if e[3] == 2 and e[4][1] != "up"]
        assert pos150 != list(range(len(pos150))), "the failing queries must not be a prefix of the batch"
        assert dl["fallback_queries"] >= len(pos150) > 0, f"{what}: the 150 must fall back ({dl}, {len(pos150)})"
        q, ks, ms, ent = batch([0, 1, 2], [("inside", "ms"), ("past", "ms"), ("past", "up"), ("inside", "none")])
        got, dl = run(ix, orc, q, ks, ms, f"{what} large route")
        for b, e in enumerate(ent):
            if e[3] >= 0 and e[4] == ("past", "ms"):      # the whole group and the rows above it are hits
                assert got[2][b] >= c["above"] + c["sizes"][e[3]], (what, b, e[3])


# --------------------------------------------------------------------------- 4. mostly falling back
@pytest.mark.parametrize("d", [511, 512])
@pytest.mark.parametrize("tier", EXACT_TIERS)
def test_mostly_falling_back(rb, oracle_mod, tier, d):
    """1,100 queries, most of them at a k inside a 150-duplicate group, scattered through the batch at their own k and
    threshold: the exhaustive kernel's failing-query list is not a prefix, and n_blocks * K > 768 with k_q << K."""
    rng, rows, wide, narrow = sweep_corpus(d, 300 + d)
    rows = tier_rows(rows, tier)
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        orc = Oracle(oracle_mod, rows)
        q, ks, ms, must = fallback_batch(rng, d, rows, wide, SEAM)
        assert len(must) > SEAM // 2 and must[0] > 0
        _, dl = run(ix, orc, q, ks, ms, f"{tier} d={d} mostly falling back")
        assert dl["fallback_queries"] >= len(must), f"{tier} d={d}: {dl}, {len(must)} must fall back"


# --------------------------------------------------------------------------- 5. widths
def widths_cases():
    out = [(d, t) for d in WIDTHS for t in TIERS]
    return out + [(65536, "split"), (65536, "f32host")]


@pytest.mark.parametrize("d,tier", widths_cases())
def test_widths(rb, oracle_mod, d, tier):
    """route_corpus (tie groups of 150 and 60, tombstones, a zero row) at every width and tier: a mixed batch of 16
    pool queries repeated at 64 positions with their own k and threshold, on the scan and the large route - every
    finalize_each_kernel instantiation, finalize's d-chunking and dpad != d."""
    rng, rows, live, q, wide, narrow = route_corpus(d, d)
    rows = tier_rows(rows, tier)
    pool = batch_pool(rng, d, wide, narrow, n=16)
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        ix.tombstone(np.flatnonzero(live == 0))
        orc = Oracle(oracle_mod, stored(rows, tier), live)
        qi = np.array(draw(rng, 64, list(range(16))))
        hit = float(orc.hits(pool[1], None)[1][4])
        for route, kc in (("scan", SCAN_K), ("large", LARGE_K)):
            ks = draw(rng, 64, list(kc))
            ms = draw(rng, 64, [None, 0.0, -0.0, 0.3, hit, float(np.nextafter(hit, 2.0)), -np.inf, 0.9])
            run(ix, orc, pool[qi], ks, ms, f"{tier} d={d} {route}")


# --------------------------------------------------------------------------- 6. the float range
FLOAT_TIERS = ("bf16", "f64", "f64host", "scan_f16")


def float_queries(rng, base):
    """One query per SCALES rung and per SPECIAL class, the zero query, and as many ordinary ones, interleaved."""
    qs = [scaled(base[i % len(base)] + 0.1 * rng.standard_normal(base.shape[1]), e) for i, e in enumerate(SCALES)]
    qs += [special(base[i], name) for i, name in enumerate(SPECIAL)]
    qs += [np.zeros(base.shape[1])]
    n_odd = len(qs)
    qs += [base[i % len(base)] + 0.1 * rng.standard_normal(base.shape[1]) for i in range(n_odd)]
    q = np.stack(qs)
    return q[rng.permutation(len(q))]


def off_band(q):
    """Queries the reference scores (finite, not all zero) outside the scan's band: each one is the exhaustive
    kernel's."""
    fin = np.isfinite(q).all(axis=1) & (q != 0).any(axis=1)
    return fin & ~in_band(q)


@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", FLOAT_TIERS)
def test_float_range_per_query(rb, oracle_mod, tier, d):
    """Off-band queries ("inf", "zero" classes, NaN element, zero query) beside ordinary ones at their own thresholds,
    +-inf and +-0 included; on the scan route the batch falls back exactly the live off-band queries more than its
    in-band queries alone do (at the same largest k, so at the same k').  Then the
    row ladder joins the corpus and every route answers across the range (large_emit_all for part of a sub-batch)."""
    rng = np.random.default_rng(d)
    rows = tier_rows(rng.standard_normal((3000, d)), tier)
    base = rows[rng.choice(3000, 8)]
    q = float_queries(rng, base)
    B = len(q)
    ths = [None, -np.inf, np.inf, 0.0, -0.0, 0.5, 0.9, -0.3]
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        orc = Oracle(oracle_mod, stored(rows, tier))
        for call in range(4):
            ks = draw(rng, B, list(SCAN_K))
            ms = [ths[(p + call) % len(ths)] for p in range(B)]
            _, dl = run(ix, orc, q, ks, ms, f"{tier} d={d} scan call {call}")
            inb = np.flatnonzero(~off_band(q))
            assert max(ks[i] for i in inb) == max(ks)
            _, dl_in = run(ix, orc, q[inb], [ks[i] for i in inb], [ms[i] for i in inb], f"{tier} d={d} in band")
            n_off = int(off_band(q).sum())
            assert dl["fallback_queries"] - dl_in["fallback_queries"] == n_off > 10, \
                f"{tier} d={d}: {dl} with {n_off} live off-band queries, {dl_in} without them"
            run(ix, orc, q, draw(rng, B, list(LARGE_K)), ms, f"{tier} d={d} large call {call}")
        extra = ladder_rows(rng, rows, base, "bf16" if tier == "bf16" else "device")
        ix.append_f64(extra)
        allrows = np.concatenate([rows, extra])
        orc = Oracle(oracle_mod, ix.read_rows_bf16(0, ix.size()) if tier == "bf16" else allrows)
        for call in range(3):
            ms = [ths[(p + call) % len(ths)] for p in range(B)]
            run(ix, orc, q, draw(rng, B, list(SCAN_K)), ms, f"{tier} d={d} row ladder scan")
            run(ix, orc, q, draw(rng, B, [113, 2000, len(allrows) + 3]), ms, f"{tier} d={d} row ladder large")


# --------------------------------------------------------------------------- 7. host-staged re-rank
@pytest.mark.parametrize("d", [15, 17, 511, 513])
@pytest.mark.parametrize("tier", ["f32host", "splithost", "f64host"])
def test_host_staged_rerank(rb, oracle_mod, tier, d):
    """Exact rows in pinned host memory: the re-rank reads them in staged chunks under each query's own cut, at
    B = 8, 300 and 1,100 on the large route, and at B = 300 on the scan route."""
    rows, q = rerank_corpus(d, tier)
    rng = np.random.default_rng(d)
    with make(rb, d, tier) as ix:
        ix.append_f64(rows)
        orc = Oracle(oracle_mod, rows)
        for B in (8, 300, SEAM):
            ks = draw(rng, B, [113, 700, 4096, 150])
            ms = draw(rng, B, [None, 0.0, 0.05, -0.1])
            _, dl = run(ix, orc, q[:B], ks, ms, f"{tier} d={d} large B={B}")
            assert dl["scan_launches"] == 2 * -(-B // SUB_BATCH), dl
        ks = draw(rng, 300, list(SCAN_K))
        run(ix, orc, q[:300], ks, draw(rng, 300, [None, 0.0, 0.05]), f"{tier} d={d} scan B=300")


# --------------------------------------------------------------------------- 8. groups
def group_corpus(G, d, seed):
    n = G * BLOCK + 777
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((40, d))
    near = rng.choice(n, (40, 6), replace=False)
    for i in range(40):
        rows[near[i]] = q[i] + 0.5 * rng.standard_normal((6, d))
    return rng, rows, q


def load_group(g, rows, tier):
    append_in_pieces((g,), tier, tc.bf16_bits(rows) if tier == "bf16" else rows)


@pytest.mark.parametrize("G", [2, 5, 8])
@pytest.mark.parametrize("tier", GROUP_TIERS)
def test_colocated_groups(rb, oracle_mod, tier, G):
    """Co-located members holding every block-cyclic slice; a 300-position batch at its own k and threshold on the
    scan, large and sorted routes."""
    d = 64
    rng, rows, q = group_corpus(G, d, 10 * G)
    rows = tier_rows(rows, tier)
    with make(rb, d, tier, rb.Group, [0] * G) as g:
        load_group(g, rows, tier)
        for m in range(G):
            assert len(member_slots(G, len(rows), m)) > 0
        orc = Oracle(oracle_mod, stored(rows, tier))
        qi = np.array(draw(rng, 300, list(range(len(q)))))
        for route, kc in (("scan", SCAN_K), ("large", LARGE_K), ("sorted", (4097, len(rows) + 7, 5))):
            B = 300 if route != "sorted" else 24
            ks = draw(rng, B, list(kc))
            hit = float(orc.hits(q[0], None)[1][3])
            ms = draw(rng, B, [None, 0.0, 0.2, hit, float(np.nextafter(hit, 2.0)), -np.inf])
            run(g, orc, q[qi[:B]], ks, ms, f"{tier} G={G} {route}")


def test_group_re_answer_with_per_query_cuts(rb, oracle_mod):
    """150 duplicates on one member: a query cut inside them fails that member's proof, every member re-answers the
    batch at each query's own cut (search_device_exact with k_each), and the merge reads the re-uploaded cuts."""
    d, G = 256, 3
    rng, rows, q = group_corpus(G, d, 77)
    u = q[0] + 0.2 * rng.standard_normal(d)
    rows[100:250] = u                          # one block: member 0
    for tier in ("f64", "bf16"):
        r = tier_rows(rows, tier)
        with make(rb, d, tier, rb.Group, [0] * G) as g:
            load_group(g, r, tier)
            orc = Oracle(oracle_mod, stored(r, tier))
            B = 200
            qi = np.array(draw(rng, B, list(range(len(q)))))
            ks = [60 if i == 0 else int(rng.integers(1, 112)) for i in qi]
            ms = draw(rng, B, [None, 0.0, 0.1])
            _, dl = run(g, orc, q[qi], ks, ms, f"group {tier} re-answer")
            assert dl["redone_batches"] >= 1, f"{tier}: the duplicates were meant to fail member 0's proof ({dl})"


def test_group_budget_split(rb, oracle_mod):
    """A large-k batch whose result blocks alone need more than kLargeBudget: several query groups, each merged at its
    own queries' cuts (each[0].k + gr.first)."""
    G, B, K = BUDGET_SPLIT["G"], BUDGET_SPLIT["B"], BUDGET_SPLIT["K"]
    assert len(budget_groups([group_result_cost(G, K)] * B)) > 1
    d = 32
    rng, rows, q = group_corpus(G, d, 5)
    with make(rb, d, "f64", rb.Group, [0] * G) as g:
        load_group(g, rows, "f64")
        orc = Oracle(oracle_mod, rows)
        qi = np.array(draw(rng, B, list(range(len(q)))))
        ks = draw(rng, B, [K, 113, 500, 2000, 150, 3000])
        ms = draw(rng, B, [None, 0.0, 0.1, -0.2])
        _, dl = run(g, orc, q[qi], ks, ms, "group budget split")
        assert min(dl["per_device_scans"]) > 2, f"expected more than one query group: {dl}"


def test_index_budget_split(rb, oracle_mod):
    """The same on an index: a sorted-route batch at k above count() (k_eff = count()) whose blocks need more than
    kLargeBudget."""
    d, n = 16, 20000
    rng = np.random.default_rng(70)
    rows = rng.standard_normal((n, d))
    q = rng.standard_normal((40, d))
    B = 900
    assert len(budget_groups([16 * n + 8] * B)) > 1
    with make(rb, d, "f64") as ix:
        ix.append_f64(rows)
        orc = Oracle(oracle_mod, rows)
        qi = np.array(draw(rng, B, list(range(40))))
        ks = draw(rng, B, [n + 7, 5, 5000, 12000, 4097])
        ms = draw(rng, B, [None, 0.0, 0.3, -0.5])
        _, dl = run(ix, orc, q[qi], ks, ms, "index budget split")
        assert dl["scan_launches"] > 2, f"expected more than one query group: {dl}"


def test_group_after_compaction_and_all_tombstoned(rb, oracle_mod):
    """Trailing members emptied by compaction, then every row tombstoned: the answers stay the oracle's."""
    d, G = 64, 5
    rng, rows, q = group_corpus(G, d, 9)
    live = np.zeros(len(rows), np.uint8)
    live[:BLOCK + 500] = 1
    with make(rb, d, "f64", rb.Group, [0] * G) as g:
        load_group(g, rows, "f64")
        g.tombstone(np.flatnonzero(live == 0))
        B = 120
        qi = np.array(draw(rng, B, list(range(len(q)))))
        for route, kc in (("scan", SCAN_K), ("large", LARGE_K)):
            run(g, Oracle(oracle_mod, rows, live), q[qi], draw(rng, B, list(kc)), draw(rng, B, [None, 0.0, 0.2]),
                f"tombstoned {route}")
        g.compact()
        kept = rows[live == 1]
        assert g.size() == len(kept)
        for route, kc in (("scan", SCAN_K), ("large", LARGE_K), ("sorted", (len(kept) + 7, 4097))):
            run(g, Oracle(oracle_mod, kept), q[qi], draw(rng, B, list(kc)), draw(rng, B, [None, 0.0, 0.2]),
                f"compacted {route}")
        g.tombstone(np.arange(len(kept)))
        for kc in (SCAN_K, LARGE_K):
            got = g.search_each(q[qi], draw(rng, B, list(kc)), draw(rng, B, [None, -np.inf, 0.0]))
            assert (got[2] == 0).all() and (got[0] == -1).all()
            assert (got[1].view(np.uint64) == 0x7FF8000000000000).all()


# --------------------------------------------------------------------------- 9. state changes
def test_after_every_mutation_beside_the_graph(rb, oracle_mod):
    """search_each after tombstone, overwrite, compact, trim (which releases the cut buffers), set_tier into and out of
    every tier and growth past a presized twin; small searches replayed from the captured graph in between keep
    replaying and stay the oracle's."""
    d = 100
    rng = np.random.default_rng(12)
    rows = tier_rows(rng.standard_normal((6000, d)), "f32")
    q = rows[rng.choice(6000, 24)] + 0.3 * rng.standard_normal((24, d))
    live = np.ones(len(rows), np.uint8)
    B = SEAM
    qi = np.array(draw(rng, B, list(range(24))))

    def each(h, what):
        o = Oracle(oracle_mod, rows, None if live.all() else live)
        for route, kc in (("scan", SCAN_K), ("large", LARGE_K)):
            run(h, o, q[qi], draw(rng, B, list(kc)), draw(rng, B, [None, 0.0, 0.3, 0.6]), f"{what} {route}")
        g0 = h.stats()["graph_replays"]
        for m in (0.3, None):
            got = h.search(q[:8], 10, m)
            es, ev, ec = expected(o, q[:8], [10] * 8, [m] * 8)
            check_block(got, (es, ev, ec), f"{what} graph search")
        assert h.stats()["graph_replays"] == g0 + 2, f"{what}: the small searches must replay the captured graph"
        SEEN["graph_replays"] = SEEN.get("graph_replays", 0) + 2

    with make(rb, d, "f64") as ix, make(rb, d, "f64", cap=64) as grow:
        ix.append_f64(rows[:3000])
        grow.append_f64(rows[:3000])
        ix.search(q[:8], 10, 0.3)                 # capture the graph before anything else
        ix.append_f64(rows[3000:])
        for i in range(3000, 6000, 1000):
            grow.append_f64(rows[i:i + 1000])
        each(ix, "appended")
        each(grow, "grown")
        dead = rng.choice(6000, 400, replace=False)
        ix.tombstone(dead)
        live[dead] = 0
        each(ix, "tombstoned")
        slots = np.flatnonzero(live)[:50]
        new = tier_rows(q[np.arange(50) % 24] + 0.1 * rng.standard_normal((50, d)), "f32")
        ix.overwrite_f64_batch(slots, new)
        rows[slots] = new
        each(ix, "overwritten")
        ix.compact()
        rows, live = rows[live == 1], np.ones(int(live.sum()), np.uint8)
        each(ix, "compacted")
        ix.trim()
        each(ix, "trimmed")
        for name, kw in (("f64host", dict(f64_on_host=True)), ("scan_f16", dict(f64_on_host=False, scan_f16=True)),
                         ("f32", dict(scan_f16=False, exact_rows="f32")), ("f32host", dict(f64_on_host=True)),
                         ("splithost", dict(exact_rows="f32_split")), ("split", dict(f64_on_host=False)),
                         ("f64", dict(exact_rows="f64"))):
            ix.set_tier(**kw)
            each(ix, f"set_tier -> {name}")
