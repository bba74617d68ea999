"""GPU suite (-m gpu): min_score where it cuts.  Every search route and storage tier against the oracle at thresholds
with many live rows inside the scan's error bound eps_q on either side, on tie groups whose common score is the
threshold, at the cosine ends (+-1, +-0) and at non-finite and extreme thresholds.

The threshold enters the engine in several places, each with its own rounding: the scan's initial raw threshold
(prep_queries_kernel, from min_score - eps_q), the scan's filter, the finalize proof (count < k_fetch is proven when
no dropped row can reach min_score), the large-k select (theta = max(T - 2 eps, thr_init)), the exact `>= min_score`
of finalize, the exhaustive fallback, the large-k re-rank and the unbounded sort, and the key of the captured search
graph.  A slip in any of them changes which rows sit on the threshold's side of the answer.

Each query is scored by the oracle once per index state; every threshold's answer is derived from those scores on the
host (threshold_cases.hits: keep `>=`, stable sort by score descending), a derivation tests/test_thresholds_host.py
pins against the oracle's own search.  Answers are compared as ids, counts and float64 score bytes.  Retry, fallback
and flagged counts go into the assertion messages."""
import numpy as np
import pytest

import threshold_cases as tc
from test_gpu_exact_paths import counters, first_pass
from test_gpu_float_range import score_bytes, search_device

pytestmark = pytest.mark.gpu

TIERS = ("bf16", "device", "host", "f16")
F64_TIERS = ("device", "host", "f16")


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def make_index(rb, d, tier, cls=None, **kw):
    cls = cls or rb.Index
    return cls(d, keep_f64=tier != "bf16", f64_on_host=tier == "host", scan_f16=tier == "f16", **kw)


class Oracle:
    """The oracle's scores of each query over the stored rows (NaN for tombstoned rows), computed once, and every
    threshold's answer derived from them."""

    def __init__(self, oracle_mod, stored, live=None):
        self.o, self.stored, self.live = oracle_mod, stored, live
        self._scores, self._hits = {}, {}

    def scores(self, q):
        key = np.asarray(q, dtype=np.float64).tobytes()
        if key not in self._scores:
            s = self.o.scores(self.stored, q)
            if self.live is not None:
                s[self.live == 0] = np.nan
            self._scores[key] = s
        return self._scores[key]

    def hits(self, q, ms):
        key = (np.asarray(q, dtype=np.float64).tobytes(), None if ms is None else np.float64(ms).tobytes())
        if key not in self._hits:
            self._hits[key] = tc.hits(self.scores(q), ms)
        return self._hits[key]


def compare(orc, got, q, k, ms, what):
    """got = (slots [B, k], scores [B, k], counts [B], ...) against the oracle's first k hits of each query."""
    slots, scores, counts = got[0], got[1], got[2]
    bad = []
    for b in range(len(q)):
        es, ev = orc.hits(q[b], ms)
        n = min(k, len(es))
        if (int(counts[b]) != n or not np.array_equal(slots[b, :n], es[:n])
                or scores[b, :n].tobytes() != ev[:n].tobytes()):
            diff = np.flatnonzero(slots[b, :min(n, int(counts[b]))] != es[:min(n, int(counts[b]))])[:6]
            bad.append((b, int(counts[b]), n, diff.tolist()))
    assert not bad, f"{what} k={k} min_score={ms!r}: {len(bad)} of {len(q)} queries differ from the oracle " \
                    f"(query, count, want, slots): {bad[:8]}"


def check_proven(orc, ix, q32, k, ms, what):
    """Answers search_device_async flags as proven exact are the oracle's; returns how many it flagged."""
    s, v, c, f = first_pass(ix, q32, k, ms)
    assert set(np.unique(f)) <= {0, 1}
    ok = np.flatnonzero(f == 0)
    if len(ok):
        compare(orc, (s[ok], v[ok], c[ok]), q32[ok].astype(np.float64), k, ms, what + " proven first pass")
    return int((f == 1).sum())


def stats_line(ix):
    st = ix.stats()
    return f"retries {st['retry_batches']}, fallback {st['fallback_queries']}"


def every_route(orc, ix, q, ms, what, group=False, general=True):
    """Every route at one threshold; returns how many first-pass answers were left unproven.  general=False leaves
    out the > 128-query batch."""
    q32 = q.astype(np.float32)
    q32w = q32.astype(np.float64)
    big = np.concatenate([q] * (1 + 128 // len(q)))            # > 128 queries: the ungraphed general path
    w = f"{what} [{stats_line(ix)}]"
    n = ix.count()
    compare(orc, ix.search(q, tc.K, ms), q, tc.K, ms, w + " search f64")
    if general:
        compare(orc, ix.search(big, tc.K, ms), big, tc.K, ms, w + " search f64 B>128")
    compare(orc, ix.search_large(q, 200, ms), q, 200, ms, w + " search_large")
    compare(orc, ix.search_large(q, 4096, ms), q, 4096, ms, w + " search_large")
    compare(orc, ix.search_unbounded(q, 4500, ms), q, 4500, ms, w + " search_unbounded")
    compare(orc, ix.search_unbounded(q, n + 7, ms), q, n + 7, ms, w + " search_unbounded")
    if group:
        return 0
    compare(orc, ix.search(q32, tc.K, ms), q32w, tc.K, ms, w + " search f32")
    compare(orc, search_device(ix, q32, tc.K, ms), q32w, tc.K, ms, w + " search_device")
    return check_proven(orc, ix, q32, tc.K, ms, w)


def check_exact_scores(orc, ix, q, thresholds, what):
    """exact_scores are the oracle's bytes, and `>=` applied to them on the host gives the oracle's answers."""
    got = ix.exact_scores(q)
    for b in range(len(q)):
        assert score_bytes(got[b]) == score_bytes(orc.scores(q[b])), f"{what}: exact_scores of query {b}"
        for ms in thresholds:
            s, v = tc.hits(got[b], ms)
            es, ev = orc.hits(q[b], ms)
            assert np.array_equal(s, es) and v.tobytes() == ev.tobytes(), f"{what}: exact_scores >= {ms!r}"


def band_thresholds(orc, c):
    out = list(tc.FIXED_LADDER)
    for i, q in enumerate(c["q"]):
        out += tc.ladder(orc.scores(q), c["band"][i], c["t"][i])
    return out


def load_band(rb, oracle_mod, ix, c, tier):
    ix.append_f64(c["rows"])
    if tier == "bf16":
        assert np.array_equal(ix.read_rows_bf16(0, ix.size()), c["stored"])
    return Oracle(oracle_mod, c["stored"])


# --------------------------------------------------------------------------- the band ladder
@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", TIERS)
def test_band_ladder_on_every_route(rb, oracle_mod, tier, d):
    """Four queries, each with ~1500 rows spread over [t - 3 eps, t + 3 eps]; every threshold of every query's ladder
    and the fixed ladder, on every route."""
    c = tc.band_corpus(d, tier == "bf16", seed=10 + d)
    with make_index(rb, d, tier) as ix:
        orc = load_band(rb, oracle_mod, ix, c, tier)
        ths = band_thresholds(orc, c)
        unproven = 0
        for i, ms in enumerate(ths):
            # the host tier's exhaustive kernel reads the float64 rows over PCIe, so there a 132-query batch that
            # falls back costs seconds: the general path is taken at every fifth threshold
            unproven += every_route(orc, ix, c["q"], ms, f"{tier} d={d} band", general=tier != "host" or i % 5 == 0)
        check_exact_scores(orc, ix, c["q"], ths, f"{tier} d={d}")
        r, f = counters(ix)
        print(f"{tier} d={d}: {len(ths)} thresholds, retries {r}, fallback {f}, first-pass unproven {unproven}")


@pytest.mark.parametrize("n_dev", [1, 3])
@pytest.mark.parametrize("tier", TIERS)
def test_band_ladder_on_a_group(rb, oracle_mod, tier, n_dev):
    from common import group_devices
    d = 100
    c = tc.band_corpus(d, tier == "bf16", seed=77)
    with make_index(rb, d, tier, cls=rb.Group, devices=group_devices(n_dev)) as g:
        orc = load_band(rb, oracle_mod, g, c, "group")
        for ms in band_thresholds(orc, c):
            every_route(orc, g, c["q"], ms, f"{tier} group of {n_dev}", group=True)


# --------------------------------------------------------------------------- a tie group on the threshold
@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", TIERS)
def test_tie_group_on_the_threshold(rb, oracle_mod, tier, d):
    """5, 70 and 150 exact duplicates whose common score is min_score, 8 rows above them and rows within the bound
    below.  A k_fetch inside the group: the 70 duplicates take the wide retry (k' = 128) and nothing falls back, the
    150 reach the exhaustive kernel.  A k_fetch past the group leaves count < k_fetch; a threshold one ulp above the
    group drops all of it."""
    c = tc.tie_corpus(d, tier == "bf16", seed=d)
    with make_index(rb, d, tier) as ix:
        ix.append_f64(c["rows"])
        orc = Oracle(oracle_mod, c["stored"])
        for g, size in enumerate(c["sizes"]):
            q1, ms = c["q"][g:g + 1], float(c["ms"][g])
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
            assert int(got[2][0]) == c["above"] + size
            up = float(np.nextafter(ms, np.inf))
            got = ix.search(q1, k_cut, up)
            compare(orc, got, q1, k_cut, up, f"{what} [{stats_line(ix)}] one ulp above")
            assert int(got[2][0]) == c["above"], f"{what}: one ulp above the group must drop all of it"
            for m in (ms, up, float(np.nextafter(ms, -np.inf))):
                every_route(orc, ix, c["q"], m, what)


# --------------------------------------------------------------------------- the ends, and non-finite thresholds
@pytest.mark.parametrize("tier,huge", [("bf16", False), ("device", False), ("host", False), ("f16", False),
                                       ("device", True), ("f16", True)])
def test_ends_and_extreme_thresholds(rb, oracle_mod, tier, huge):
    """d = 8: multiples of each query (1 / -1 or one ulp off), rows scoring +0 (and, with 2^600 rows, -0), zero rows,
    and tombstoned multiples sitting on the thresholds; every threshold of the fixed ladder and of the ends."""
    c = tc.ends_corpus(8, tier == "bf16", seed=8, huge=huge)
    live = np.ones(len(c["rows"]), np.uint8)
    dead = c["multiples"][::4]
    with make_index(rb, 8, tier) as ix:
        ix.append_f64(c["rows"])
        ix.tombstone(dead)
        live[dead] = 0
        orc = Oracle(oracle_mod, c["stored"], live)
        ths = set()
        for q in c["q"]:
            ths |= {np.float64(v).tobytes() for v in tc.ends_ladder(oracle_mod.scores(c["stored"], q))}
        ths = [float(np.frombuffer(b)[0]) for b in sorted(ths)]
        unproven = sum(every_route(orc, ix, c["q"], ms, f"{tier} ends huge={huge}") for ms in ths)
        check_exact_scores(orc, ix, c["q"], ths, f"{tier} ends")
        for ms in ths:                      # tombstoned rows on the threshold are never returned
            for b in range(len(c["q"])):
                assert not np.isin(orc.hits(c["q"][b], ms)[0], dead).any()
        print(f"{tier} ends huge={huge}: {len(ths)} thresholds, {stats_line(ix)}, unproven {unproven}")


def test_nan_threshold_is_refused_on_every_route(rb, oracle_mod):
    import torch
    from common import group_devices
    from runbookai_b200._native import RBK_EINVAL, RbkError
    d = 100
    rng = np.random.default_rng(1)
    rows, q = rng.standard_normal((3000, d)), rng.standard_normal((4, d))
    nan = float("nan")
    B = len(q)
    qd = torch.from_numpy(q.astype(np.float32)).cuda()
    s = torch.empty((B, tc.K), dtype=torch.int64, device="cuda")
    v = torch.empty((B, tc.K), dtype=torch.float64, device="cuda")
    cn = torch.empty(B, dtype=torch.int32, device="cuda")
    f = torch.empty(B, dtype=torch.int32, device="cuda")
    with rb.Index(d, keep_f64=True) as ix, rb.Group(d, group_devices(3), keep_f64=True) as g:
        ix.append_f64(rows)
        g.append_f64(rows)
        calls = {
            "search f64": lambda: ix.search(q, tc.K, nan),
            "search f64 B>128": lambda: ix.search(np.concatenate([q] * 40), tc.K, nan),
            "search f32": lambda: ix.search(q.astype(np.float32), tc.K, nan),
            "search_large": lambda: ix.search_large(q, 200, nan),
            "search_unbounded": lambda: ix.search_unbounded(q, 4500, nan),
            "search_device": lambda: ix.search_device(qd.data_ptr(), B, tc.K, nan, s.data_ptr(), v.data_ptr(),
                                                      cn.data_ptr()),
            "search_device_async": lambda: ix.search_device_async(qd.data_ptr(), B, tc.K, nan, s.data_ptr(),
                                                                  v.data_ptr(), cn.data_ptr(), f.data_ptr()),
            "group search": lambda: g.search(q, tc.K, nan),
            "group search f32": lambda: g.search(q.astype(np.float32), tc.K, nan),
            "group search_large": lambda: g.search_large(q, 200, nan),
            "group search_unbounded": lambda: g.search_unbounded(q, 4500, nan),
        }
        for name, call in calls.items():
            before = (ix.stats()["searches"], g.stats()["searches"])
            with pytest.raises(RbkError) as e:
                call()
            assert e.value.status == RBK_EINVAL, name
            assert (ix.stats()["searches"], g.stats()["searches"]) == before, name
        torch.cuda.synchronize()
        # and the index still answers
        orc = Oracle(oracle_mod, rows)
        compare(orc, ix.search(q, tc.K, 0.1), q, tc.K, 0.1, "after NaN")
        compare(orc, g.search(q, tc.K, 0.1), q, tc.K, 0.1, "group after NaN")


# --------------------------------------------------------------------------- the captured graph
@pytest.mark.parametrize("tier", TIERS)
def test_graph_replay_follows_the_threshold(rb, oracle_mod, tier):
    """One B <= 128 batch searched at ms (a hit's score), one ulp above, ms again, -0, +0 and -inf: each call launches
    the captured graph once and each answer is the oracle's, so the graph is never replayed at a stale threshold."""
    d = 100
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((4000, d))
    q = rows[:4] + 0.3 * rng.standard_normal((4, d))
    if tier == "bf16":
        rows = tc.bf16_f64(rows)
    with make_index(rb, d, tier) as ix:
        ix.append_f64(rows)
        orc = Oracle(oracle_mod, tc.stored(rows, tier == "bf16"))
        ms = float(orc.hits(q[0], None)[1][2])          # the third hit of query 0
        for m in (ms, float(np.nextafter(ms, np.inf)), ms, -0.0, 0.0, -np.inf, ms):
            g0 = ix.stats()["graph_replays"]
            got = ix.search(q, tc.K, m)
            assert ix.stats()["graph_replays"] == g0 + 1, m
            compare(orc, got, q, tc.K, m, f"{tier} graph [{stats_line(ix)}]")
        assert int(ix.search(q, tc.K, ms)[2][0]) == 3 and int(ix.search(q, tc.K, np.nextafter(ms, 1.0))[2][0]) == 2


# --------------------------------------------------------------------------- mutations move rows across the threshold
def far_row(rng, d):
    """A row as far from its bf16 rounding as rounding gets (each element just under half a bf16 step above 1): it
    sets the corpus angle eps_c, about 2^-8."""
    return (1.0 + 2.0 ** -8 - 2.0 ** -30) * np.sign(rng.standard_normal(d))


@pytest.mark.parametrize("tier", TIERS)
def test_mutations_move_rows_across_the_threshold(rb, oracle_mod, tier):
    d = 100
    bf16 = tier == "bf16"
    c = tc.band_corpus(d, bf16, seed=31, per_band=600, n_random=1500)
    rows = c["rows"].copy()
    live = np.ones(len(rows), np.uint8)
    q = c["q"]
    rng = np.random.default_rng(3)
    with make_index(rb, d, tier) as ix:
        orc = load_band(rb, oracle_mod, ix, c, tier)
        sc = orc.scores(q[0])
        band = c["band"][0]
        mid = band[np.argmin(np.abs(sc[band] - c["t"][0]))]
        ms = float(sc[mid])
        below = band[(sc[band] < ms) & (sc[band] >= ms - c["eps"][0])][:30]
        assert len(below) == 30

        def run(what, thresholds=None):
            o = Oracle(oracle_mod, tc.stored(rows, bf16), live if not live.all() else None)
            for m in thresholds or (ms, float(np.nextafter(ms, np.inf)), float(np.nextafter(ms, -np.inf))):
                every_route(o, ix, q, m, f"{tier} {what}")
            return o

        # rows just below ms are overwritten with the row scoring exactly ms: 31 rows now tie on the threshold
        ix.overwrite_f64_batch(below, np.repeat(rows[mid][None, :], len(below), axis=0))
        rows[below] = rows[mid]
        o = run("overwritten to ms")
        assert int((o.scores(q[0]) == ms).sum()) == 31

        # the tie group tombstoned, then compacted away
        on = np.r_[below, mid]
        ix.tombstone(on)
        live[on] = 0
        run("tombstoned at ms")
        old_to_new = ix.compact()
        keep = live.astype(bool)
        assert (old_to_new[keep] == np.arange(keep.sum())).all()
        rows, live = rows[keep], live[keep]
        run("compacted")

        # the tier changes in place
        if not bf16:
            for to in [t for t in F64_TIERS if t != tier] + [tier]:
                ix.set_tier(f64_on_host=to == "host", scan_f16=to == "f16")
                run(f"set_tier -> {to}")

        # a row whose bf16 rounding is far from it raises the corpus bound eps_c: the scan's initial threshold of
        # the next search must use the new bound, so the answers it proves stay the oracle's
        slot = int(np.flatnonzero(live)[5])
        far = far_row(rng, d)
        if bf16:
            far = tc.bf16_f64(far)
        ix.overwrite_f64(slot, far)
        rows[slot] = far
        ms2 = [float(v) for v in (tc.ladder(run("far row").scores(q[0]), np.flatnonzero(
            np.abs(sc[keep] - c["t"][0]) < 3 * c["eps"][0]), c["t"][0]))]
        run("far row, band ladder", ms2)
