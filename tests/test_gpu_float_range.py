"""GPU suite (-m gpu): every search route against the oracle when a query or a row sits near the ends of the float32 /
bf16 exponent range or past them, on every tier.

The scan reads bf16 (or scaled fp16) copies and accumulates in fp32; its error bound (DESIGN.md §6) holds only while
the copies are live and the products stay inside fp32's normal range.  Queries and rows scaled by a ladder of powers of
two (float_range_cases.SCALES) land on either side of each of those boundaries: bf16 zeros, float32 overflow, fp32
product underflow and overflow, and float64 norms that underflow to 0 (cosine +-Infinity) or overflow (cosine +-0).

Bar: ids, counts and float64 score bytes equal to the oracle's (so -0 vs +0 counts), on search (float64 and float32
queries, a graph-replayed batch and a general one), search_device, search_large, search_unbounded and exact_scores;
an answer search_device_async flags as proven is the oracle's.  Where a case has to leave the scan for the exhaustive
kernel, the stats() counters say it did."""
import numpy as np
import pytest

from float_range_cases import SCALES, scaled
from test_gpu_exact_paths import check, check_proven, counters, oracle_answers

pytestmark = pytest.mark.gpu

TIERS = ("bf16", "device", "host", "f16")
N_PLAIN = 5000
LADDER = sorted(SCALES)
MIN_SCORES = (None, 0.0, 0.5)
# Inputs whose largest element lies in [2^-40, 2^40] stay on the scan; the rest are answered exactly (DESIGN.md §6).
SCAN_BAND = 40


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def make_index(rb, d, tier, cls=None, **kw):
    cls = cls or rb.Index
    return cls(d, keep_f64=tier != "bf16", f64_on_host=tier == "host", scan_f16=tier == "f16", **kw)


def bf16_f64(x):
    from runbookai_b200 import synth
    with np.errstate(over="ignore"):
        return synth.bf16_round(np.asarray(x, dtype=np.float64).astype(np.float32)).astype(np.float64)


def stored_rows(ix, rows, tier):
    return rows if tier != "bf16" else ix.read_rows_bf16(0, ix.size())


def in_band(x):
    a = np.abs(np.asarray(x, dtype=np.float64))
    m = np.where(np.isfinite(a), a, 0.0).max(axis=-1)
    return (m >= 2.0 ** -SCAN_BAND) & (m < 2.0 ** SCAN_BAND)


def score_bytes(v):
    """float64 bytes (-0 and +0 differ), every NaN one value."""
    return [b"nan" if x != x else x.tobytes() for x in np.asarray(v, dtype=np.float64)]


def search_device(ix, q32, k, ms):
    import torch
    B = len(q32)
    qd = torch.from_numpy(np.ascontiguousarray(q32, dtype=np.float32)).cuda()
    s = torch.empty((B, k), dtype=torch.int64, device="cuda")
    v = torch.empty((B, k), dtype=torch.float64, device="cuda")
    c = torch.empty(B, dtype=torch.int32, device="cuda")
    ix.search_device(qd.data_ptr(), B, k, ms, s.data_ptr(), v.data_ptr(), c.data_ptr())
    torch.cuda.synchronize()
    return s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy()


def all_routes(oracle_mod, ix, stored, live, q, what, group=False):
    """Every route on float64 queries q (and their float32 copies) at each min_score; returns how many queries the
    first pass left unproven."""
    n = ix.count()
    with np.errstate(over="ignore"):
        q32 = q.astype(np.float32)
    q32w = q32.astype(np.float64)
    big = np.concatenate([q] * (1 + 200 // len(q)))           # > 128 queries: the ungraphed path
    unproven = 0
    for ms in MIN_SCORES:
        w = f"{what} min_score={ms}"
        check(oracle_mod, ix.search(q, 10, ms), stored, live, q, 10, ms, w + " search f64")
        check(oracle_mod, ix.search(big, 10, ms), stored, live, big, 10, ms, w + " search f64 B>128")
        check(oracle_mod, ix.search(q32, 10, ms), stored, live, q32w, 10, ms, w + " search f32")
        check(oracle_mod, ix.search_large(q, 200, ms), stored, live, q, 200, ms, w + " search_large 200")
        check(oracle_mod, ix.search_large(q, 4096, ms), stored, live, q, 4096, ms, w + " search_large 4096")
        for k in (4500, n + 7):
            check(oracle_mod, ix.search_unbounded(q, k, ms), stored, live, q, k, ms, f"{w} search_unbounded {k}")
        if not group:
            check(oracle_mod, search_device(ix, q32, 10, ms), stored, live, q32w, 10, ms, w + " search_device")
            unproven += check_proven(oracle_mod, ix, stored, live, q32, 10, ms)
    got = ix.exact_scores(q)
    for b in range(len(q)):
        want = oracle_mod.scores(stored, q[b])
        if live is not None:
            want[live == 0] = np.nan
        assert score_bytes(got[b]) == score_bytes(want), f"{what}: exact_scores of query {b}"
    return unproven


def plain_corpus(d, tier, seed):
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((N_PLAIN, d))
    return rng, (bf16_f64(rows) if tier == "bf16" else rows)


# --------------------------------------------------------------------------- queries across the range
@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", TIERS)
def test_query_scale_ladder(rb, oracle_mod, tier, d):
    """Ordinary rows; each query is a corpus row plus noise, scaled by one rung of the ladder (and +-2^30, which stay
    on the scan).  Queries past the scan's band must reach the exhaustive kernel."""
    rng, rows = plain_corpus(d, tier, d)
    es = LADDER + [-30, 30]
    base = rows[rng.choice(N_PLAIN, len(es))] + 0.1 * rng.standard_normal((len(es), d))
    q = np.stack([scaled(base[i], e) for i, e in enumerate(es)])
    with make_index(rb, d, tier) as ix:
        ix.append_f64(rows)
        stored = stored_rows(ix, rows, tier)
        _, f0 = counters(ix)
        ix.search(q, 10, None)
        _, f1 = counters(ix)
        n_out = int((~in_band(q)).sum())
        assert f1 - f0 >= n_out, f"{tier}: {f1 - f0} queries fell back, {n_out} are outside the scan's band"
        all_routes(oracle_mod, ix, stored, None, q, f"{tier} d={d} query ladder")


# --------------------------------------------------------------------------- rows across the range
def ladder_rows(rng, rows, q, tier):
    """One near-neighbour of each query per rung, scaled by that rung; the default tier gets their bf16 roundings."""
    extra = []
    for i, e in enumerate(LADDER):
        near = q[i % len(q)] + 0.05 * rng.standard_normal(q.shape[1])
        extra.append(scaled(near, e))
    extra = np.stack(extra)
    if tier == "bf16":
        extra = bf16_f64(extra)
    return extra


@pytest.mark.parametrize("d", [100, 1536])
@pytest.mark.parametrize("tier", TIERS)
def test_row_scale_ladder_and_mutations(rb, oracle_mod, tier, d):
    """A mixed-scale corpus: ordinary rows plus one row per rung, near one of the queries.  Every route must score the
    rungs the reference scores - the 2^-565 row's +-Infinity first, the 2^600 row's +-0 among the zeros.  Then the
    rungs are tombstoned (the answers become the plain corpus's), an ordinary row is overwritten with an extreme one and
    back, and the index is compacted."""
    rng, rows = plain_corpus(d, tier, 10 + d)
    q = rows[rng.choice(N_PLAIN, 8)] + 0.1 * rng.standard_normal((8, d))
    extra = ladder_rows(rng, rows, q, tier)
    allrows = np.concatenate([rows, extra])
    live = np.ones(len(allrows), np.uint8)
    with make_index(rb, d, tier) as ix:
        ix.append_f64(allrows)
        stored = stored_rows(ix, allrows, tier)
        out_of_band = ~in_band(stored if stored.dtype != np.uint16 else bf16_rows_f64(stored))
        _, f0 = counters(ix)
        ix.search(q, 10, None)
        _, f1 = counters(ix)
        if out_of_band[N_PLAIN:].any():
            assert f1 - f0 == len(q), f"{tier}: rows outside the scan's band must send every query to the fallback"
        all_routes(oracle_mod, ix, stored, None, q, f"{tier} d={d} row ladder")

        # tombstoned: the plain corpus's answers
        ix.tombstone(np.arange(N_PLAIN, len(allrows)))
        live[N_PLAIN:] = 0
        for ms in MIN_SCORES:
            got = ix.search(q, 10, ms)
            check(oracle_mod, got, stored, live, q, 10, ms, f"{tier} tombstoned")
            want = oracle_answers(oracle_mod, stored[:N_PLAIN], None, q, 10, ms)
            assert (got[0] == want[0]).all() and (got[2] == want[2]).all()
        check(oracle_mod, ix.search_large(q, 200, None), stored, live, q, 200, None, f"{tier} tombstoned large")

        # an ordinary row overwritten with a tiny one and back; rows with a non-finite element stay out
        slot = 17
        for new in (scaled(q[0], -565), scaled(q[1], 600), np.full(d, np.nan), rows[slot]):
            if tier == "bf16":
                new = bf16_f64(new)
            ix.overwrite_f64(slot, new)
            allrows[slot] = new
            stored = stored_rows(ix, allrows, tier)
            for ms in (None, 0.5):
                check(oracle_mod, ix.search(q, 10, ms), stored, live, q, 10, ms, f"{tier} overwritten")
                check(oracle_mod, ix.search_large(q, 200, ms), stored, live, q, 200, ms, f"{tier} overwritten large")

        # compacted: the rungs are gone for good
        ix.compact()
        stored = stored_rows(ix, allrows[:N_PLAIN], tier)
        for ms in MIN_SCORES:
            check(oracle_mod, ix.search(q, 10, ms), stored, None, q, 10, ms, f"{tier} compacted")
        check(oracle_mod, ix.search_unbounded(q, N_PLAIN + 3, None), stored, None, q, N_PLAIN + 3, None,
              f"{tier} compacted unbounded")


def bf16_rows_f64(u16):
    return (np.asarray(u16, dtype=np.uint32) << 16).view(np.float32).astype(np.float64)


# --------------------------------------------------------------------------- ties of +-Infinity and +-0
@pytest.mark.parametrize("tier", TIERS)
def test_infinity_and_signed_zero_ties_in_every_sort(rb, oracle_mod, tier):
    """A 2^-565 query scores +Infinity on every row with a positive dot and -Infinity on the rest; an ordinary query
    scores the 2^600 rows +0 and -0.  Every device sort (finalize, the exhaustive merge, large-k and the segmented
    sort) must treat these ties as ties and order them by slot."""
    d = 64
    rng = np.random.default_rng(64)
    rows = rng.standard_normal((3000, d))
    if tier != "bf16":
        rows[::7] = scaled(rows[::7], 600)
    else:
        rows = bf16_f64(rows)
    q = rng.standard_normal((6, d))
    q[:3] = scaled(q[:3], -565)
    with make_index(rb, d, tier) as ix:
        ix.append_f64(rows)
        stored = stored_rows(ix, rows, tier)
        all_routes(oracle_mod, ix, stored, None, q, f"{tier} ties")


# --------------------------------------------------------------------------- a Group
@pytest.mark.parametrize("n_dev", [1, 2])
def test_group_across_the_range(rb, oracle_mod, n_dev):
    from common import group_devices
    d = 100
    rng, rows = plain_corpus(d, "device", 77)
    q = rows[rng.choice(N_PLAIN, len(LADDER))] + 0.1 * rng.standard_normal((len(LADDER), d))
    q = np.stack([scaled(q[i], e) for i, e in enumerate(LADDER)])
    allrows = np.concatenate([rows, ladder_rows(rng, rows, q[LADDER.index(0)][None, :], "device")])
    with rb.Group(d, group_devices(n_dev), keep_f64=True) as g:
        g.append_f64(allrows)
        all_routes(oracle_mod, g, allrows, None, q, f"group on {n_dev} GPUs", group=True)


# --------------------------------------------------------------------------- the bound, where the scan still answers
@pytest.mark.parametrize("tier", ["bf16", "device"])
def test_scan_scores_within_the_bound_inside_the_band(rb, tier):
    """Queries and rows scaled anywhere inside [2^-40, 2^40] stay on the scan; debug_scores must stay within the bound
    the proof uses: (d+8) 2^-22 + angle(q, bf16 q) + the corpus angle (KEEP_F64)."""
    from test_gpu_exact_paths import angle_bound
    d, n = 256, 3000
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((n, d))
    rows = np.stack([scaled(r, e) for r, e in zip(rows, rng.integers(-36, 36, n))])
    if tier == "bf16":
        rows = bf16_f64(rows)
    q = rng.standard_normal((12, d))
    q = np.stack([scaled(r, e) for r, e in zip(q, [-37, -30, -20, -1, 0, 1, 20, 30, 37, 0, -36, 36])])
    q = q.astype(np.float32).astype(np.float64)
    assert in_band(rows).all() and in_band(q).all()
    ref = (q @ rows.T) / (np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(rows, axis=1)[None, :])
    eps = (d + 8) * 2.0 ** -22 + angle_bound(q) + (angle_bound(rows).max() if tier != "bf16" else 0.0)
    with make_index(rb, d, tier) as ix:
        ix.append_f64(rows)
        got = ix.debug_scores(q.astype(np.float32)).astype(np.float64)
    err = np.abs(got - ref)
    worst = np.unravel_index(np.argmax(err - eps[:, None]), err.shape)
    assert (err <= eps[:, None]).all(), (worst, err[worst], eps[worst[0]])
