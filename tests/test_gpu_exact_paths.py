"""GPU suite (-m gpu) for the paths that make a search exact when the first pass cannot prove it: the wide retry
(k' = 128) and the exhaustive fp64 fallback (exact_scan_kernel + exact_merge_kernel), on float64 rows (KEEP_F64, on
the device and in pinned host memory) and on bf16 rows.

Every answer is compared with the oracle over the rows the index stores - the float64 rows, or read_rows_bf16 -
ids, counts and the bytes of the float64 scores.  Every case built to reach the retry or the fallback asserts through
the stats() counters that it did, so a later change cannot quietly stop exercising the path.

- The d = 1536 case of random float64 rows with queries near corpus rows, with and without compaction.
- Proof soundness: a first-pass answer whose flag says "proven exact" equals the oracle's.
- Bound soundness: on a KEEP_F64 index the scan's approximate cosine stays within
  eps_q = (d+8) 2^-22 + angle(q, bf16 q) + max_rows angle(c, bf16 c), the bound the proof uses.
- The exhaustive kernel alone (tie groups wider than the retry), exact_scores, and a sweep over tiers, widths, launch
  shapes, k_fetch, min_score, tombstones, compaction, small and unevenly split corpora, and a one-GPU Group."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TIERS = ("device", "host", "bf16")


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def make_index(rb, d, tier, cls=None, **kw):
    cls = cls or rb.Index
    return cls(d, keep_f64=tier != "bf16", f64_on_host=tier == "host", **kw)


def stored_rows(ix, corpus, tier):
    """What the oracle must read: the float64 rows a KEEP_F64 index keeps, or the bf16 rows themselves."""
    return corpus if tier != "bf16" else ix.read_rows_bf16(0, ix.size())


def oracle_answers(oracle_mod, stored, live, q, k, ms):
    """(slots, scores, counts) of the oracle for every query; float64 corpora are answered one query per thread."""
    q = np.ascontiguousarray(q, dtype=np.float64)
    if stored.dtype == np.uint16:
        return oracle_mod.search_batch_verify(stored, q, k, ms, live=live)
    nq = len(q)
    out_s = np.full((nq, k), -1, dtype=np.int64)
    out_v = np.full((nq, k), np.nan)
    out_c = np.zeros(nq, dtype=np.int32)

    def one(b):
        s, v = oracle_mod.search(stored, q[b], k, ms, live=live)
        out_s[b, :len(s)], out_v[b, :len(s)], out_c[b] = s, v, len(s)

    with ThreadPoolExecutor(oracle_mod.host_threads()) as pool:
        list(pool.map(one, range(nq)))
    return out_s, out_v, out_c


def mismatches(got, want):
    """[(query, count got, count wanted, first differing slot positions)] for every query that differs."""
    slots, scores, counts = got
    es, ev, ec = want
    bad = []
    for b in range(len(ec)):
        c = int(ec[b])
        diff = [i for i in range(c) if slots[b, i] != es[b, i] or scores[b, i].tobytes() != ev[b, i].tobytes()]
        if counts[b] != c or diff:
            bad.append((b, int(counts[b]), c, diff[:6]))
    return bad


def check(oracle_mod, got, stored, live, q, k, ms, what=""):
    bad = mismatches(got[:3], oracle_answers(oracle_mod, stored, live, q, k, ms))
    assert not bad, f"{what}: {len(bad)} of {len(q)} queries differ from the oracle (query, count, want, slots): " \
                    f"{bad[:10]}"


def counters(ix):
    st = ix.stats()
    return st["retry_batches"], st["fallback_queries"]


def first_pass(ix, q32, k, ms):
    """search_device_async: the first pass's answers and its per-query flags (1 = not proven exact)."""
    import torch
    B = len(q32)
    qd = torch.from_numpy(np.ascontiguousarray(q32, dtype=np.float32)).cuda()
    s = torch.empty((B, k), dtype=torch.int64, device="cuda")
    v = torch.empty((B, k), dtype=torch.float64, device="cuda")
    c = torch.empty(B, dtype=torch.int32, device="cuda")
    f = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    ix.search_device_async(qd.data_ptr(), B, k, ms, s.data_ptr(), v.data_ptr(), c.data_ptr(), f.data_ptr())
    torch.cuda.synchronize()
    return s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy(), f.cpu().numpy()


def check_proven(oracle_mod, ix, stored, live, q32, k, ms):
    """Every first-pass answer flagged 0 ("proven exact") is the oracle's.  Returns how many were flagged 1."""
    s, v, c, f = first_pass(ix, q32, k, ms)
    assert set(np.unique(f)) <= {0, 1}
    proven = np.flatnonzero(f == 0)
    if len(proven):
        qp = q32[proven].astype(np.float64)
        bad = mismatches((s[proven], v[proven], c[proven]), oracle_answers(oracle_mod, stored, live, qp, k, ms))
        bad = [(int(proven[t[0]]),) + t[1:] for t in bad]
        assert not bad, f"answers flagged proven exact differ from the oracle (query, count, want, slots): {bad[:10]}"
    return int((f == 1).sum())


# --------------------------------------------------------------------------- the reported case
D_REPORTED, N_REPORTED, KEEP_EVERY = 1536, 200000, 10


@pytest.fixture(scope="module")
def reported_corpus(rb):
    """200 000 torch.randn float64 rows at d = 1536, generated on the device as the trim test does.  The tests append
    them from a host copy: a device append reads its rows on the index's own stream, which is not ordered after the
    stream that generated them."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(5)
    rows = np.empty((N_REPORTED, D_REPORTED))
    for first in range(0, N_REPORTED, 25000):
        rows[first:first + 25000] = torch.randn(25000, D_REPORTED, dtype=torch.float64, device="cuda",
                                                generator=g).cpu().numpy()
    return rows


@pytest.mark.parametrize("compacted", [False, True], ids=["whole", "compacted"])
@pytest.mark.parametrize("tier", ["device", "host"])
def test_random_f64_rows_at_1536_match_the_oracle(rb, oracle_mod, reported_corpus, tier, compacted):
    """Random float64 rows at d = 1536, queries = a corpus row + 0.05 noise, no threshold, with and without
    tombstoning 9 rows in 10 and compacting.  At k_fetch 20 the k-th hit sits among near-tied random rows and the
    wide retry settles the batch; at k_fetch 112 the first pass already has k' = 128, so every query it cannot prove
    goes straight to the exhaustive fallback."""
    import torch
    if torch.cuda.mem_get_info()[0] < 8 << 30:
        pytest.skip("needs about 8 GB of free device memory")
    d, n = D_REPORTED, N_REPORTED
    with make_index(rb, d, tier) as ix:
        for first in range(0, n, 25000):
            t = torch.from_numpy(reported_corpus[first:first + 25000]).cuda()
            ix.append_f64_device(t.data_ptr(), len(t))
            del t
        corpus = reported_corpus
        if compacted:
            ix.tombstone(np.setdiff1d(np.arange(n), np.arange(0, n, KEEP_EVERY)))
            ix.compact()
            corpus = np.ascontiguousarray(reported_corpus[::KEEP_EVERY])
        assert ix.size() == len(corpus)
        rng = np.random.default_rng(9)
        q = corpus[rng.choice(len(corpus), 64)] + 0.05 * rng.standard_normal((64, d))
        r0, f0 = counters(ix)
        got = ix.search(q, 20, None)                          # a 64-query batch: graph replay, then the retry
        r1, f1 = counters(ix)
        check(oracle_mod, got, corpus, None, q, 20, None, f"{tier}, k 20: retries {r1 - r0}, fallback {f1 - f0}")
        if not compacted:
            assert r1 > r0, "the batch was meant to take the wide retry"
        got = ix.search(q, 112, None)
        r2, f2 = counters(ix)
        check(oracle_mod, got, corpus, None, q, 112, None, f"{tier}, k 112: fallback {f2 - f1}")
        assert r2 == r1 and f2 > f1, "queries were meant to reach the exhaustive fallback"
        # float32 queries, and the first pass alone: answers flagged proven exact are the oracle's
        q32 = q.astype(np.float32)
        check(oracle_mod, ix.search(q32, 112, None), corpus, None, q32, 112, None, f"{tier}, f32 queries")
        for k in (20, 112):
            check_proven(oracle_mod, ix, corpus, None, q32, k, None)


# --------------------------------------------------------------------------- bound soundness
def bf16_f64(x):
    """float64 -> float32 (RNE) -> bf16 (RNE), as the ingest and prep kernels round, back in float64."""
    from runbookai_b200 import synth
    return synth.bf16_round(np.asarray(x, dtype=np.float64).astype(np.float32)).astype(np.float64)


def angle_bound(x):
    """asin(||x - bf16(x)|| / ||x||) per row."""
    x = np.atleast_2d(x)
    r = np.linalg.norm(x - bf16_f64(x), axis=1) / np.linalg.norm(x, axis=1)
    return np.arcsin(np.minimum(r, 1.0))


@pytest.mark.parametrize("kind", ["gaussian", "positive"])
@pytest.mark.parametrize("d", [768, 1536, 2048])
def test_keep_f64_scan_scores_stay_within_the_proof_bound(rb, kind, d):
    n, b = 5000, 16
    rng = np.random.default_rng(d + (kind == "positive"))
    if kind == "gaussian":
        corpus = rng.standard_normal((n, d))
        q = rng.standard_normal((b, d))
    else:
        corpus = np.abs(rng.standard_normal((n, d))) + 0.05
        q = np.abs(rng.standard_normal((b, d))) + 0.05
        q[0] = 1.0
    # a row whose bf16 rounding is as far from it as rounding gets (each element just under a half step of 2^-7
    # above 1 rounds down): its angle is about 2^-8, far above a random row's, so it sets eps_c_max
    far = (1.0 + 2.0 ** -8 - 2.0 ** -30) * (np.sign(rng.standard_normal(d)) if kind == "gaussian" else 1.0)
    corpus[17] = far
    q[1] = far * (1.0 + 2.0 ** -12 * rng.standard_normal(d))     # and a query that scores that row near 1
    q = q.astype(np.float32).astype(np.float64)                  # debug_scores takes float32 queries
    ref = (q @ corpus.T) / (np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(corpus, axis=1)[None, :])
    c_max = angle_bound(corpus).max()
    assert np.argmax(angle_bound(corpus)) == 17 and c_max > 2.0 ** -9
    eps = (d + 8) * 2.0 ** -22 + angle_bound(q) + c_max
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(corpus)
        got = ix.debug_scores(q.astype(np.float32)).astype(np.float64)
    err = np.abs(got - ref)
    worst = np.unravel_index(np.argmax(err - eps[:, None]), err.shape)
    assert (err <= eps[:, None]).all(), (worst, err[worst], eps[worst[0]])
    assert err[1, 17] <= eps[1]


# --------------------------------------------------------------------------- the exhaustive kernel alone
def tie_corpus(rng, d, n_rand, above, group_size, q_per_group, noise=0.05):
    """Random float64 rows plus, for each group g, `group_size` exact duplicates of one vector u_g and above[g]
    distinct rows nearer the group's queries than u_g.  A query of group g is u_g + w_g + noise, so the duplicates tie
    at ranks above[g] .. above[g] + group_size - 1.  Returns (rows, queries, group of each query, duplicate slots)."""
    rows = [rng.standard_normal((n_rand, d))]
    qs, owner, dup_slots = [], [], []
    n = n_rand
    for g, m in enumerate(above):
        u = rng.standard_normal(d)
        w = 0.2 * rng.standard_normal(d)
        block = np.concatenate([np.repeat(u[None, :], group_size, axis=0),
                                u[None, :] + np.linspace(0.9, 0.3, m)[:, None] * w[None, :]])
        perm = rng.permutation(len(block))
        dup_slots.append(n + np.flatnonzero(perm < group_size))
        rows.append(block[perm])
        n += len(block)
        qs.append(u[None, :] + w[None, :] + noise * rng.standard_normal((q_per_group, d)))
        owner += [g] * q_per_group
    return np.concatenate(rows), np.concatenate(qs), np.array(owner), dup_slots


@pytest.mark.parametrize("tier", TIERS)
def test_tie_groups_wider_than_the_retry_take_the_exhaustive_kernel(rb, oracle_mod, tier):
    """More than 128 exact duplicates at the k-th position of every query: the retry's k' = 128 cannot hold the group,
    so every query of the batch is answered by exact_scan_kernel / exact_merge_kernel."""
    d, B, k = 1536, 48, 20
    rng = np.random.default_rng(1536)
    rows, q, _, _ = tie_corpus(rng, d, 3000, above=[8] * 6, group_size=150, q_per_group=B // 6)
    with make_index(rb, d, tier) as ix:
        ix.append_f64(rows)
        stored = stored_rows(ix, rows, tier)
        r0, f0 = counters(ix)
        got = ix.search(q, k, None)
        r1, f1 = counters(ix)
        check(oracle_mod, got, stored, None, q, k, None, tier)
        assert f1 - f0 == B and r1 - r0 == 1, "every query's tie group is wider than k' = 128"
        assert check_proven(oracle_mod, ix, stored, None, q.astype(np.float32), k, None) == B


@pytest.mark.parametrize("tier", ["device", "host"])
def test_exact_scores_are_the_oracle_scores_at_1536(rb, oracle_mod, tier):
    """exact_scores runs the dot and norm chains the fallback runs: bit-identical to the oracle's cosines."""
    d = 1536
    rng = np.random.default_rng(77)
    rows = rng.standard_normal((20000, d))
    q = rows[[3, 19999, 777]] + 0.05 * rng.standard_normal((3, d))
    dead = [5, 6, 19998]
    with make_index(rb, d, tier) as ix:
        ix.append_f64(rows)
        ix.tombstone(dead)
        got = ix.exact_scores(q)
    for b in range(len(q)):
        want = oracle_mod.scores(rows, q[b])
        want[dead] = np.nan
        assert got[b].tobytes() == want.tobytes(), b


# --------------------------------------------------------------------------- the sweep
# (B, k_fetch, min_score): B = 1 and 64 replay a captured graph, B = 300 is one ungraphed launch (finalize key_cap
# 8192), B = 1100 two sub-batches (1024 queries with key_cap 2048, then 76 with 16384) whose tie queries are all in
# the second one.  "band": a threshold inside the tie band, the median of the tie queries' group scores.
CASES = [(1, 1, None), (1, 20, "band"), (64, 20, None), (64, 112, 0.0), (64, 1, "band"), (300, 1, 0.0),
         (300, 112, "band"), (1100, 20, None), (1100, 112, "band")]
WIDE_ABOVE = [0, 5, 0, 5]      # rows above each wide group: k_fetch 1 falls back for the groups with none
NARROW_ABOVE = [5, 5]


def sweep_corpus(d, seed):
    """2000 random rows, four groups of 150 duplicates (wider than the retry) and two of 60 (held by the retry)."""
    rng = np.random.default_rng(seed)
    wide = tie_corpus(rng, d, 2000, WIDE_ABOVE, group_size=150, q_per_group=1)
    narrow = tie_corpus(rng, d, 0, NARROW_ABOVE, group_size=60, q_per_group=1)
    n_wide = len(wide[0])
    narrow = (narrow[0], narrow[1], narrow[2], [s + n_wide for s in narrow[3]])
    return rng, np.concatenate([wide[0], narrow[0]]), wide, narrow


def tie_queries(rng, d, src, B):
    """B queries; the last min(B, 76 if B > 1024) are the groups' queries with a little more noise (the rest are
    random), so a two-sub-batch batch has every tie query in its second sub-batch.  Returns (queries, tie groups)."""
    n_tie = B if B <= 1024 else B - 1024
    out = rng.standard_normal((B, d))
    groups = np.arange(n_tie) % len(src[3])
    out[B - n_tie:] = src[1][groups] + 0.01 * rng.standard_normal((n_tie, d))
    return out, groups


def group_scores(rows, src, q, groups):
    u = rows[[src[3][g][0] for g in groups]]
    return np.einsum("ij,ij->i", q, u) / (np.linalg.norm(q, axis=1) * np.linalg.norm(u, axis=1))


@pytest.mark.parametrize("d", [1536, 1001, 8])
@pytest.mark.parametrize("tier", TIERS)
def test_retry_and_fallback_sweep(rb, oracle_mod, tier, d):
    rng, rows, wide, narrow = sweep_corpus(d, 100 + d)
    n = len(rows)
    live = np.ones(n, np.uint8)
    with make_index(rb, d, tier) as ix:
        ix.append_f64(rows)
        for phase in ("whole", "tombstoned", "compacted"):
            if phase == "tombstoned":
                # every tenth duplicate of each wide group (135 stay: still wider than the retry) and random rows
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
            stored = stored_rows(ix, rows_now, tier)
            for B, k, ms in CASES:
                for kind in ("wide", "narrow") if (B, k) == (64, 20) else ("wide",):
                    src = wide_now if kind == "wide" else narrow_now
                    q, groups = tie_queries(rng, d, src, B)
                    m = float(np.median(group_scores(rows_now, src, q[B - len(groups):], groups))) if ms == "band" else ms
                    r0, f0 = counters(ix)
                    got = ix.search(q, k, m)
                    r1, f1 = counters(ix)
                    what = f"{tier} d={d} {phase} B={B} k={k} min_score={m} {kind}"
                    check(oracle_mod, got, stored, lv, q, k, m, what)
                    if kind == "narrow":     # 60 duplicates: the retry holds them and nothing falls back
                        assert r1 - r0 == 1 and f1 == f0, what
                    elif ms != "band":       # the duplicates straddle the k-th hit of every group with < k rows above
                        above = np.array(WIDE_ABOVE)[groups]
                        assert f1 - f0 >= int((above < k).sum()) > 0, what
                    else:                    # the group scores sit within the scan's error of the threshold
                        assert f1 - f0 >= 1, what


@pytest.mark.parametrize("tier", TIERS)
@pytest.mark.parametrize("n_rand,above", [(60, [0]), (4853, [0, 7]), (67460, [0, 7])])
def test_fallback_block_split(rb, oracle_mod, tier, n_rand, above):
    """The exhaustive scan splits the rows into min(2 x SMs, ceil(n / 256)) blocks of ceil(n / blocks) rows: a corpus
    below 256 rows (one block), and row counts that leave the last block a short chunk."""
    d, k = 1001, 20
    rng = np.random.default_rng(n_rand)
    rows, q, _, _ = tie_corpus(rng, d, n_rand, above=above, group_size=150, q_per_group=4)
    with make_index(rb, d, tier) as ix:
        ix.append_f64(rows)
        stored = stored_rows(ix, rows, tier)
        _, f0 = counters(ix)
        got = ix.search(q, k, None)
        check(oracle_mod, got, stored, None, q, k, None, f"{tier} n={len(rows)}")
        assert counters(ix)[1] - f0 == len(q)


def test_one_gpu_group_re_answers_through_the_fallback(rb, oracle_mod):
    """A Group whose member cannot prove a query re-answers the batch; at d = 1536 with KEEP_F64 that re-answer goes
    through the exhaustive kernel.  A group of one member and one of two (on one GPU when the machine has one)."""
    from common import group_devices
    d, k = 1536, 20
    rng = np.random.default_rng(4)
    rows, q, _, _ = tie_corpus(rng, d, 9000, above=[3, 0, 9], group_size=150, q_per_group=5)
    for devices in (group_devices(1), group_devices(2)):
        with rb.Group(d, devices, keep_f64=True) as g:
            g.append_f64(rows)
            f0 = g.stats()["fallback_queries"]
            got = g.search(q, k, None)
            check(oracle_mod, got, rows, None, q, k, None, f"group on {devices}")
            st = g.stats()
            assert st["fallback_queries"] > f0 and st["redone_batches"] >= 1
            got = g.search(q[:1], 112, 0.0)
            check(oracle_mod, got, rows, None, q[:1], 112, 0.0, f"group on {devices}, one query")
