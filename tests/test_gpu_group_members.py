"""GPU suite (-m gpu): device groups of two to eight members co-located on one GPU (the device list repeats device 0,
so the members exchange their blocks with device copies instead of NCCL).  Each group is fed the same calls as a single
Index and must answer bit for bit as it does - slots, score bytes, counts and the -1 / NaN tails - on every route; a
subset of every case is also checked against the fp64 oracle.

The cases aim at what only runs when G > 1: the block-cyclic global slots that the finalize, exhaustive, large-k and
segmented-sort kernels write, the merge over G blocks (ties between members, k_eff-wide blocks, empty and partly
filled members, the OR of the exactness flags and the re-answer it triggers), appends split across blocks and members,
overwrites and tombstones split by member, compaction across members and a tier change on every member.  The merge
kernel is also tested on its own against oracle.merge_lists."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_compact import all_answers, assert_same_through_map, expected_map
from test_gpu_exact_paths import check, counters, tie_corpus
from test_gpu_group_compact import append, bit_equal, corpus_for, make, member_rows, routes, runs_dead

pytestmark = pytest.mark.gpu

BLOCK = 4096
GS = (2, 3, 5, 8)
APPENDS = (1, 4095, 4097, 7000, 3 * BLOCK)     # straddle block and member boundaries
PEAK = {"redone_batches": 0, "fallback_queries": 0}


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


@pytest.fixture(scope="module", autouse=True)
def report_peaks():
    yield
    print(f"\n[group members] most redone_batches of one group {PEAK['redone_batches']}, "
          f"most fallback_queries of one group {PEAK['fallback_queries']}")


def note(g):
    st = g.stats()
    for key in PEAK:
        PEAK[key] = max(PEAK[key], st[key])
    return st


def colocated(G):
    return [0] * G


def expected_member_rows(G, n, d):
    """rbk_group_plan.h member_rows: the rows member d holds when the group has n slots."""
    full, rem = divmod(n, BLOCK)
    return (full // G) * BLOCK + (BLOCK if d < full % G else 0) + (rem if d == full % G else 0)


def member_slots(G, n, d):
    """The global slots member d holds, in its local row order."""
    s = np.arange(n)
    return s[(s // BLOCK) % G == d]


def append_in_pieces(handles, tier, rows):
    """The same appends on every handle, in the APPENDS sizes in turn; each returns its first global slot."""
    r0, i = 0, 0
    while r0 < len(rows):
        m = APPENDS[i % len(APPENDS)]
        for h in handles:
            assert append(h, tier, rows[r0:r0 + m]) == r0
        r0 += m
        i += 1


def check_members(rb, g, ix, tier):
    """Every member's size is member_rows(G, BLOCK, n, d), and its stored rows are its block-cyclic slice of the
    index's."""
    G, n = len(g.devices), ix.size()
    lib = rb._native.lib
    stored = (ix.read_rows_f16 if tier == "f16" else ix.read_rows_bf16)(0, n)
    for d in range(G):
        assert lib.rbk_index_size(C.c_void_p(lib.rbk_group_member(g._h, d))) == expected_member_rows(G, n, d), d
        assert (member_rows(rb, g, d, tier) == stored[member_slots(G, n, d)]).all(), d


def answers(h, q, hit):
    """routes() (search f64 / f32 at k 1 / 20 / 112, search_large 500 / 4096, unbounded 4097, three thresholds) plus k 7,
    min_score 0.0 and a score some row has exactly, B of 1 / 129 / 1100, search_large 113 / 1000, search_unbounded
    at count, count + 7 and far above it, and the exact scores."""
    out = routes(h, q, 4097)
    for k in (1, 7, 20, 112):
        out[(k, 0.0, "f64")] = h.search(q, k, 0.0)[:3]
        out[(k, hit, "f64")] = h.search(q, k, hit)[:3]
    for ms in (None, 0.5):
        out[(7, ms, "f64")] = h.search(q, 7, ms)[:3]
    big = np.concatenate([q] * (1 + 1100 // len(q)))[:1100]
    for B in (1, 129, 1100):
        out[(20, None, f"B{B}")] = h.search(big[:B], 20, None)[:3]
        out[(20, 0.5, f"B{B}f32")] = h.search(big[:B].astype(np.float32), 20, 0.5)[:3]
    for k in (113, 1000):
        out[(k, None, "large")] = h.search_large(q, k, None)[:3]
    out[(4096, hit, "large")] = h.search_large(q, 4096, hit)[:3]
    c = h.count()
    for k in (max(c, 1), c + 7, far_k(c)):
        out[(k, None, "unbounded4")] = h.search_unbounded(q[:4], k, None)[:3]
    out["exact"] = (h.exact_scores(q),)
    return out


def far_k(count):
    return 3 * count + 5000


def oracle_subset(oracle_mod, got, stored, live, q, hit, count, what):
    for key in ((20, None, "f64"), (112, 0.5, "f64"), (7, hit, "f64"), (1, 0.0, "f64"), (1000, None, "large"),
                (4096, hit, "large")):
        check(oracle_mod, got[key], stored, live, q, key[0], key[1], f"{what} {key}")
    for k in (count + 7, far_k(count)):
        check(oracle_mod, got[(k, None, "unbounded4")], stored, live, q[:4], k, None, f"{what} unbounded {k}")


def hit_score(ix, q):
    """A score that a row has exactly: query 0's fifth hit (a min_score equal to it keeps that row)."""
    s, v, c, _ = ix.search(q[:1], 5, None)
    return float(v[0, c[0] - 1])


# --------------------------------------------------------------------------- placement and every route
SIZES = {"under_one_block": lambda G: 1000, "one_block": lambda G: BLOCK, "last_member_thin": lambda G: (G - 1) * BLOCK + 1,
         "partial_middle": lambda G: 2 * G * BLOCK + 777}


@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("G", GS)
def test_placement_and_every_route(rb, oracle_mod, G, size):
    """Only member 0 holds rows (n < BLOCK, n = BLOCK), the last member holds nothing or one row, a partial block sits
    on a middle member: the group answers every route as the index does, and as the oracle does."""
    from runbookai_b200 import synth
    n, d = SIZES[size](G), 64
    corpus = synth.random_corpus(n, d, 10 * G + len(size))
    q = synth.random_queries(33, d, G).astype(np.float64)
    synth.plant_neighbours(corpus, q.astype(np.float32), 3, G)
    with rb.Group(d, colocated(G)) as g, rb.Index(d) as ix:
        append_in_pieces((g, ix), "bf16", corpus)
        assert g.size() == g.count() == n
        check_members(rb, g, ix, "bf16")
        hit = hit_score(ix, q)
        got = answers(g, q, hit)
        assert bit_equal(got, answers(ix, q, hit))
        oracle_subset(oracle_mod, got, corpus, None, q, hit, n, f"G={G} n={n}")
        note(g)


def test_many_scan_tiles_per_member(rb, oracle_mod):
    """150k x 64 over three members: every member's scan runs many corpus tiles."""
    from runbookai_b200 import synth
    n, d, G = 150_000, 64, 3
    corpus = synth.random_corpus(n, d, 150)
    q = synth.random_queries(33, d, 151).astype(np.float64)
    synth.plant_neighbours(corpus, q.astype(np.float32), 10, 152)
    with rb.Group(d, colocated(G)) as g, rb.Index(d) as ix:
        append_in_pieces((g, ix), "bf16", corpus)
        check_members(rb, g, ix, "bf16")
        hit = hit_score(ix, q)
        got = answers(g, q, hit)
        assert bit_equal(got, answers(ix, q, hit))
        oracle_subset(oracle_mod, got, corpus, None, q, hit, n, "150k rows on 3 members")


@pytest.mark.parametrize("G", [2, 8])
def test_empty_and_all_tombstoned_groups(rb, G):
    from runbookai_b200 import synth
    d = 64
    q = synth.random_queries(5, d, 3).astype(np.float64)
    with rb.Group(d, colocated(G)) as g, rb.Index(d) as ix:
        empty = all_answers(ix, q)
        assert bit_equal(all_answers(g, q), empty)
        # the quiet NaN every other path writes (an empty index once wrote all-ones bits instead)
        assert all((c == 0).all() and (s == -1).all() and (v.view(np.uint64) == 0x7FF8000000000000).all()
                   for s, v, c in empty.values())
        assert g.exact_scores(q).shape == (5, 0)
        corpus = synth.random_corpus(G * BLOCK + 5, d, 4)
        for h in (g, ix):
            h.append_bf16(corpus)
            h.tombstone(np.arange(len(corpus)))
        got = routes(g, q, 4097)
        assert bit_equal(got, routes(ix, q, 4097))
        assert all((c == 0).all() for _, _, c in got.values())
        assert np.isnan(g.exact_scores(q)).all()


# --------------------------------------------------------------------------- ties across members
@pytest.mark.parametrize("G", GS)
def test_ties_across_members(rb, oracle_mod, G):
    """A group of identical rows spread over every member's blocks, more on each member than its first-pass candidate
    margin, with the k cut inside it: the members' proofs fail, the flag travels through the merge, the batch is
    re-answered, and the tied slots come back in ascending order.  Exact ties on both sides of block boundaries, and
    a min_score equal to the tie score."""
    from runbookai_b200 import synth
    n, d = 2 * G * BLOCK + 777, 64
    corpus = synth.random_corpus(n, d, 200 + G)
    q = synth.random_queries(9, d, 201 + G).astype(np.float64)
    pair = np.array([BLOCK - 1, BLOCK, 2 * BLOCK - 1, 2 * BLOCK])       # member 0 | 1 | ... block boundaries
    corpus[pair] = synth.f32_to_bf16_bits((q[1] * 0.7).astype(np.float32))
    dup = np.setdiff1d(np.linspace(0, n - 1, max(300, 60 * G)).astype(np.int64), pair)
    assert len(np.unique((dup // BLOCK) % G)) == G
    corpus[dup] = synth.f32_to_bf16_bits((q[0] * 0.5).astype(np.float32))
    with rb.Group(d, colocated(G)) as g, rb.Index(d) as ix:
        for h in (g, ix):
            h.append_bf16(corpus)
        r0 = note(g)["redone_batches"]
        s, v, c, _ = g.search(q, 20, None)
        assert note(g)["redone_batches"] > r0, "the tie group was meant to fail the members' proofs"
        assert s[0].tolist() == dup[:20].tolist()
        assert bit_equal({0: (s, v, c)}, {0: ix.search(q, 20, None)[:3]})
        assert g.search(q[1:2], 2, None)[0][0].tolist() == [BLOCK - 1, BLOCK]
        assert g.search(q[1:2], 4, None)[0][0].tolist() == pair.tolist()
        tie = float(v[0, 0])
        got, want = {}, {}
        for h, out in ((g, got), (ix, want)):
            out["k112"] = h.search(q, 112, tie)[:3]
            out["k20f32"] = h.search(q.astype(np.float32), 20, None)[:3]
            out["large"] = h.search_large(q, 4096, tie)[:3]
            out["large_all"] = h.search_large(q, 4096, None)[:3]
            out["unbounded"] = h.search_unbounded(q[:4], n + 7, tie)[:3]
            out["unbounded_all"] = h.search_unbounded(q[:4], 5000, None)[:3]
        assert bit_equal(got, want)
        assert got["k112"][2][0] == 112 and got["large"][2][0] == len(dup)       # min_score is inclusive
        assert got["large"][0][0, :len(dup)].tolist() == dup.tolist()
        check(oracle_mod, (s, v, c), corpus, None, q, 20, None, f"G={G} k 20")
        check(oracle_mod, got["k112"], corpus, None, q, 112, tie, f"G={G} k 112 at the tie score")
        check(oracle_mod, got["large"], corpus, None, q, 4096, tie, f"G={G} large 4096 at the tie score")
        check(oracle_mod, got["unbounded_all"], corpus, None, q[:4], 5000, None, f"G={G} unbounded 5000")
        note(g)


# --------------------------------------------------------------------------- the exhaustive kernels with G > 1
@pytest.mark.parametrize("G", [2, 5, 8])
def test_exhaustive_kernel_on_a_member_past_slot_0(rb, oracle_mod, G):
    """Tie groups of 150 exact duplicates (wider than the retry's 128) on member 1: its queries are answered by the
    exhaustive kernel there, whose slots must be global ones."""
    d, k = 256, 20
    rng = np.random.default_rng(G)
    ties, q, _, dup = tie_corpus(rng, d, BLOCK + 50, above=[3, 0], group_size=150, q_per_group=4)
    rows = np.concatenate([ties, rng.standard_normal((G * BLOCK, d))])
    assert all(((s // BLOCK) % G == 1).all() for s in dup)
    with rb.Group(d, colocated(G), keep_f64=True) as g, rb.Index(d, keep_f64=True) as ix:
        for h in (g, ix):
            h.append_f64(rows)
        _, f0 = counters(g)
        got = {"k20": g.search(q, k, None)[:3], "k112": g.search(q, 112, 0.0)[:3]}
        assert counters(g)[1] > f0, "the tie groups were meant to reach the exhaustive kernel"
        assert bit_equal(got, {"k20": ix.search(q, k, None)[:3], "k112": ix.search(q, 112, 0.0)[:3]})
        check(oracle_mod, got["k20"], rows, None, q, k, None, f"G={G} k {k}")
        check(oracle_mod, got["k112"], rows, None, q, 112, 0.0, f"G={G} k 112")
        note(g)


@pytest.mark.parametrize("G", [3, 8])
def test_off_band_rows_send_every_member_to_the_exhaustive_kernel(rb, oracle_mod, G):
    """A float64 row below the scan's band (its bf16 copy is zero) on every member: every member answers through the
    exhaustive kernel, and search_large through large_emit_all, with the oracle's global slots."""
    from float_range_cases import scaled
    from test_gpu_float_range import all_routes
    d = 100
    rng = np.random.default_rng(300 + G)
    n = G * BLOCK + 500
    rows = rng.standard_normal((n, d))
    q = rows[rng.choice(n, 4)] + 0.1 * rng.standard_normal((4, d))
    for m in range(G):
        rows[m * BLOCK + 10 + m] = scaled(q[m % 4] + 0.05 * rng.standard_normal(d), -160)
    with rb.Group(d, colocated(G), keep_f64=True) as g, rb.Index(d, keep_f64=True) as ix:
        for h in (g, ix):
            h.append_f64(rows)
        _, f0 = counters(g)
        got = g.search(q, 10, None)[:3]
        per = [p["fallback_queries"] for p in note(g)["per_device"]]
        assert counters(g)[1] > f0 and all(f > 0 for f in per), per
        assert bit_equal({0: got}, {0: ix.search(q, 10, None)[:3]})
        assert bit_equal(routes(g, q, n + 7), routes(ix, q, n + 7))
        all_routes(oracle_mod, g, rows, None, q, f"{G} co-located members, off-band rows", group=True)
        note(g)


# --------------------------------------------------------------------------- tiers
@pytest.mark.parametrize("G,tier", [(3, "bf16"), (3, "device"), (3, "host"), (3, "f16"), (2, "bf16"), (2, "host"),
                                    (5, "bf16"), (5, "host"), (8, "bf16"), (8, "host")])
def test_tiers(rb, oracle_mod, G, tier):
    n, d = 2 * G * BLOCK + 777, 96
    corpus = corpus_for(tier, n, d, 400 + G)
    rng = np.random.default_rng(401 + G)
    if tier == "bf16":
        from runbookai_b200 import synth
        q = synth.random_queries(12, d, 402 + G).astype(np.float64)
    else:
        q = corpus[rng.choice(n, 12)] + 0.2 * rng.standard_normal((12, d))
    live = runs_dead(n, rng, 0.3)
    with make(rb, rb.Group, d, tier, colocated(G)) as g, make(rb, rb.Index, d, tier) as ix:
        append_in_pieces((g, ix), tier, corpus)
        for h in (g, ix):
            h.tombstone(np.flatnonzero(live == 0))
        check_members(rb, g, ix, tier)
        got = routes(g, q, 4097)
        assert bit_equal(got, routes(ix, q, 4097))
        assert g.exact_scores(q).tobytes() == ix.exact_scores(q).tobytes()
        for key in ((20, None, "f64"), (112, 0.05, "f32"), (4096, 0.05, "large"), (4097, None, "unbounded")):
            qq = q.astype(np.float32).astype(np.float64) if key[2] == "f32" else q
            check(oracle_mod, got[key], corpus, live, qq, key[0], key[1], f"{tier} G={G} {key}")
        note(g)


# --------------------------------------------------------------------------- mutation
@pytest.mark.parametrize("G", [3, 8])
def test_overwrite_tombstone_clear_trim(rb, oracle_mod, G):
    """overwrite_f64_batch across members (a slot named twice takes its last row; a tombstoned slot returns
    RBK_EINVAL after the live slots on the other members are written), tombstones, clear and re-append, trim."""
    n, d = 2 * G * BLOCK + 777, 80
    rng = np.random.default_rng(500 + G)
    rows = rng.standard_normal((n, d))
    q = rows[rng.choice(n, 9)] + 0.2 * rng.standard_normal((9, d))
    live = np.ones(n, np.uint8)
    dead = BLOCK + 100                                                    # on member 1
    live[dead] = 0
    slots = np.array([m * BLOCK + 5 for m in range(2 * G)] + [dead, 5, (G - 1) * BLOCK + 6])
    new = rng.standard_normal((len(slots), d))
    new[0] = q[0] * 2.0
    new[-2] = q[1] * 3.0                                                  # slot 5 again: this row wins
    with rb.Group(d, colocated(G), keep_f64=True) as g, rb.Index(d, keep_f64=True) as ix:
        for h in (g, ix):
            h.append_f64(rows)
            h.tombstone([dead])
            with pytest.raises(rb.RbkError) as e:
                h.overwrite_f64_batch(slots, new)
            assert e.value.status == rb._native.RBK_EINVAL
        for s, r in zip(slots, new):
            if s != dead:
                rows[s] = r
        got = routes(g, q, 4097)
        assert bit_equal(got, routes(ix, q, 4097))
        assert got[(1, None, "f64")][0][1, 0] == 5                          # the last row named for slot 5
        check(oracle_mod, got[(20, None, "f64")], rows, live, q, 20, None, f"G={G} after overwrite")
        gone = np.concatenate([np.arange(BLOCK - 50, BLOCK + 50), rng.choice(n, 500, replace=False)])
        live[gone] = 0
        for h in (g, ix):
            h.tombstone(gone)
        got = routes(g, q, 4097)
        assert bit_equal(got, routes(ix, q, 4097))
        check(oracle_mod, got[(112, 0.05, "f64")], rows, live, q, 112, 0.05, f"G={G} after tombstones")
        for h in (g, ix):
            h.clear()
            assert h.size() == 0 and h.search(q, 5, None)[2].sum() == 0
        again = rows[:BLOCK * G + 3]
        append_in_pieces((g, ix), "device", again)
        assert bit_equal(routes(g, q, 4097), routes(ix, q, 4097))
        g.trim()
        ix.trim()
        got = routes(g, q, 4097)
        assert bit_equal(got, routes(ix, q, 4097))
        check(oracle_mod, got[(20, 0.05, "f64")], again, None, q, 20, 0.05, f"G={G} re-appended and trimmed")
        note(g)


# --------------------------------------------------------------------------- compaction
def assert_like_a_new_group(rb, g, f, tier):
    lib = rb._native.lib
    for m in range(len(g.devices)):
        assert lib.rbk_index_size(C.c_void_p(lib.rbk_group_member(g._h, m))) == \
            lib.rbk_index_size(C.c_void_p(lib.rbk_group_member(f._h, m))), m
        assert (member_rows(rb, g, m, tier) == member_rows(rb, f, m, tier)).all(), m


def test_compaction_leaves_trailing_members_empty(rb, oracle_mod):
    """Five members, survivors that fill fewer than two blocks: members 2-4 end up empty, then appends refill them."""
    G, n, d = 5, 2 * 5 * BLOCK + 777, 96
    rng = np.random.default_rng(600)
    corpus = rng.standard_normal((n, d))
    q = corpus[rng.choice(n, 6)] + 0.1 * rng.standard_normal((6, d))
    live = np.zeros(n, np.uint8)
    live[rng.choice(n, BLOCK + 1500, replace=False)] = 1
    keep = live.astype(bool)
    with rb.Group(d, colocated(G), keep_f64=True) as g, rb.Group(d, colocated(G), keep_f64=True) as f:
        g.append_f64(corpus)
        g.tombstone(np.flatnonzero(~keep))
        before = routes(g, q, 3000)
        m = g.compact()
        assert (m == expected_map(live)).all()
        f.append_f64(corpus[keep])
        assert g.size() == g.count() == f.size() == keep.sum()
        lib = rb._native.lib
        assert [lib.rbk_index_size(C.c_void_p(lib.rbk_group_member(g._h, i))) for i in range(2, G)] == [0, 0, 0]
        assert_like_a_new_group(rb, g, f, "device")
        after = routes(g, q, 3000)
        assert bit_equal(after, routes(f, q, 3000))
        assert_same_through_map(before, after, m)
        check(oracle_mod, after[(20, None, "f64")], corpus[keep], None, q, 20, None, "after compaction")
        extra = rng.standard_normal((3 * BLOCK + 5, d))
        for h in (g, f):
            assert h.append_f64(extra) == keep.sum()
        assert_like_a_new_group(rb, g, f, "device")
        final = routes(g, q, 3000)
        assert bit_equal(final, routes(f, q, 3000))
        rows = np.concatenate([corpus[keep], extra])
        check(oracle_mod, final[(112, 0.05, "f64")], rows, None, q, 112, 0.05, "after compaction and appends")


def test_compaction_of_a_large_keep_f64_corpus_across_members(rb, oracle_mod):
    """200k x 1536 KEEP_F64 over three members, half the rows deleted in runs: the plan moves the survivors in many
    64 MB staging chunks between members."""
    from runbookai_b200 import synth
    G, n, d = 3, 200_000, 1536
    corpus = synth.random_corpus(n, d, 700)
    q = synth.random_queries(16, d, 701).astype(np.float64)
    synth.plant_neighbours(corpus, q.astype(np.float32), 30, 702)
    live = runs_dead(n, np.random.default_rng(703))
    keep = live.astype(bool)
    with rb.Group(d, colocated(G), keep_f64=True) as g:
        g.append_bf16(corpus)
        g.tombstone(np.flatnonzero(~keep))
        m = g.compact()
        assert (m == expected_map(live)).all()
        with rb.Group(d, colocated(G), keep_f64=True) as f:
            f.append_bf16(corpus[keep])
            assert_like_a_new_group(rb, g, f, "bf16")
            got = {"f64": g.search(q, 20, 0.05)[:3], "large": g.search_large(q[:8], 1000, 0.05)[:3]}
            assert bit_equal(got, {"f64": f.search(q, 20, 0.05)[:3], "large": f.search_large(q[:8], 1000, 0.05)[:3]})
        check(oracle_mod, got["f64"], corpus[keep], None, q, 20, 0.05, "200k x 1536 after compaction")


# --------------------------------------------------------------------------- the layers above
def test_vector_store_and_retriever_over_co_located_members(rb, tmp_path, monkeypatch):
    from common import HashEmbedder, OracleIndex
    from test_compact_host import QUERIES, _answers, _docs
    from runbookai_b200 import embedder, retriever
    from runbookai_b200.retriever import KnowledgeRetriever
    from runbookai_b200.vector_store import VectorStore
    embedder.configure(HashEmbedder(64))
    monkeypatch.setattr(retriever, "_COMPACT_MIN_DEAD", 64)
    try:
        rnd = [0]
        vs = VectorStore(str(tmp_path / "vectors.db"), index_factory=lambda d, dev: rb.Group(d, colocated(3)))
        ref = VectorStore(str(tmp_path / "ref.db"), index_factory=lambda d, dev: OracleIndex(d))
        r = KnowledgeRetriever({"storePath": str(tmp_path / "k.db"), "sources": [lambda since: _docs(rnd[0])]},
                               vector_store=vs)
        rr = KnowledgeRetriever({"storePath": str(tmp_path / "rk.db"), "sources": [lambda since: _docs(rnd[0])]},
                                vector_store=ref)
        for rnd[0] in range(6):
            r.sync()
            rr.sync()
            assert _answers(vs) == _answers(ref) and _answers(vs, 60) == _answers(ref, 60)
            assert r.search(QUERIES[0]) == rr.search(QUERIES[0])
        assert isinstance(vs._index, rb.Group) and vs._index.stats()["devices"] == 3
        r.close()
        rr.close()
    finally:
        embedder.reset()


# --------------------------------------------------------------------------- the merge kernel on its own
def shard_lists(rng, G, B, k):
    """Per shard and query, a list sorted by (score desc, slot asc) of 0..k entries.  Slots are unique across the shards
    of a query and interleave between them; scores come from a small set (long runs of equal scores, negative ones,
    -0.0 and +0.0, which compare equal so the slot decides).  Some shards and some queries are empty; the entries past
    a list's count hold junk the merge must not read."""
    values = np.array([0.75, 0.5, 0.5 + 2.0 ** -40, 0.0, -0.0, -0.25, -1.0, 1e-300, -1e-300])
    slots = np.full((G, B, k), 12345678, np.int64)
    scores = np.full((G, B, k), np.inf)
    counts = rng.integers(0, k + 1, (G, B)).astype(np.int32)
    counts[rng.random((G, B)) < 0.2] = 0
    counts[:, rng.random(B) < 0.1] = 0
    if B > 1:
        counts[:, 0] = 0                                                    # an all-empty query
        counts[:, -1] = k                                                   # a query with every shard full
    if G > 1:
        counts[1] = 0                                                       # an all-empty shard
    for b in range(B):
        total = int(counts[:, b].sum())
        pool = rng.permutation(4 * G * k + 16)[:total]
        owner = np.repeat(np.arange(G), counts[:, b])
        for g in range(G):
            s = pool[owner == g]
            v = values[rng.integers(0, len(values), len(s))] if rng.random() < 0.7 else rng.standard_normal(len(s))
            order = np.lexsort((s, -v))
            slots[g, b, :len(s)], scores[g, b, :len(s)] = s[order], v[order]
    return slots, scores, counts


@pytest.mark.parametrize("k", [1, 24, 112, 4096])
@pytest.mark.parametrize("B", [1, 33, 200])
@pytest.mark.parametrize("G", [1, 2, 5, 8, 16])
def test_merge_kernel_against_the_oracle(rb, oracle_mod, native, G, B, k):
    import torch
    rng = np.random.default_rng(G * 1000 + B * 10 + k)
    slots, scores, counts = shard_lists(rng, G, B, k)
    es, ev, ec = oracle_mod.merge_lists([(slots[g], scores[g], counts[g]) for g in range(G)], k)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream

    def merged(os_, ov, oc):
        torch.cuda.synchronize()
        s, v, c = os_.cpu().numpy(), ov.cpu().numpy(), oc.cpu().numpy()
        assert (c == ec).all()
        assert (s == es).all() and v.tobytes() == ev.tobytes()              # -0.0 vs +0.0 and the NaN tails too

    out = (torch.empty((B, k), dtype=torch.int64, device=dev), torch.empty((B, k), dtype=torch.float64, device=dev),
           torch.empty((B,), dtype=torch.int32, device=dev))
    gs, gv, gc = (torch.from_numpy(x).to(dev) for x in (slots, scores, counts))
    native.merge_topk_device(0, stream, G, B, k, gs.data_ptr(), gv.data_ptr(), gc.data_ptr(),
                             *(t.data_ptr() for t in out))
    merged(*out)
    # packed blocks, as one all-gather (or the co-located copies) leaves them, with exactness flags
    blk, off_f = native.packed_block_bytes(B, k), native.packed_flags_offset(B, k)
    flags = (rng.random((G, B)) < 0.15).astype(np.int32)
    packed = np.zeros(G * blk, np.uint8)
    for g in range(G):
        o = g * blk
        packed[o:o + B * k * 8] = slots[g].reshape(-1).view(np.uint8)
        packed[o + B * k * 8:o + B * k * 16] = scores[g].reshape(-1).view(np.uint8)
        packed[o + B * k * 16:o + B * k * 16 + B * 4] = counts[g].view(np.uint8)
        packed[o + off_f:o + off_f + B * 4] = flags[g].view(np.uint8)
    pd = torch.from_numpy(packed).to(dev)
    of = torch.zeros((B + 1,), dtype=torch.int32, device=dev)
    want = np.bitwise_or.reduce(flags, axis=0)
    for rep in (1, 2, 3):
        out = tuple(torch.empty_like(t) for t in out)
        native.merge_topk_packed_device(0, stream, G, B, k, pd.data_ptr(), *(t.data_ptr() for t in out), of.data_ptr())
        merged(*out)
        got = of.cpu().numpy()
        assert (got[:B] == want).all() and got[B] == rep * int(want.sum())   # the running dirty count
