"""Executable specification of the scan epilogue's candidate filter (runbookai_b200/csrc/rbk_epilogue.cuh).

The CUDA filter drops a row as soon as its approximate score is not above the query's current threshold, and
the threshold comes from several concurrent sources (start threshold, own-list compaction, a global histogram
fed by every unit's appends, the seeded first tile, thresholds published by other units).  The whole scheme is
exact only if every one of those numbers is a LOWER bound on the query's final k'-th best score.  This model
replays the same rules in numpy - units x tiles x 32-column chunks, per-(unit, query) lists with capacity and
compaction, 1024-bin histogram with "count each row at most once", two seeds per chunk of the first tile,
rotating publisher - on adversarial score streams, and checks the invariants the proof of exactness
(DESIGN.md §6) rests on.  It is a model of the algorithm, not of the kernel: the GPU suite tests the kernel.
"""
import numpy as np
import pytest

BINS, CAP, ROOM, TILE, CHUNK = 1024, 256, 64, 256, 32


def score_bin(a):
    return int(min(max(int((a + 1.0) * (BINS * 0.5)), 0), BINS - 1))


def bin_edge(b):
    e = b * (2.0 / BINS) - 1.0 - 1e-6
    return e - abs(e) * 1e-6


class Unit:
    def __init__(self, rows):
        self.rows = rows            # global row ids of this unit's corpus range, in scan order
        self.thr = -np.inf
        self.tb = -1
        self.list = []              # (score, row)
        self.dropped_max = -np.inf  # best score this unit ever dropped
        self.compactions = 0


def run_filter(scores, n_units, kprime, rng, seed_first_tile=True, publish=True, seed_whole_tile=False):
    """scores: approximate cosine per row (one query).  Units scan disjoint contiguous ranges, interleaved tile
    by tile in a random order (units are not synchronised on the GPU either).  Returns (units, hist)."""
    n = len(scores)
    bounds = [n * u // n_units for u in range(n_units + 1)]
    units = [Unit(np.arange(bounds[u], bounds[u + 1])) for u in range(n_units)]
    hist = np.zeros(BINS, dtype=np.int64)
    gthr = -np.inf
    counted = set()

    def hist_add(row):
        assert row not in counted, "a row was counted twice"
        counted.add(row)
        hist[score_bin(scores[row])] += 1

    def refresh(u):
        cum = 0
        for b in range(BINS - 1, u.tb, -1):
            cum += hist[b]
            if cum >= kprime:
                u.tb = b
                u.thr = max(u.thr, bin_edge(b))
                return True
        return False

    def compact(u):
        u.list.sort(key=lambda e: (-e[0], e[1]))
        for sc, _ in u.list[kprime:]:
            u.dropped_max = max(u.dropped_max, sc)
        if len(u.list) >= kprime:
            u.thr = max(u.thr, u.list[kprime - 1][0])
        u.list = u.list[:kprime]
        u.compactions += 1

    n_tiles = [-(-len(u.rows) // TILE) for u in units]
    progress = [0] * n_units
    while any(progress[i] < n_tiles[i] for i in range(n_units)):
        i = int(rng.choice([j for j in range(n_units) if progress[j] < n_tiles[j]]))
        u, it = units[i], progress[i]
        rows = u.rows[it * TILE:(it + 1) * TILE]
        u.thr = max(u.thr, gthr)                                   # adopt the published threshold
        if publish and it != 0 and i == it % n_units:              # rotating publisher
            u.tb = max(u.tb, score_bin(u.thr) - 1) if u.thr > -np.inf else u.tb
            refresh(u)
            gthr = max(gthr, u.thr)
        nohist = False
        if it == 0 and seed_first_tile:                            # seeding pass: two best rows of every chunk
            step = len(rows) if seed_whole_tile else CHUNK         # whole-tile seeding: two per tile
            for c0 in range(0, len(rows), step):
                ch = rows[c0:c0 + step]
                for r in ch[np.argsort(-scores[ch], kind="stable")[:2]]:
                    if scores[r] > u.thr:
                        hist_add(int(r))
            refresh(u)
            gthr = max(gthr, u.thr)
            nohist = True
        for c0 in range(0, len(rows), 2 * CHUNK):                  # the regular pass, 64 columns per step
            for r in rows[c0:c0 + 2 * CHUNK]:
                if scores[r] > u.thr:
                    u.list.append((float(scores[r]), int(r)))
                    if not nohist:
                        hist_add(int(r))
                else:
                    u.dropped_max = max(u.dropped_max, float(scores[r]))
            if len(u.list) > CAP - ROOM:
                compact(u)
            assert len(u.list) <= CAP
        progress[i] += 1
    return units, hist


def check_invariants(scores, units, hist, kprime):
    order = np.lexsort((np.arange(len(scores)), -scores))          # (score desc, row asc)
    kth = scores[order[kprime - 1]] if len(scores) >= kprime else -np.inf
    # 1. every threshold ever used is a lower bound on the final k'-th best score
    for u in units:
        assert u.thr <= kth, (u.thr, kth)
        assert u.dropped_max <= kth
    # 2. histogram counts are lower bounds on the true counts, bin by bin
    true = np.bincount([score_bin(s) for s in scores], minlength=BINS)
    assert (hist <= true).all()
    # 3. what the finalize kernel's proof uses: with tau = the k'-th best score among ALL kept candidates, no
    #    dropped row scores above tau (ties AT tau may be dropped - the proof's comparison is strict, and a tie
    #    across the boundary sends the query to the wide rescan / exhaustive kernel), so every row strictly
    #    above tau is a candidate
    union = sorted((e for u in units for e in u.list), key=lambda e: (-e[0], e[1]))
    kept = {r for _, r in union}
    if len(union) >= kprime:
        tau = union[kprime - 1][0]
        assert tau <= kth
    else:
        tau = -np.inf
        assert len(kept) == len(scores)          # nothing may have been dropped without k' candidates in hand
    assert max(u.dropped_max for u in units) <= tau
    assert all(int(r) in kept for r in np.nonzero(scores > tau)[0])
    # without ties at the boundary the k' best keys ARE the true top-k'
    if len(scores) > kprime and scores[order[kprime - 1]] > scores[order[kprime]]:
        assert [r for _, r in union[:kprime]] == order[:kprime].tolist()
    return union


@pytest.mark.parametrize("name", ["gaussian", "ascending", "descending", "ties", "two_level", "few_rows"])
@pytest.mark.parametrize("kprime", [32, 128])
def test_filter_thresholds_are_lower_bounds(name, kprime):
    rng = np.random.default_rng(hash((name, kprime)) % (1 << 31))
    n = 6000
    if name == "gaussian":
        s = np.clip(rng.normal(0, 0.05, n), -1, 1)
    elif name == "ascending":            # worst case for a streaming top-k: every row beats the threshold
        s = np.sort(np.clip(rng.normal(0, 0.05, n), -1, 1))
    elif name == "descending":
        s = -np.sort(-np.clip(rng.normal(0, 0.05, n), -1, 1))
    elif name == "ties":                 # 300 exact duplicates straddling every boundary
        s = np.clip(rng.normal(0, 0.05, n), -1, 1)
        s[rng.choice(n, 300, replace=False)] = 0.25
    elif name == "two_level":            # only two distinct values: bins saturate
        s = np.where(rng.random(n) < 0.5, 0.1, 0.1000001)
    else:
        n = 40
        s = np.clip(rng.normal(0, 0.3, n), -1, 1)
    s = s.astype(np.float32).astype(np.float64)
    for n_units in (1, 5):
        for seed_first_tile, publish, whole in ((True, True, False), (True, True, True), (False, True, False),
                                                (True, False, False)):
            units, hist = run_filter(s, n_units, kprime, rng, seed_first_tile, publish, whole)
            check_invariants(s, units, hist, kprime)
    if name == "ascending":              # the model does go through the compaction path
        assert any(u.compactions > 0 for u in units)
