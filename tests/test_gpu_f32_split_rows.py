"""GPU suite (-m gpu) for split float32 exact rows (RBK_INDEX_KEEP_F32_SPLIT).  A split index and a KEEP_F32 twin with
the same placement are fed the same float32-exact rows through every mutation entry point.  On data without a low half
of exactly 0x8000 every output and stats counter must match; with such ties planted the answers must match and the
stored scan bits must follow the split rule (bf16 rounded to nearest, ties away from zero).  Refusals, storage bytes,
extreme values, every tier change into and out of the split, and groups are checked too, against the oracle."""
import numpy as np
import pytest

from common import group_devices
from test_gpu_f32_rows import (STATS, Sequence, answers, assert_same_answers, check_oracle, f32x, group_answers,
                               member_state, same)

pytestmark = pytest.mark.gpu

KEEP64, HOST, KEEP32, F16, SPLIT = 1, 2, 64, 16, 128
PLACES = {"dev": 0, "host": HOST}


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def make(rb, d, flags, cap=0):
    return rb.Index(d, capacity_hint=cap, keep_f64=bool(flags & KEEP64), keep_f32=bool(flags & KEEP32),
                    keep_f32_split=bool(flags & SPLIT), f64_on_host=bool(flags & HOST), scan_f16=bool(flags & F16))


def exact_name(flags):
    return "f64" if flags & KEEP64 else ("f32" if flags & KEEP32 else "f32_split")


def split_hi(rows):
    """The split rule's scan copy of float32-exact values (rbk_internal.h)."""
    u = np.ascontiguousarray(rows, dtype=np.float32).view(np.uint32)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    return np.where(nan, np.uint32(0x7FFF), (u + np.uint32(0x8000)) >> 16).astype(np.uint16)


def retie(a, tie):
    """float32-exact float64 values: tie=False moves every low half of exactly 0x8000 one ulp on; tie=True plants that
    low half in about one element in eight."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).copy()
    if tie:
        pick = (np.arange(u.size).reshape(u.shape) % 8) == 3
        u[pick] = (u[pick] & 0xFFFF0000) | 0x8000
    else:
        u[(u & 0xFFFF) == 0x8000] += 1
    return u.view(np.float32).astype(np.float64)


def split_sequence(d, seed, tie, **kw):
    seq = Sequence(d, seed, **kw)
    for name in ("r64", "rdv", "over1", "over", "tail"):
        setattr(seq, name, retie(getattr(seq, name), tie))
    seq.r32 = retie(seq.r32, tie).astype(np.float32)
    if kw.get("ties", True):
        seq.r64[100:300] = seq.r64[99]
    seq.q = np.concatenate([seq.r64[99:100], seq.q[1:]])
    return seq


def low_halves(corpus):
    return (np.ascontiguousarray(corpus, dtype=np.float32).view(np.uint32) & 0xFFFF)


def assert_same_answers_only(a, b, skip=("debug",)):
    """The same slots, scores and counts (the decision-side outputs may differ)."""
    for key in a:
        if key in skip:
            continue
        assert all(same(x, y) for x, y in zip(a[key][:-1], b[key][:-1])), key


@pytest.mark.parametrize("tie", [False, True], ids=["tie_free", "ties"])
@pytest.mark.parametrize("d", [7, 768])
@pytest.mark.parametrize("place", list(PLACES))
def test_twins_answer_alike(rb, oracle_mod, place, d, tie):
    seq = split_sequence(d, 40 + d, tie)
    corpus, live = seq.oracle_rows()
    assert (low_halves(corpus) == 0x8000).any() == tie
    with make(rb, d, SPLIT | PLACES[place]) as ix, make(rb, d, KEEP32 | PLACES[place]) as twin:
        assert ix.flags == SPLIT | PLACES[place]
        assert same(seq.run(ix), seq.run(twin))               # compaction maps
        assert ix.size() == twin.size() == len(corpus) and ix.count() == twin.count()
        assert same(ix.read_rows_bf16(0, ix.size()), split_hi(corpus))
        a, b = answers(ix, seq.q), answers(twin, seq.q)
        if tie:
            assert_same_answers_only(a, b)
        else:
            assert_same_answers(a, b)                          # every output and counter
            assert same(ix.read_rows_bf16(0, ix.size()), twin.read_rows_bf16(0, twin.size()))
        assert any(x[-1][STATS.index("fallback_queries")] > 0 for x in a.values())   # the tie group's fallback
        for key in (("search", 40, 20, None), ("search", 200, 112, 0.5), ("search", 1, 1, 0.5)):
            B, k, ms = key[1], key[2], key[3]
            check_oracle(oracle_mod, a[key][:3], corpus, live, seq.q[:B], k, ms)
        check_oracle(oracle_mod, a[("large", 700)][:3], corpus, live, seq.q[:6], 700, 0.05)
        check_oracle(oracle_mod, a["unbounded"][:3], corpus, live, seq.q[:3], 5000, None)
        exact = a["exact"][0]
        for b_ in range(3):                                    # exact_scores: the oracle's fp64 cosine of every row
            es, ev = oracle_mod.search(corpus, seq.q[b_], len(corpus), None, live=live)
            assert exact[b_, es].tobytes() == ev.tobytes()
        # storage: 2*dpad + 2*d + 12 device bytes per row (the low halves on the host with RBK_INDEX_ROWS_ON_HOST)
        (dv, hv), (dt, ht) = ix.storage_bytes(), twin.storage_bytes()
        if PLACES[place]:
            assert (dv, hv) == (dt, ht // 2)
        else:
            assert hv == ht == 0 and dt - dv > 0 and (dt - dv) % (2 * d) == 0
        ix.trim(), twin.trim()
        assert_same_answers_only(answers(ix, seq.q[:40]), answers(twin, seq.q[:40]))
        ix.clear(), twin.clear()
        ix.append_f64(seq.tail), twin.append_f64(seq.tail)
        assert_same_answers_only(answers(ix, seq.q[:40]), answers(twin, seq.q[:40]))


def test_storage_bytes_formula(rb):
    d, cap = 1536, 4096
    dpad = (d + 63) // 64 * 64
    with make(rb, d, SPLIT, cap=cap) as a, make(rb, d, SPLIT | HOST, cap=cap) as h, make(rb, d, KEEP32, cap=cap) as t:
        dev, host = a.storage_bytes()
        assert host == 0 and dev == t.storage_bytes()[0] - cap * d * 2
        assert h.storage_bytes() == (dev - cap * d * 2, cap * d * 2)
        # per row: 2*dpad + 2*d + 12 (rows, exact low halves, norm2, inv_norm), plus the tombstone bit and one tile of
        # inv_norm padding, which every tier shares
        per_row = 2 * dpad + 2 * d + 12
        assert dev == cap * per_row + cap // 8 + 256 * 4


def test_extreme_rows(rb, oracle_mod):
    d = 16
    rng = np.random.default_rng(12)
    rows = f32x(rng.standard_normal((400, d)))
    tiny = np.float32(1e-45)
    rows[1, 0], rows[2, 1], rows[3, 2], rows[4, 3] = np.nan, np.inf, -np.inf, -0.0
    rows[5, :] = float(tiny) * np.arange(1, d + 1)              # subnormals only
    rows[6, 4] = float(np.float32(1.1754942e-38))              # the largest subnormal
    rows[7, :] = f32x(np.full(d, 3.4028235e38) * np.where(np.arange(d) % 2, 1, -1))   # float32 max
    rows[8, 0] = float(np.uint32(0x7F7F8000).view(np.float32))  # its scan copy rounds to inf
    rows[9, :] = 0.0                                            # a zero row
    rows[10, 0] = 2.0 ** 50                                     # off-band
    rows[11, :] = retie(rows[11:12], True)[0]
    q = rng.standard_normal((12, d))
    live = np.ones(len(rows), np.uint8)
    for place in PLACES.values():
        with make(rb, d, SPLIT | place) as ix, make(rb, d, KEEP32 | place) as twin:
            ix.append_f64(rows), twin.append_f64(rows)
            ix.overwrite_f64(12, rows[5]), twin.overwrite_f64(12, rows[5])
            corpus = rows.copy()
            corpus[12] = rows[5]
            got, want = answers(ix, q), answers(twin, q)
            assert_same_answers_only(got, want, skip=("debug", "exact"))
            # exact scores: bit for bit, except that a row holding a NaN scores NaN with another payload (the split keeps
            # a NaN a NaN, not its payload bits)
            e, t = got["exact"][0], want["exact"][0]
            nan_row = np.isnan(corpus).any(axis=1)
            assert same(e[:, ~nan_row], t[:, ~nan_row]) and np.isnan(e[:, nan_row]).all() and np.isnan(t[:, nan_row]).all()
            bits = ix.read_rows_bf16(0, ix.size())
            assert same(bits, split_hi(corpus))
            assert bits[1, 0] == 0x7FFF and (bits[8, 0] & 0x7FFF) == 0x7F80
            for k, ms in ((20, None), (5, 0.3)):
                check_oracle(oracle_mod, ix.search(q, k, ms)[:3], corpus, live, q, k, ms)


@pytest.mark.parametrize("entry", ["append_f64", "append_f64_device", "overwrite_f64", "overwrite_f64_batch"])
@pytest.mark.parametrize("bad", [0.1, 1e39])
def test_refusal_leaves_the_index_untouched(rb, entry, bad):
    import torch
    from runbookai_b200._native import RBK_ENOTF32, NotFloat32Error
    d = 32
    rng = np.random.default_rng(19)
    rows = retie(rng.standard_normal((500, d)), True)
    q = rng.standard_normal((20, d))
    with make(rb, d, SPLIT | HOST) as ix:
        ix.append_f64(rows)
        ix.tombstone([4, 9])
        before = (ix.size(), ix.count(), ix.storage_bytes(), ix.search(q, 20, None)[:3], ix.exact_scores(q[:2]),
                  ix.read_rows_bf16(0, ix.size()))
        new = f32x(rng.standard_normal((3, d)))
        new[1, 7] = bad
        with pytest.raises(NotFloat32Error) as e:
            if entry == "append_f64":
                ix.append_f64(new)
            elif entry == "append_f64_device":
                t = torch.from_numpy(new).cuda()
                ix.append_f64_device(t.data_ptr(), len(new))
            elif entry == "overwrite_f64":
                ix.overwrite_f64(11, new[1])
            else:
                ix.overwrite_f64_batch([11, 4, 12], new)
        assert e.value.status == RBK_ENOTF32
        after = (ix.size(), ix.count(), ix.storage_bytes(), ix.search(q, 20, None)[:3], ix.exact_scores(q[:2]),
                 ix.read_rows_bf16(0, ix.size()))
        assert before[:3] == after[:3]
        assert all(same(x, y) for x, y in zip(before[3], after[3]))
        assert same(before[4], after[4]) and same(before[5], after[5])


def test_tier_changes_into_and_out_of_the_split(rb, oracle_mod):
    d = 768
    seq = split_sequence(d, 23, True)
    corpus, live = seq.oracle_rows()
    path = [SPLIT, KEEP32, SPLIT | HOST, KEEP64 | F16, SPLIT, KEEP32 | F16, SPLIT | HOST, KEEP64 | HOST, SPLIT | HOST,
            KEEP32 | HOST | F16, SPLIT, KEEP64, SPLIT]
    with make(rb, d, path[0]) as ix:
        seq.run(ix)
        start = answers(ix, seq.q)
        for flags in path[1:]:
            ix.set_tier(exact_rows=exact_name(flags), f64_on_host=bool(flags & HOST), scan_f16=bool(flags & F16))
            assert ix.flags == flags
            assert_same_answers_only(start, answers(ix, seq.q))
            with make(rb, d, flags) as fresh:
                seq.run(fresh)
                assert ix.storage_bytes() == fresh.storage_bytes()
                bits = (lambda x: x.read_rows_f16 if flags & F16 else x.read_rows_bf16)
                assert same(bits(ix)(0, ix.size()), bits(fresh)(0, fresh.size())), flags
            if flags & SPLIT:
                assert same(ix.read_rows_bf16(0, ix.size()), split_hi(corpus))
        check_oracle(oracle_mod, ix.search(seq.q[:20], 20, None)[:3], corpus, live, seq.q[:20], 20, None)


def test_narrowing_into_the_split_refused_by_a_tombstoned_slot(rb):
    from runbookai_b200._native import NotFloat32Error
    d = 48
    rng = np.random.default_rng(5)
    rows = f32x(rng.standard_normal((400, d)))
    rows[123, 5] = 0.1
    q = rng.standard_normal((8, d))
    with make(rb, d, KEEP64) as ix:
        ix.append_f64(rows)
        ix.tombstone([123])
        before = (ix.flags, ix.storage_bytes(), ix.search(q, 20, None)[:3], ix.read_rows_bf16(0, 400))
        for host in (False, True):
            with pytest.raises(NotFloat32Error):
                ix.set_tier(exact_rows="f32_split", f64_on_host=host)
            assert (ix.flags, ix.storage_bytes()) == before[:2]
            assert all(same(x, y) for x, y in zip(before[2], ix.search(q, 20, None)[:3]))
            assert same(before[3], ix.read_rows_bf16(0, 400))
        ix.compact()
        ix.set_tier(exact_rows="f32_split")
        assert ix.flags == SPLIT


def test_group_of_three(rb, oracle_mod):
    from runbookai_b200._native import NotFloat32Error
    n, d = 3, 64
    rng = np.random.default_rng(77)
    rows = retie(rng.standard_normal((4096 * n + 500, d)), True)
    rows[1000:1200] = rows[999]
    q = np.concatenate([rows[999:1000], rng.standard_normal((199, d))])
    dead = np.arange(50, 4096 * n, 7)
    devs = group_devices(n)
    with rb.Group(d, devs, keep_f32_split=True) as g, rb.Group(d, devs, keep_f32=True) as t, \
            make(rb, d, SPLIT) as single:
        for x in (g, t, single):
            x.append_f64(rows[:4096 * n - 10])
            x.append_f32(rows[4096 * n - 10:].astype(np.float32))
            x.overwrite_f64_batch([3, 4097], rows[:2])
            x.tombstone(dead)
        m = g.compact()                                        # moves rows between members
        assert same(m, t.compact()) and same(m, single.compact())
        a, b = group_answers(g, q), group_answers(t, q)
        for key in a:
            assert all(same(x, y) for x, y in zip(a[key], b[key])), key
        s = {("search", 200, 20, None): single.search(q[:200], 20, None)[:3]}
        assert all(same(x, y) for x, y in zip(a[("search", 200, 20, None)], s[("search", 200, 20, None)]))
        corpus = rows.copy()
        corpus[3], corpus[4097] = rows[0], rows[1]
        keep = np.ones(len(rows), bool)
        keep[dead] = False
        check_oracle(oracle_mod, a[("search", 200, 20, None)], corpus[keep], np.ones(keep.sum(), np.uint8), q, 20, None)
        state = (g.size(), g.count(), member_state(rb, g))
        bad = f32x(rng.standard_normal((4096 * n, d)))
        bad[-1, 0] = 0.1
        with pytest.raises(NotFloat32Error):
            g.append_f64(bad)
        assert (g.size(), g.count(), member_state(rb, g)) == state
        for flags in (KEEP64 | HOST, SPLIT | HOST, KEEP32 | F16, SPLIT):
            g.set_tier(exact_rows=exact_name(flags), f64_on_host=bool(flags & HOST), scan_f16=bool(flags & F16))
            assert g.flags == flags
            got = group_answers(g, q)
            for key in a:
                assert all(same(u, v) for u, v in zip(a[key], got[key])), (flags, key)
