"""GPU suite (-m gpu) for the fp16 scan of float64-backed indexes (RBK_INDEX_SCAN_F16).

- Storage bits: read_rows_f16 is numpy's scaled round-to-nearest-even with subnormals flushed, for tiny, huge, wide
  and zero rows from float64, float32 and bf16 sources on the host and on the device; rows a bf16 index never matches
  are never matched here either.
- Bound soundness: debug_scores stays within eps_q = (d+8) 2^-22 + angle(q, h_q 2^-e) + max_rows angle(c, h_c 2^-e).
- Differential: a bf16-tier and an fp16-tier index fed the same calls give the oracle's answers, and each other's, on
  every search route, on both float64 placements and in a one-GPU Group.
- The point of the feature: queries whose k-th and k'-th exact scores sit between the two tiers' bounds make the bf16
  tier retry and let the fp16 tier prove its first pass.
- Tie groups wider than the retry still reach the exhaustive kernel."""
import numpy as np
import pytest

from test_gpu_exact_paths import check, check_proven, counters, oracle_answers, tie_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


# --------------------------------------------------------------------------- the storage rule in numpy
def f16_scale(x):
    """Per-row e = 15 - E, E the frexp exponent of max |x| over the finite elements (0 for rows without any)."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    amax = np.where(np.isfinite(x), np.abs(x), 0.0).max(axis=1)
    e = 15 - np.frexp(amax)[1]
    return np.where(amax > 0, e, 0)


def f16_store(x):
    """(fp16 values, e) of the rule: RNE_f16(x * 2^e) in one rounding, subnormal results flushed to signed zeros."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    e = f16_scale(x)
    with np.errstate(over="ignore", invalid="ignore"):
        h = np.ldexp(x, e[:, None]).astype(np.float16)
    sub = np.isfinite(h) & (h != 0) & (np.abs(h) < np.float16(2.0 ** -14))
    h[sub] = np.where(np.signbit(h[sub]), np.float16(-0.0), np.float16(0.0))
    return h, e


def f16_angle(x):
    """asin(||x 2^e - h|| / ||x 2^e||) per row: the angle between x and what the index stores for it."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    h, e = f16_store(x)
    y = np.ldexp(x, e[:, None])
    r = np.linalg.norm(y - h.astype(np.float64), axis=1) / np.linalg.norm(y, axis=1)
    return np.arcsin(np.minimum(r, 1.0))


def bf16_f64(x):
    from runbookai_b200 import synth
    return synth.bf16_round(np.asarray(x, dtype=np.float64).astype(np.float32)).astype(np.float64)


def bf16_angle(x):
    x = np.atleast_2d(x)
    r = np.linalg.norm(x - bf16_f64(x), axis=1) / np.linalg.norm(x, axis=1)
    return np.arcsin(np.minimum(r, 1.0))


def acc_eps(d):
    return (d + 8) * 2.0 ** -22


def bits_to_f64(bits):
    return (np.asarray(bits, dtype=np.uint32) << 16).view(np.float32).astype(np.float64)


# --------------------------------------------------------------------------- 1. storage bits
def awkward_rows(rng, d):
    rows = rng.standard_normal((12, d))
    rows[0] *= 1e-300                                                       # far below fp16 and float32
    rows[1] *= 1e300                                                        # far above float32
    rows[2] = 0.0
    rows[3] = np.ldexp(np.sign(rng.standard_normal(d)), rng.integers(-40, 1, d))   # 41 binades in one row
    rows[4] = np.ldexp(rng.standard_normal(d), rng.integers(-60, 60, d))    # 120 binades
    rows[5, : d // 2] = 0.0
    rows[6] = -0.0
    rows[6, 3] = 2.0 ** -1070                                               # a subnormal double as the maximum
    rows[7] *= 2.0 ** 14 + 8                                                # maxima near the top of the scale
    rows[8] = 1.0 + 2.0 ** -11 - 2.0 ** -30                                 # every element just under a half step
    rows[9, 0] = -(2.0 ** 20)                                               # one large element, the rest flushed
    return rows


@pytest.mark.parametrize("d", [96, 1001])
def test_stored_bits_follow_the_scaled_rne_rule(rb, d):
    import torch
    rng = np.random.default_rng(d)
    f64 = awkward_rows(rng, d)
    f32 = rng.standard_normal((10, d)).astype(np.float32)
    f32[0] *= np.float32(1e-30)
    f32[1, :5] = 0.0
    f32[2] = np.ldexp(np.sign(rng.standard_normal(d)), rng.integers(-35, 1, d)).astype(np.float32)
    from runbookai_b200 import synth
    bf = synth.f32_to_bf16_bits(rng.standard_normal((10, d)).astype(np.float32) * np.float32(3e-20))
    n1 = len(f64)
    # slots: f64 from the host | f64 from the device | f32 rows, then overwritten from f64 | bf16 host | bf16 device
    want = np.concatenate([f64, f64, f64[: len(f32)], bits_to_f64(bf), bits_to_f64(bf)])
    for on_host in (False, True):
        with rb.Index(d, keep_f64=True, f64_on_host=on_host, scan_f16=True) as ix:
            ix.append_f64(f64)
            t = torch.from_numpy(f64).cuda()
            torch.cuda.synchronize()
            ix.append_f64_device(t.data_ptr(), n1)
            ix.append_f32(f32)
            f32_bits = ix.read_rows_f16(2 * n1, len(f32))
            assert (f32_bits == f16_store(f32.astype(np.float64))[0].view(np.uint16)).all(), "float32 source"
            ix.append_bf16(bf)
            ix.overwrite_f64_batch(2 * n1 + np.arange(len(f32)), f64[: len(f32)])
            tb = torch.from_numpy(bf.view(np.int16)).cuda()
            torch.cuda.synchronize()
            ix.append_bf16_device(tb.data_ptr(), len(bf))
            got = ix.read_rows_f16(0, ix.size())
            with pytest.raises(rb.RbkError, match="rbk_index_read_rows_f16"):
                ix.read_rows_bf16(0, 1)
        h, _ = f16_store(want[: len(got)])
        assert got.shape == h.shape
        bad = np.argwhere(got != h.view(np.uint16))
        assert len(bad) == 0, (on_host, bad[:5], got[tuple(bad[0])], h.view(np.uint16)[tuple(bad[0])])
        assert not ((got & 0x7C00) == 0)[got & 0x7FFF != 0].any(), "no stored value is subnormal"
    with rb.Index(d, keep_f64=True) as ix:
        ix.append_f64(f64)
        with pytest.raises(rb.RbkError, match="rbk_index_read_rows_bf16"):
            ix.read_rows_f16(0, 1)


def test_rows_dead_under_bf16_are_dead_under_f16(rb):
    """The scan's liveness of a row (a finite 1/||c||) is the bf16 tier's: rows past float32's range, rows whose bf16
    rounding is zero, zero rows and rows with non-finite elements never get an approximate score in either tier."""
    d = 64
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((8, d))
    rows[0] *= 1e300
    rows[1] *= 1e-300
    rows[2] = 0.0
    rows[3, 5] = np.inf
    rows[4, 6] = np.nan
    rows[5] *= 1e-42                                              # bf16 keeps some of these (float32 subnormals)
    q = rng.standard_normal((3, d)).astype(np.float32)
    out = []
    for f16 in (False, True):
        with rb.Index(d, keep_f64=True, scan_f16=f16) as ix:
            ix.append_f64(rows)
            out.append(np.isnan(ix.debug_scores(q)))
    assert (out[0] == out[1]).all(), (out[0], out[1])
    assert out[1][:, [0, 1, 2, 3, 4]].all() and not out[1][:, [6, 7]].any()


# --------------------------------------------------------------------------- 2. bound soundness
@pytest.mark.parametrize("kind", ["gaussian", "positive"])
@pytest.mark.parametrize("d", [768, 1536, 2048])
def test_f16_scan_scores_stay_within_the_proof_bound(rb, kind, d):
    n, b = 5000, 16
    rng = np.random.default_rng(d + (kind == "positive"))
    if kind == "gaussian":
        corpus = rng.standard_normal((n, d)) * np.exp(rng.uniform(-20, 20, (n, 1)))
        q = rng.standard_normal((b, d))
    else:
        corpus = np.abs(rng.standard_normal((n, d))) + 0.05
        q = np.abs(rng.standard_normal((b, d))) + 0.05
        q[0] = 1.0
    # the worst fp16 rounding: every element just under a half step above 1 rounds down, an angle of about 2^-11
    far = (1.0 + 2.0 ** -11 - 2.0 ** -30) * (np.sign(rng.standard_normal(d)) if kind == "gaussian" else 1.0)
    corpus[17] = far
    q[1] = far * (1.0 + 2.0 ** -14 * rng.standard_normal(d))     # and a query that scores that row near 1
    q = q.astype(np.float32).astype(np.float64)
    ref = (q @ corpus.T) / (np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(corpus, axis=1)[None, :])
    ang = f16_angle(corpus)
    assert np.argmax(ang) == 17 and ang.max() > 2.0 ** -12
    eps = acc_eps(d) + f16_angle(q) + ang.max()
    eps_bf16 = acc_eps(d) + bf16_angle(q) + bf16_angle(corpus).max()
    assert (eps < eps_bf16).all()
    with rb.Index(d, keep_f64=True, scan_f16=True) as ix:
        ix.append_f64(corpus)
        got = ix.debug_scores(q.astype(np.float32)).astype(np.float64)
    err = np.abs(got - ref)
    worst = np.unravel_index(np.argmax(err - eps[:, None]), err.shape)
    assert (err <= eps[:, None]).all(), (worst, err[worst], eps[worst[0]])
    assert err[1, 17] <= eps[1]


# --------------------------------------------------------------------------- 3. differential
PLACEMENTS = ("device", "host", "group")


def make(rb, d, placement, f16):
    if placement == "group":
        return rb.Group(d, [0], keep_f64=True, scan_f16=f16)
    return rb.Index(d, keep_f64=True, f64_on_host=placement == "host", scan_f16=f16)


def routes(rb, ix, q, live):
    """Every search route's answer: {name: (slots, scores, counts)}."""
    import torch
    out = {}
    q64 = np.ascontiguousarray(q)
    out["graph"] = ix.search(q64[:64], 20, None)[:3]
    out["general"] = ix.search(q64, 20, 0.0)[:3]
    out["f32"] = ix.search(q64[:64].astype(np.float32), 24, None)[:3]
    out["large"] = ix.search_large(q64[:40], 600, None)[:3]
    out["unbounded"] = ix.search_unbounded(q64[:8], 5000, 0.0)[:3]
    out["exact_scores"] = ix.exact_scores(q64[:4])
    if isinstance(ix, rb.Index):
        B, k = 64, 20
        qd = torch.from_numpy(q64[:B].astype(np.float32)).cuda()
        s = torch.empty((B, k), dtype=torch.int64, device="cuda")
        v = torch.empty((B, k), dtype=torch.float64, device="cuda")
        c = torch.empty(B, dtype=torch.int32, device="cuda")
        ix.search_device(qd.data_ptr(), B, k, None, s.data_ptr(), v.data_ptr(), c.data_ptr())
        torch.cuda.synchronize()
        out["device"] = (s.cpu().numpy(), v.cpu().numpy(), c.cpu().numpy())
    return out


ROUTE_ARGS = {"graph": (64, 20, None, np.float64), "general": (None, 20, 0.0, np.float64),
              "f32": (64, 24, None, np.float32), "large": (40, 600, None, np.float64),
              "unbounded": (8, 5000, 0.0, np.float64), "device": (64, 20, None, np.float32)}


def check_routes(oracle_mod, got, corpus, live, q, what):
    for name, ans in got.items():
        if name == "exact_scores":
            for b in range(len(ans)):
                want = oracle_mod.scores(corpus, q[b])
                if live is not None:
                    want[live == 0] = np.nan
                assert ans[b].tobytes() == want.tobytes(), (what, name, b)
            continue
        B, k, ms, dt = ROUTE_ARGS[name]
        qq = q[:B].astype(dt).astype(np.float64)
        check(oracle_mod, ans, corpus, live, qq, k, ms, f"{what} {name}")


def same(a, b):
    for name in a:
        if name == "exact_scores":
            assert a[name].tobytes() == b[name].tobytes(), name
        else:
            for x, y in zip(a[name], b[name]):
                assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), name


@pytest.mark.parametrize("placement", PLACEMENTS)
def test_bf16_and_f16_tiers_answer_alike_through_every_mutation(rb, oracle_mod, placement):
    d = 384
    rng = np.random.default_rng(384)
    base = rng.standard_normal((64, d))
    def batch(n):   # clustered rows, so near-ties and retries happen, at scales from 1e-6 to 1e6
        rows = base[rng.integers(0, 64, n)] + 0.15 * rng.standard_normal((n, d))
        return rows * np.exp(rng.uniform(-14, 14, (n, 1)))
    q = base[rng.integers(0, 64, 300)] + 0.15 * rng.standard_normal((300, d))
    with make(rb, d, placement, False) as a, make(rb, d, placement, True) as b:
        corpus = np.zeros((0, d))
        live = np.zeros(0, dtype=np.uint8)
        for n in (700, 1500, 3000, 2200):                                  # several growths
            rows = batch(n)
            for ix in (a, b):
                ix.append_f64(rows)
            corpus = np.concatenate([corpus, rows])
            live = np.concatenate([live, np.ones(n, dtype=np.uint8)])
        rows32 = batch(500).astype(np.float32)
        for ix in (a, b):
            ix.append_f32(rows32)
        corpus = np.concatenate([corpus, rows32.astype(np.float64)])
        live = np.concatenate([live, np.ones(500, dtype=np.uint8)])
        slots = rng.choice(len(corpus), 300, replace=False)
        slots[-1] = slots[0]                                                # a repeated slot takes its last row
        over = batch(300)
        dead = np.setdiff1d(rng.choice(len(corpus), 900, replace=False), slots)
        for ix in (a, b):
            ix.tombstone(dead)
        live[dead] = 0
        for ix in (a, b):
            ix.overwrite_f64_batch(slots, over)
        corpus[slots[:-1]] = over[:-1]
        corpus[slots[-1]] = over[-1]
        with pytest.raises(rb.RbkError, match="tombstoned"):               # a dead slot stays dead in both tiers
            a.overwrite_f64_batch(np.array([dead[0]]), batch(1))
        with pytest.raises(rb.RbkError, match="tombstoned"):
            b.overwrite_f64_batch(np.array([dead[0]]), batch(1))
        ga, gb = routes(rb, a, q, live), routes(rb, b, q, live)
        check_routes(oracle_mod, gb, corpus, live, q, f"{placement} f16 before compaction")
        same(ga, gb)
        if placement != "group":
            for ix in (a, b):
                ix.compact()
            corpus, live = np.ascontiguousarray(corpus[live == 1]), None
            dev = [ix.storage_bytes() for ix in (a, b)]
            assert dev[0] == dev[1], dev                                   # the same bytes per row in both tiers
        for ix in (a, b):
            ix.trim()
        more = batch(4000)
        for ix in (a, b):
            ix.append_f64(more)
        corpus = np.concatenate([corpus, more])
        if live is not None:
            live = np.concatenate([live, np.ones(len(more), dtype=np.uint8)])
        ga, gb = routes(rb, a, q, live), routes(rb, b, q, live)
        check_routes(oracle_mod, gb, corpus, live, q, f"{placement} f16 after compaction and trim")
        same(ga, gb)
        for ix in (a, b):
            ix.clear()
            ix.append_f64(more[:1000])
        ga, gb = routes(rb, a, q, None), routes(rb, b, q, None)
        check_routes(oracle_mod, gb, more[:1000], None, q, f"{placement} f16 after clear")
        same(ga, gb)


# --------------------------------------------------------------------------- 4. the point of the feature
def planted_case(d, n_rand, k, n_lo, s_hi, gap, seed):
    """Random rows plus, per query, k rows of exact score s_hi and n_lo rows of exact score s_hi - gap against it (the
    planted rows are s q^ + sqrt(1 - s^2) u, u orthogonalised exactly against q^ and scaled at random)."""
    rng = np.random.default_rng(seed)
    B = 8
    q = rng.standard_normal((B, d))
    rows = [rng.standard_normal((n_rand, d))]
    for b in range(B):
        qh = q[b] / np.linalg.norm(q[b])
        for s, m in ((s_hi, k), (s_hi - gap, n_lo)):
            u = rng.standard_normal((m, d))
            u -= (u @ qh)[:, None] * qh[None, :]
            u -= (u @ qh)[:, None] * qh[None, :]
            u /= np.linalg.norm(u, axis=1)[:, None]
            rows.append((s * qh[None, :] + np.sqrt(1 - s * s) * u) * np.exp(rng.uniform(-5, 5, (m, 1))))
    return np.concatenate(rows), q


def kth(v, k):
    return np.sort(v)[::-1][k - 1]


def test_f16_proves_what_bf16_must_retry(rb, oracle_mod):
    d, k, kprime = 1536, 20, 48
    corpus, q = planted_case(d, 3000, k, 100, 0.6, 1.9e-3, seed=15)
    q = q.astype(np.float32).astype(np.float64)
    cn = corpus / np.linalg.norm(corpus, axis=1)[:, None]
    exact = (q / np.linalg.norm(q, axis=1)[:, None]) @ cn.T
    # the device's bounds, from the data: the bf16 one from below, the fp16 one from above
    eps_b = (acc_eps(d) + bf16_angle(q) + bf16_angle(corpus).max()) * (1 - 1e-6)
    eps_h = (acc_eps(d) + f16_angle(q) + f16_angle(corpus).max()) * (1 + 1e-6) + 1e-12
    cb = bf16_f64(q) @ (bf16_f64(corpus)).T / (np.linalg.norm(bf16_f64(q), axis=1)[:, None]
                                                * np.linalg.norm(bf16_f64(corpus), axis=1)[None, :])
    hq, _ = f16_store(q)
    hc, _ = f16_store(corpus)
    hq, hc = hq.astype(np.float64), hc.astype(np.float64)
    ch = hq @ hc.T / (np.linalg.norm(hq, axis=1)[:, None] * np.linalg.norm(hc, axis=1)[None, :])
    for b in range(len(q)):
        s_k = kth(exact[b], k)
        # bf16: the k'-th approximate score is at least kth(cb) - acc, and s_k does not clear it by eps_b
        assert s_k <= kth(cb[b], kprime) - acc_eps(d) + eps_b[b], b
        # fp16: the k'-th approximate score is at most kth(ch) + acc, and s_k clears it by more than eps_h
        assert s_k > kth(ch[b], kprime) + acc_eps(d) + eps_h[b], b
    want = oracle_answers(oracle_mod, corpus, None, q, k, None)
    for f16 in (False, True):
        with rb.Index(d, keep_f64=True, scan_f16=f16) as ix:
            ix.append_f64(corpus)
            r0, f0 = counters(ix)
            got = ix.search(q, k, None)
            r1, f1 = counters(ix)
            check(oracle_mod, got, corpus, None, q, k, None, f"f16={f16}")
            assert [s.tobytes() for s in got[:3]] == [s.tobytes() for s in want], f16
            if f16:
                assert r1 == r0 and f1 == f0, "the fp16 tier proves its first pass"
            else:
                assert r1 > r0, "the bf16 tier cannot prove its first pass"


# --------------------------------------------------------------------------- 5. wide tie groups
@pytest.mark.parametrize("on_host", [False, True], ids=["device", "host"])
def test_tie_groups_wider_than_the_retry_reach_the_exhaustive_kernel(rb, oracle_mod, on_host):
    d, B, k = 1536, 48, 20
    rng = np.random.default_rng(1536)
    rows, q, _, _ = tie_corpus(rng, d, 3000, above=[8] * 6, group_size=150, q_per_group=B // 6)
    with rb.Index(d, keep_f64=True, f64_on_host=on_host, scan_f16=True) as ix:
        ix.append_f64(rows)
        r0, f0 = counters(ix)
        got = ix.search(q, k, None)
        r1, f1 = counters(ix)
        check(oracle_mod, got, rows, None, q, k, None, "f16")
        assert f1 - f0 == B and r1 - r0 == 1, "every query's tie group is wider than k' = 128"
        assert check_proven(oracle_mod, ix, rows, None, q.astype(np.float32), k, None) == B
