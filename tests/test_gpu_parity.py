"""GPU suite (-m gpu): the CUDA path, called through the C ABI, against the oracle on the
same seeded inputs.  Bar: returned ids identical, fp64 scores bit-identical (the engine
re-ranks in the reference's exact operation order), approximate scan scores within the
engine's own error bound.  Nothing here reads the reference checkout."""
import json
import math
import os

import numpy as np
import pytest

from common import HashEmbedder, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def check_against_oracle(oracle_mod, ix, corpus, queries, k_fetch, min_score, live=None, nq=None, slot_base=0):
    slots, scores, counts, _ = ix.search(queries, k_fetch, min_score)
    nq = queries.shape[0] if nq is None else min(nq, queries.shape[0])
    es, ev, ec = oracle_mod.search_batch_mt(corpus, queries[:nq].astype(np.float64), k_fetch, min_score, live=live)
    for b in range(nq):
        assert counts[b] == ec[b], (b, counts[b], ec[b])
        assert (slots[b, :ec[b]] == es[b, :ec[b]] + slot_base).all(), (b, slots[b], es[b])
        assert (scores[b, :ec[b]] == ev[b, :ec[b]]).all(), (b, scores[b], ev[b])   # bit-exact fp64
        assert (slots[b, ec[b]:] == -1).all() and np.isnan(scores[b, ec[b]:]).all()
    return slots, scores, counts


def test_golden_fixtures_on_gpu(rb, oracle_mod):
    g = load_golden()
    for c in g["cases"]:
        with rb.Index(c["d"]) as ix:
            ix.append_f64(c["rows_f64"])
            k_fetch = 2 * (c["top_k"] or 10)
            s, v, n, _ = ix.search(c["query_f64"], k_fetch, c["min_score"] or 0.5)
            assert s[0, :n[0]].tolist() == c["scan_slots"]
            assert v[0, :n[0]].tolist() == c["scan_scores_f64"].tolist()
            s, v, n, _ = ix.search(c["query_f64"], c["top_k"], None)     # findMostSimilar
            assert s[0, :n[0]].tolist() == c["fms_slots"]
            assert v[0, :n[0]].tolist() == c["fms_scores_f64"].tolist()


def test_scan_scores_within_error_bound(rb):
    from runbookai_b200 import synth
    for n, d, b in ((1000, 384, 5), (777, 100, 3), (2500, 768, 130), (600, 1536, 2)):
        c = synth.random_corpus(n, d, 1)
        c[17] = 0                                   # zero row -> NaN
        q = synth.random_queries(b, d, 2)
        with rb.Index(d) as ix:
            ix.append_bf16(c)
            got = ix.debug_scores(q)
        cf = synth.bf16_bits_to_f32(c).astype(np.float64)
        qf = q.astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            ref = (qf @ cf.T) / (np.linalg.norm(qf, axis=1)[:, None] * np.linalg.norm(cf, axis=1)[None, :])
        assert np.isnan(got[:, 17]).all()
        ok = np.ones(n, dtype=bool)
        ok[17] = False
        eps = (d + 8) * 2.0 ** -22                 # rbk::accumulation_eps
        assert np.abs(got[:, ok] - ref[:, ok]).max() <= eps


@pytest.mark.parametrize("n,d,b,k,planted,min_score", [
    (10_000, 384, 1, 5, 10, 0.5),       # BASELINE config 1 (reference-scale)
    (10_000, 384, 1, 5, 0, 0.5),        # same, nothing passes the threshold
    (1, 8, 1, 1, 0, None),              # single row
    (255, 64, 3, 5, 6, 0.5),            # < one tile
    (257, 72, 3, 5, 6, None),           # one row into the second tile, d not a multiple of 64
    (5000, 100, 7, 16, 20, 0.5),        # d % 8 != 0 (padded pitch)
    (30_000, 768, 130, 16, 32, 0.5),    # 2 query blocks, ragged
    (40_000, 1024, 256, 32, 0, None),   # config-4 width, k_fetch 64
    (20_000, 1536, 5, 56, 0, None),     # the reference's default d, max k_fetch
    (150_000, 768, 64, 16, 0, None),    # many tiles per CTA: running thresholds + compaction
    (4000, 100, 200, 8, 12, 0.5),       # two query blocks with a padded, non-multiple-of-64 dim
    (60_000, 384, 1100, 16, 0, None),   # > 1024 queries: two sub-batches (1024 + 76) in one call
    (3000, 2048, 140, 5, 4, 0.5),       # wide rows (64 k-blocks of 32), two query blocks
])
def test_parity_shapes(rb, oracle_mod, n, d, b, k, planted, min_score):
    from runbookai_b200 import synth
    corpus = synth.random_corpus(n, d, 100 + n % 97)
    queries = synth.random_queries(b, d, 200 + d)
    if planted:
        synth.plant_neighbours(corpus, queries, min(planted, n // max(b, 1)), 300)
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        check_against_oracle(oracle_mod, ix, corpus, queries, 2 * k if 2 * k <= 112 else k, min_score, nq=64)
        assert ix.stats()["fallback_queries"] == 0 or planted   # random data never needs the fallback


def test_exact_ties_and_the_exhaustive_fallback(rb, oracle_mod):
    """Duplicate rows give exact score ties across the candidate boundary: the proof of
    exactness fails, the exhaustive fp64 kernel answers, order is still (score, slot)."""
    from runbookai_b200 import synth
    n, d = 6000, 128
    corpus = synth.random_corpus(n, d, 7)
    q = synth.random_queries(3, d, 8)
    row = synth.f32_to_bf16_bits(q[0] * 0.5)
    dup_slots = np.random.default_rng(9).choice(n, 200, replace=False)
    corpus[dup_slots] = row                            # 200 rows with cosine exactly equal
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        s, v, c = check_against_oracle(oracle_mod, ix, corpus, q, 20, 0.5)
        assert s[0, :20].tolist() == sorted(dup_slots.tolist())[:20]
        assert ix.stats()["fallback_queries"] >= 1 and ix.stats()["retry_batches"] >= 1   # 200 ties > 128 candidates
        check_against_oracle(oracle_mod, ix, corpus, q, 112, None)


def test_moderate_tie_groups_are_settled_by_the_wide_rescan(rb, oracle_mod):
    """70 duplicated rows tie across a 48-candidate boundary: the first proof fails, one more scan with
    k' = 128 holds the whole tie group and proves the answer - no exhaustive pass."""
    from runbookai_b200 import synth
    n, d = 20000, 128
    corpus = synth.random_corpus(n, d, 17)
    q = synth.random_queries(5, d, 18)
    dup_slots = np.random.default_rng(19).choice(n, 70, replace=False)
    corpus[dup_slots] = synth.f32_to_bf16_bits(q[1] * 0.25)
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        s, v, c = check_against_oracle(oracle_mod, ix, corpus, q, 20, None)
        assert s[1, :20].tolist() == sorted(dup_slots.tolist())[:20]
        st = ix.stats()
        assert st["retry_batches"] >= 1 and st["fallback_queries"] == 0
        check_against_oracle(oracle_mod, ix, corpus, q, 20, 0.5)
        assert ix.stats()["fallback_queries"] == 0


def test_multi_device_index_single_process(rb, oracle_mod):
    """multi_device.py on real indexes: one host process, rows dealt block-cyclically over two device indexes
    (two GPUs when the box has them, else both on GPU 0), host merge == the oracle on the whole corpus."""
    import torch
    from runbookai_b200 import synth
    from runbookai_b200.multi_device import MultiDeviceIndex
    n, d = 30_000, 256
    corpus = synth.random_corpus(n, d, 41)
    q = synth.random_queries(9, d, 42)
    synth.plant_neighbours(corpus, q, 12, 43)
    devs = [0, 1] if torch.cuda.device_count() > 1 else [0, 0]
    with MultiDeviceIndex(d, devices=devs, block=1024) as ix:
        for r0 in range(0, n, 7000):                       # appends that straddle blocks and devices
            assert ix.append_bf16(corpus[r0:r0 + 7000]) == r0
        check_against_oracle(oracle_mod, ix, corpus, q, 24, 0.5)
        check_against_oracle(oracle_mod, ix, corpus, q, 24, None)
        dead = np.random.default_rng(44).choice(n, 500, replace=False)
        ix.tombstone(dead)
        live = np.ones(n, dtype=np.uint8)
        live[dead] = 0
        check_against_oracle(oracle_mod, ix, corpus, q, 24, None, live=live)
        assert ix.count() == n - 500 and ix.stats()["devices"] == 2


def test_group_one_handle_many_gpus_matches_oracle(rb, oracle_mod):
    """rbk_group_*: the in-library multi-GPU index (one host process, one call per search: per-GPU scans, ONE
    ncclAllGather of the packed blocks, merge kernel, one synchronisation).  Two GPUs when the box has them (NCCL
    path), else a one-GPU group (same code minus the collective).  Rows are dealt out in 4096-row blocks, so appends
    straddle blocks and devices; ties across devices, tombstones, bulk overwrite and the dirty-flag re-answer path
    (a tie group larger than any candidate margin) are all checked against the oracle on the whole corpus."""
    import torch
    from runbookai_b200 import Group, synth
    n, d = 30_000, 256
    corpus = synth.random_corpus(n, d, 141)
    q = synth.random_queries(9, d, 142)
    synth.plant_neighbours(corpus, q, 12, 143)
    corpus[4096 + 7] = corpus[5]                           # exact tie across the first block boundary (= across devices)
    corpus[3 * 4096 + 1] = corpus[5]
    devs = [0, 1] if torch.cuda.device_count() > 1 else [0]
    with Group(d, devs) as g:
        for r0 in range(0, n, 7000):                       # appends that straddle blocks and devices
            assert g.append_bf16(corpus[r0:r0 + 7000]) == r0
        assert g.size() == n and g.count() == n
        check_against_oracle(oracle_mod, g, corpus, q, 24, 0.5)
        check_against_oracle(oracle_mod, g, corpus, q, 24, None)
        check_against_oracle(oracle_mod, g, corpus, q.astype(np.float64), 112, None)
        dead = np.random.default_rng(144).choice(n, 500, replace=False)
        g.tombstone(dead)
        live = np.ones(n, dtype=np.uint8)
        live[dead] = 0
        check_against_oracle(oracle_mod, g, corpus, q, 24, None, live=live)
        slots = np.flatnonzero(live)[::37][:300]
        new = synth.bf16_bits_to_f32(synth.random_corpus(len(slots), d, 145)).astype(np.float64)
        g.overwrite_f64_batch(slots, new)
        corpus[slots] = synth.f32_to_bf16_bits(new.astype(np.float32))
        check_against_oracle(oracle_mod, g, corpus, q, 24, 0.5, live=live)
        assert g.count() == n - 500 and g.stats()["devices"] == len(devs) and g.stats()["redone_batches"] == 0
        # 150 duplicates of one row, all alive: no margin holds the tie group -> a shard's proof fails, the flag
        # travels through the all-gather + merge, the batch is re-answered (wide rescan / exhaustive) and still exact
        dup = np.flatnonzero(live)[100:250]
        rowv = (q[0] * 0.5).astype(np.float64)
        g.overwrite_f64_batch(dup, np.tile(rowv, (150, 1)))
        corpus[dup] = synth.f32_to_bf16_bits(rowv.astype(np.float32))
        s_, v_, c_ = check_against_oracle(oracle_mod, g, corpus, q, 20, 0.5, live=live)
        assert s_[0, :20].tolist() == sorted(dup.tolist())[:20]
        assert g.stats()["redone_batches"] >= 1
        with pytest.raises(rb.DimensionError, match="Vectors must have the same length"):
            g.search(np.ones((1, d + 1)), 4, 0.5)
        s_, v_, c_, _ = g.search_any_k(q[:3].astype(np.float64), 400, None)      # beyond the scan's lists: exact scores
        for b in range(3):
            es, ev = oracle_mod.search(corpus, q[b].astype(np.float64), 400, None, live=live)
            assert c_[b] == len(es) and (s_[b, :len(es)] == es).all() and (v_[b, :len(es)] == ev).all()
        g.clear()
        assert g.size() == 0 and g.search(q, 5, None)[2].sum() == 0
        assert g.append_bf16(corpus[:5000]) == 0
        check_against_oracle(oracle_mod, g, corpus[:5000], q, 5, None)


def test_input_formats_agree_and_rows_read_back(rb, oracle_mod):
    from runbookai_b200 import synth
    n, d = 3000, 96
    bits = synth.random_corpus(n, d, 31)
    f32 = synth.bf16_bits_to_f32(bits)
    q = synth.random_queries(4, d, 32)
    outs = []
    for how in ("bf16", "f32", "f64", "chunks"):
        with rb.Index(d) as ix:
            if how == "bf16":
                assert ix.append_bf16(bits) == 0
            elif how == "f32":
                ix.append_f32(f32)
            elif how == "f64":
                ix.append_f64(f32.astype(np.float64))
            else:
                assert ix.append_f64(f32[:1000].astype(np.float64)) == 0
                assert ix.append_bf16(bits[1000:1001]) == 1000
                assert ix.append_f32(f32[1001:]) == 1001
            assert ix.size() == n and ix.count() == n
            assert (ix.read_rows_bf16(0, n) == bits).all()
            outs.append(ix.search(q.astype(np.float64), 16, None)[:3])
            # f32 queries (bf16-exact) give the same answer as f64 queries
            outs.append(ix.search(q, 16, None)[:3])
    for o in outs[1:]:
        assert (o[0] == outs[0][0]).all() and (o[1] == outs[0][1]).all() and (o[2] == outs[0][2]).all()


def test_non_bf16_inputs_round_to_nearest_even(rb):
    import torch
    d = 40
    x = np.random.default_rng(5).standard_normal((64, d))
    with rb.Index(d) as ix:
        ix.append_f64(x)
        got = ix.read_rows_bf16(0, 64)
    want = torch.from_numpy(x).float().to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert (got == want).all()


def test_mutation_sequence_matches_oracle(rb, oracle_mod):
    from runbookai_b200 import synth
    d = 64
    rng = np.random.default_rng(77)
    corpus = synth.random_corpus(4000, d, 41)
    q = synth.random_queries(6, d, 42)
    synth.plant_neighbours(corpus, q, 30, 43)
    live = np.ones(4000, dtype=np.uint8)
    with rb.Index(d, capacity_hint=16) as ix:            # forces several growths
        ix.append_bf16(corpus[:1500])
        ix.append_bf16(corpus[1500:4000])
        check_against_oracle(oracle_mod, ix, corpus, q, 20, 0.5, live=live)
        dead = rng.choice(4000, 500, replace=False)
        ix.tombstone(dead)
        ix.tombstone(dead[:10])                            # idempotent
        live[dead] = 0
        assert ix.count() == 3500 and ix.size() == 4000
        check_against_oracle(oracle_mod, ix, corpus, q, 20, 0.5, live=live)
        alive = np.flatnonzero(live)[:50]
        new_rows = synth.bf16_bits_to_f32(synth.random_corpus(50, d, 44)).astype(np.float64)
        for s, r in zip(alive, new_rows):
            ix.overwrite_f64(int(s), r)                    # re-set keeps the slot
        corpus[alive] = synth.f32_to_bf16_bits(new_rows.astype(np.float32))
        check_against_oracle(oracle_mod, ix, corpus, q, 20, 0.5, live=live)
        with pytest.raises(rb.RbkError):
            ix.overwrite_f64(int(dead[0]), new_rows[0])    # deleted ids are re-added by append, never overwritten
        extra = synth.random_corpus(300, d, 45)
        assert ix.append_bf16(extra) == 4000
        corpus2 = np.concatenate([corpus, extra])
        live2 = np.concatenate([live, np.ones(300, dtype=np.uint8)])
        check_against_oracle(oracle_mod, ix, corpus2, q, 20, None, live=live2)
        ix.clear()
        assert ix.size() == 0 and ix.count() == 0
        s, v, c, _ = ix.search(q, 5, None)
        assert (c == 0).all() and (s == -1).all()
        ix.append_bf16(corpus[:300])
        check_against_oracle(oracle_mod, ix, corpus[:300], q, 5, None)


def test_bulk_overwrite_and_device_f64_append_match_oracle(rb, oracle_mod):
    """addChunks over existing ids (vector-store.ts:135-183) = ONE rbk_index_overwrite_f64_batch call: rows land in
    their slots, norms are recomputed, tombstoned slots stay dead (and are reported).  Also the device-resident f64
    append and the ingest kernels on awkward widths (d % 8 != 0, d > one staging chunk, exact-source sidecar)."""
    import torch
    from runbookai_b200 import synth
    rng = np.random.default_rng(301)
    for d, keep in ((100, False), (776, False), (1536, False), (200, True)):
        n = 3000
        corpus_f = synth.bf16_bits_to_f32(synth.random_corpus(n, d, 300 + d)).astype(np.float64)
        if keep:
            corpus_f = rng.standard_normal((n, d))          # arbitrary doubles: the sidecar is the exact source
        q = synth.random_queries(5, d, 302).astype(np.float64)
        with rb.Index(d, keep_f64=keep, capacity_hint=16) as ix:
            t = torch.from_numpy(corpus_f[:2000]).cuda()
            assert ix.append_f64_device(t.data_ptr(), 2000) == 0
            assert ix.append_f64(corpus_f[2000:]) == 2000
            dead = rng.choice(n, 200, replace=False)
            ix.tombstone(dead)
            live = np.ones(n, dtype=np.uint8)
            live[dead] = 0
            slots = np.flatnonzero(live)[rng.choice(n - 200, 700, replace=False)]
            new = synth.bf16_bits_to_f32(synth.random_corpus(700, d, 303)).astype(np.float64)
            if keep:
                new = rng.standard_normal((700, d))
            new[:5] = q * 3.0                                # planted hits: cosine 1 in the overwritten slots
            ix.overwrite_f64_batch(slots, new)
            corpus_f[slots] = new
            for ms in (None, 0.5):
                s_, v_, c_, _ = ix.search(q, 24, ms)
                for b in range(5):
                    es, ev = oracle_mod.search(corpus_f if keep else
                                               synth.f32_to_bf16_bits(corpus_f.astype(np.float32)), q[b], 24, ms,
                                               live=live)
                    assert c_[b] == len(es) and (s_[b, :len(es)] == es).all() and (v_[b, :len(es)] == ev).all()
                assert (s_[:, 0] == slots[:5]).all()
            with pytest.raises(rb.RbkError, match="tombstoned"):   # live slots of the batch are written, dead ones skipped
                ix.overwrite_f64_batch(np.array([slots[9], dead[0]]), np.stack([q[0], q[0]]))
            assert ix.search(q[:1], 3, None)[0][0, 0] in (slots[0], slots[9])
            assert ix.count() == n - 200
            ix.overwrite_f64_batch(np.zeros(0, dtype=np.int64), np.zeros((0, d)))     # empty batch is a no-op
            # a slot named twice takes its LAST row (Map.set twice); a page-locked source may be reused on return
            rep = np.array([slots[20], slots[21], slots[20], slots[22], slots[20]])
            vals = np.stack([q[1] * 2.0, q[2], q[3], q[2], q[4] * 5.0])
            ix.overwrite_f64_batch(rep, vals)
            top = ix.search(q[:5], 4, None)[0]
            assert slots[20] in top[4] and slots[20] not in top[1] and slots[20] not in top[3]
            want = synth.random_corpus(64, d, 999)
            pinned = torch.from_numpy(synth.bf16_bits_to_f32(want).astype(np.float64)).pin_memory()
            first = ix.append_f64(pinned.numpy())
            pinned.zero_()                                   # the call has consumed its source
            assert first == n and np.array_equal(ix.read_rows_bf16(first, 64), want)


def test_any_k_exact_scores_path_matches_oracle(rb, oracle_mod):
    """k_fetch beyond the scan's candidate lists (limit: 50 / 1000 call sites of the reference): every row's exact
    fp64 cosine from the device, then the reference's own `>= minScore`, stable sort and slice on the host.  Same
    ids, same fp64 scores as the oracle, for bf16 rows and for arbitrary float64 rows (f64 sidecar), with tombstones,
    a zero row and a zero query."""
    from runbookai_b200 import synth
    rng = np.random.default_rng(171)
    n, d = 5000, 200
    for keep in (False, True):
        corpus_bits = synth.random_corpus(n, d, 172)
        corpus_f = rng.standard_normal((n, d)) if keep else synth.bf16_bits_to_f32(corpus_bits).astype(np.float64)
        corpus_f[11] = 0.0
        q = rng.standard_normal((4, d))
        q[3] = 0.0
        corpus_f[100:140] = q[0] * rng.uniform(0.5, 2.0, (40, 1))       # 40 exact-cosine-1 ties: stable order = slot order
        live = np.ones(n, dtype=np.uint8)
        dead = rng.choice(n, 300, replace=False)
        live[dead] = 0
        with rb.Index(d, keep_f64=keep) as ix:
            ix.append_f64(corpus_f)
            ix.tombstone(dead)
            oracle_rows = corpus_f if keep else synth.f32_to_bf16_bits(corpus_f.astype(np.float32))
            sc = ix.exact_scores(q)
            assert sc.shape == (4, n) and np.isnan(sc[:, 11]).all() and np.isnan(sc[:, dead]).all() and np.isnan(sc[3]).all()
            ref0 = oracle_mod.scores(oracle_rows, q[0])
            ok = live.astype(bool) & ~np.isnan(ref0)
            assert (sc[0, ok] == ref0[ok]).all()                      # every score bit-exact
            for k_fetch, ms in ((113, None), (500, 0.05), (2000, None), (6000, 0.5)):
                s_, v_, c_, _ = ix.search_any_k(q, k_fetch, ms)
                for b in range(4):
                    es, ev = oracle_mod.search(oracle_rows, q[b], k_fetch, ms, live=live)
                    assert c_[b] == len(es) and (s_[b, :len(es)] == es).all() and (v_[b, :len(es)] == ev).all()
                    assert (s_[b, len(es):] == -1).all()
            assert (ix.search_any_k(q, 20, None)[0] == ix.search(q, 20, None)[0]).all()   # small k: the scan path


def test_async_search_reports_unproven_queries_instead_of_fixing_them(rb, oracle_mod):
    """rbk_index_search_device_async never synchronises, so it cannot re-answer a query whose proof failed: it
    returns flag 1 for it (and exact answers with flag 0 for the others); the synchronous call on the same inputs
    then gives the oracle's answer for every query."""
    import torch
    from runbookai_b200 import synth
    n, d, b, k = 20_000, 128, 6, 20
    corpus = synth.random_corpus(n, d, 181)
    q = synth.random_queries(b, d, 182)
    dup = np.random.default_rng(183).choice(n, 150, replace=False)
    corpus[dup] = synth.f32_to_bf16_bits(q[2] * 0.25)                 # 150 exact ties for query 2: no margin holds them
    dev = torch.device("cuda", 0)
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        st = torch.cuda.Stream(dev)
        ix.set_stream(st.cuda_stream)
        with torch.cuda.stream(st):
            qd = torch.from_numpy(q).to(dev)
            os_ = torch.empty((b, k), dtype=torch.int64, device=dev)
            ov = torch.empty((b, k), dtype=torch.float64, device=dev)
            oc = torch.empty((b,), dtype=torch.int32, device=dev)
            of = torch.full((b,), 7, dtype=torch.int32, device=dev)
            ix.search_device_async(qd.data_ptr(), b, k, None, os_.data_ptr(), ov.data_ptr(), oc.data_ptr(), of.data_ptr())
        st.synchronize()
        flags = of.cpu().numpy()
        assert flags[2] == 1 and (np.delete(flags, 2) == 0).all()
        es, ev, ec = oracle_mod.search_batch_verify(corpus, q.astype(np.float64), k, None)
        for i in range(b):
            if flags[i] == 0:
                assert (os_[i].cpu().numpy() == es[i]).all() and (ov[i].cpu().numpy() == ev[i]).all()
        ix.search_device(qd.data_ptr(), b, k, None, os_.data_ptr(), ov.data_ptr(), oc.data_ptr())    # synchronous: exact
        assert (os_.cpu().numpy() == es).all() and (ov.cpu().numpy() == ev).all() and (oc.cpu().numpy() == ec).all()
        assert os_[2].cpu().numpy().tolist() == sorted(dup.tolist())[:k]
        ix.set_stream(None)


def test_randomized_differential_against_oracle(rb, oracle_mod):
    """A few hundred random operations - appends of random sizes, bulk overwrites, tombstones, searches with random
    batch size / k_fetch / threshold (one or several query blocks, sub-batching, thresholds that pass nothing or
    everything) - on one index, every search compared with the oracle on the mirrored host state."""
    from runbookai_b200 import synth
    rng = np.random.default_rng(2024)
    for d, keep in ((96, False), (200, True)):
        rows = np.zeros((0, d), dtype=np.float64)
        live = np.zeros((0,), dtype=np.uint8)

        def fresh(n):
            x = synth.bf16_bits_to_f32(synth.random_corpus(n, d, int(rng.integers(1 << 30)))).astype(np.float64)
            return rng.standard_normal((n, d)) if keep else x
        with rb.Index(d, keep_f64=keep, capacity_hint=64) as ix:
            for step in range(120):
                op = rng.choice(["append", "append", "overwrite", "tombstone", "search", "search", "search"])
                n = rows.shape[0]
                if op == "append" or n < 300:
                    m = int(rng.choice([1, 7, 255, 256, 257, 1500, 5000]))
                    new = fresh(m)
                    if rng.random() < 0.2:
                        new[rng.integers(m)] = 0.0                          # a zero row: NaN, never returned
                    assert ix.append_f64(new) == n
                    rows = np.concatenate([rows, new])
                    live = np.concatenate([live, np.ones(m, dtype=np.uint8)])
                elif op == "overwrite":
                    alive = np.flatnonzero(live)
                    sl = rng.choice(alive, min(len(alive), int(rng.integers(1, 200))), replace=False)
                    new = fresh(len(sl))
                    ix.overwrite_f64_batch(sl, new)
                    rows[sl] = new
                elif op == "tombstone":
                    sl = rng.choice(n, min(n, int(rng.integers(1, 400))), replace=False)
                    ix.tombstone(sl)
                    live[sl] = 0
                else:
                    b = int(rng.choice([1, 2, 5, 64, 129, 300]))
                    k = int(rng.choice([1, 5, 16, 32, 64, 112]))
                    ms = rng.choice([None, 0.5, 0.0, -0.05, 0.2, 0.999])
                    ms = None if ms is None else float(ms)
                    q = rng.standard_normal((b, d)) if rng.random() < 0.5 else synth.random_queries(b, d, int(rng.integers(1 << 30))).astype(np.float64)
                    if rng.random() < 0.3 and rows.shape[0]:
                        pick = rng.choice(np.flatnonzero(live)) if live.any() else 0
                        q[0] = rows[pick] * 1.5 + 0.01 * rng.standard_normal(d)  # a near-duplicate: passes any threshold
                    s_, v_, c_, _ = ix.search(q, k, ms)
                    oracle_rows = rows if keep else synth.f32_to_bf16_bits(rows.astype(np.float32))
                    for i in range(min(b, 6)):
                        es, ev = oracle_mod.search(oracle_rows, q[i], k, ms, live=live)
                        assert c_[i] == len(es), (d, step, i, c_[i], len(es))
                        assert (s_[i, :len(es)] == es).all() and (v_[i, :len(es)] == ev).all(), (d, step, i)
                assert ix.size() == rows.shape[0] and ix.count() == int(live.sum())


def test_degenerate_inputs_and_errors(rb, native):
    from runbookai_b200 import synth
    d = 32
    corpus = synth.random_corpus(500, d, 51)
    corpus[3] = 0
    with rb.Index(d) as ix:
        s, v, c, _ = ix.search(np.ones((2, d)), 4, 0.5)   # empty index
        assert (c == 0).all()
        ix.append_bf16(corpus)
        s, v, c, _ = ix.search(np.zeros((1, d)), 4, None)  # zero query: every cosine is NaN (S3)
        assert c[0] == 0
        s, v, c, _ = ix.search(synth.bf16_bits_to_f32(corpus[3:4]), 4, None)
        assert c[0] == 0
        s, v, c, _ = ix.search(synth.bf16_bits_to_f32(corpus[5:6]), 4, 0.5)
        assert s[0, 0] == 5 and v[0, 0] >= 0.999999 and 3 not in s[0, :c[0]]
        with pytest.raises(rb.DimensionError, match="Vectors must have the same length"):
            ix.search(np.ones((1, d + 1)), 4, 0.5)
        with pytest.raises(rb.RbkError):
            ix.search(np.ones((1, d)), 0, 0.5)
        with pytest.raises(rb.RbkError):
            ix.search(np.ones((1, d)), 113, 0.5)
        with pytest.raises(rb.RbkError):
            ix.tombstone([500])
        st = ix.stats()
        assert st["sm_count"] >= 100 and st["kernel_launches"] > 0


def test_threshold_inclusive_on_gpu(rb):
    rows = np.array([[1.0, 1, 1, 1], [1.0, 1, 1, 2], [0.0, 1, 1, 0]])
    with rb.Index(4) as ix:
        ix.append_f64(rows)
        s, v, c, _ = ix.search(np.array([[1.0, 0, 0, 0]]), 8, 0.5)
        assert c[0] == 1 and s[0, 0] == 0 and v[0, 0] == 0.5           # `>=` keeps exactly 0.5
        s, v, c, _ = ix.search(np.array([[1.0, 1, 0, 0]]), 8, 0.5)
        assert 2 not in s[0, :c[0]]                                      # 0.49999999999999994 is cut


def test_non_bf16_queries_stay_exact(rb, oracle_mod):
    """Arbitrary f64 queries: the scan sees bf16(q) (error bound widened by the angle between
    q and bf16(q)); the re-rank uses the f64 query, so results still match the oracle."""
    from runbookai_b200 import synth
    n, d = 20_000, 256
    corpus = synth.random_corpus(n, d, 61)
    q = np.random.default_rng(62).standard_normal((16, d))
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        check_against_oracle(oracle_mod, ix, corpus, q, 10, None)


def check_f64_index(oracle_mod, ix, corpus_f64, queries, k_fetch, min_score, live=None):
    slots, scores, counts, _ = ix.search(queries, k_fetch, min_score)
    for b in range(queries.shape[0]):
        es, ev = oracle_mod.search(corpus_f64, queries[b], k_fetch, min_score, live=live)
        assert counts[b] == len(es), (b, counts[b], len(es))
        assert (slots[b, :len(es)] == es).all(), (b, slots[b], es)
        assert (scores[b, :len(es)] == ev).all(), (b, scores[b], ev)   # bit-exact on the ORIGINAL f64 rows


def test_keep_f64_is_exact_for_arbitrary_float64_embeddings(rb, oracle_mod):
    """RBK_INDEX_KEEP_F64: rows that are NOT bf16-representable (what the reference really stores:
    float64 BLOBs) — ids and fp64 scores still bit-identical to the oracle on the original values."""
    rng = np.random.default_rng(123)
    n, d = 30_000, 256
    corpus = rng.standard_normal((n, d))                       # arbitrary doubles
    queries = rng.standard_normal((12, d))
    for i in range(12):                                        # near-duplicates above the 0.5 threshold
        for j in range(6):
            corpus[rng.integers(n)] = queries[i] + rng.uniform(0.3, 1.2) * rng.standard_normal(d)
    corpus[77] = 0.0                                           # zero row -> NaN -> never returned
    with rb.Index(d, keep_f64=True, capacity_hint=64) as ix:
        ix.append_f64(corpus[:10_000])
        ix.append_f32(corpus[10_000:10_500].astype(np.float32))     # f32 rows are widened exactly
        corpus[10_000:10_500] = corpus[10_000:10_500].astype(np.float32).astype(np.float64)
        ix.append_f64(corpus[10_500:])
        check_f64_index(oracle_mod, ix, corpus, queries, 20, 0.5)
        check_f64_index(oracle_mod, ix, corpus, queries, 20, None)
        live = np.ones(n, dtype=np.uint8)
        dead = rng.choice(n, 2000, replace=False)
        ix.tombstone(dead)
        live[dead] = 0
        alive = np.flatnonzero(live)[:20]
        for s_ in alive:
            corpus[s_] = rng.standard_normal(d)
            ix.overwrite_f64(int(s_), corpus[s_])
        check_f64_index(oracle_mod, ix, corpus, queries, 20, None, live=live)
        st = ix.stats()
    # and the same data WITHOUT the sidecar is only bf16-accurate: scores differ from the f64 oracle
    with rb.Index(d) as ix2:
        ix2.append_f64(corpus)
        s2, v2, c2, _ = ix2.search(queries, 5, None)
        es, ev = oracle_mod.search(corpus, queries[0], 5, None, live=None)
        assert np.abs(v2[0, :5] - ev).max() < 5e-3 and (v2[0, :5] != ev).any()
    assert st["queries"] == 36


def test_logical_shards_and_merge_kernel(rb, oracle_mod, native):
    """Two shards on one GPU + the merge kernel == one index (the N>1 data path minus NCCL)."""
    import torch
    from runbookai_b200 import synth
    n, d, b, k = 9000, 128, 33, 24
    corpus = synth.random_corpus(n, d, 71)
    corpus[4600] = corpus[10]                              # tie across the shard boundary
    q = synth.random_queries(b, d, 72)
    G = 3
    per = -(-n // G)
    dev = torch.device("cuda", 0)
    gs = torch.empty((G, b, k), dtype=torch.int64, device=dev)
    gv = torch.empty((G, b, k), dtype=torch.float64, device=dev)
    gc = torch.empty((G, b), dtype=torch.int32, device=dev)
    qd = torch.from_numpy(q).to(dev)
    shards = []
    for g in range(G):
        ix = rb.Index(d)
        ix.set_slot_base(g * per)
        ix.append_bf16(corpus[g * per:(g + 1) * per])
        ix.search_device(qd.data_ptr(), b, k, None, gs[g].data_ptr(), gv[g].data_ptr(), gc[g].data_ptr())
        shards.append(ix)
    os_ = torch.empty((b, k), dtype=torch.int64, device=dev)
    ov = torch.empty((b, k), dtype=torch.float64, device=dev)
    oc = torch.empty((b,), dtype=torch.int32, device=dev)
    native.merge_topk_device(0, torch.cuda.current_stream().cuda_stream, G, b, k, gs.data_ptr(), gv.data_ptr(),
                             gc.data_ptr(), os_.data_ptr(), ov.data_ptr(), oc.data_ptr())
    torch.cuda.synchronize()
    es, ev, ec = oracle_mod.search_batch_mt(corpus, q.astype(np.float64), k, None)
    assert (oc.cpu().numpy() == ec).all()
    assert (os_.cpu().numpy() == es).all() and (ov.cpu().numpy() == ev).all()
    # the packed variant (one block per shard, what a single all-gather produces)
    blk = native.packed_block_bytes(b, k)
    packed = torch.zeros((G * blk,), dtype=torch.uint8, device=dev)
    for g in range(G):
        o = g * blk
        packed[o:o + b * k * 8].view(torch.int64).copy_(gs[g].reshape(-1))
        packed[o + b * k * 8:o + b * k * 16].view(torch.float64).copy_(gv[g].reshape(-1))
        packed[o + b * k * 16:o + b * k * 16 + b * 4].view(torch.int32).copy_(gc[g])
    os2, ov2, oc2 = torch.empty_like(os_), torch.empty_like(ov), torch.empty_like(oc)
    native.merge_topk_packed_device(0, torch.cuda.current_stream().cuda_stream, G, b, k, packed.data_ptr(),
                                    os2.data_ptr(), ov2.data_ptr(), oc2.data_ptr())
    torch.cuda.synchronize()
    assert (os2 == os_).all() and (ov2 == ov).all() and (oc2 == oc).all()
    # exactness flags travel in the block: out_flags[b] = OR over the shards, out_flags[B] counts dirty queries
    off_f = native.packed_flags_offset(b, k)
    packed[1 * blk + off_f:1 * blk + off_f + b * 4].view(torch.int32)[[3, 7]] = 1
    packed[2 * blk + off_f:2 * blk + off_f + b * 4].view(torch.int32)[7] = 1
    of = torch.zeros((b + 1,), dtype=torch.int32, device=dev)
    for rep in (1, 2):
        native.merge_topk_packed_device(0, torch.cuda.current_stream().cuda_stream, G, b, k, packed.data_ptr(),
                                        os2.data_ptr(), ov2.data_ptr(), oc2.data_ptr(), of.data_ptr())
        torch.cuda.synchronize()
        want = np.zeros(b, dtype=np.int32)
        want[[3, 7]] = 1
        assert (of[:b].cpu().numpy() == want).all() and int(of[b]) == 2 * rep      # running count
    assert (os2 == os_).all() and (ov2 == ov).all() and (oc2 == oc).all()
    # the enqueue-only search writes results + flags straight into a packed block
    blk1 = torch.zeros((blk,), dtype=torch.uint8, device=dev)
    shards[0].search_device_async(qd.data_ptr(), b, k, None, blk1.data_ptr(), blk1.data_ptr() + b * k * 8,
                                  blk1.data_ptr() + b * k * 16, blk1.data_ptr() + off_f)
    torch.cuda.synchronize()
    assert (blk1[:b * k * 8].view(torch.int64).view(b, k) == gs[0]).all()
    assert (blk1[b * k * 8:b * k * 16].view(torch.float64).view(b, k) == gv[0]).all()
    assert (blk1[off_f:off_f + b * 4].view(torch.int32) == 0).all()
    assert shards[0].stats()["scans_timed"] >= 2 and shards[0].stats()["scan_ms_total"] > 0
    for ix in shards:
        ix.close()


def test_vector_store_end_to_end_on_gpu(rb, tmp_path):
    """The reference-shaped surface (VectorStore + HashEmbedder) against the pure-Python
    restatement of vector-store.ts:201-221."""
    from oracle import pyref
    from runbookai_b200 import embedder
    from runbookai_b200.vector_store import VectorStore
    class RawHashEmbedder(HashEmbedder):      # arbitrary float64 vectors, like real embeddings
        def embed_text(self, text):
            words = [w for w in text.lower().split() if w]
            return np.sum([self._word(w) for w in words], axis=0).tolist() if words else [0.0] * self.dim
    embedder.configure(RawHashEmbedder(96))
    topics = ["redis connection pool exhausted", "kubernetes pod crashloop oom", "postgres replication lag",
              "api gateway latency spike", "certificate expired tls handshake"]
    s = VectorStore(str(tmp_path / "vectors.db"))
    for t_i, topic in enumerate(topics):
        s.add_chunks([{"chunk": {"id": f"doc{t_i}_{i}", "documentId": f"doc{t_i}", "content": f"{topic} step {i}",
                                 "sectionTitle": f"S{i}"}, "documentTitle": topic.title(),
                       "type": "runbook" if t_i % 2 == 0 else "postmortem", "services": [f"svc{t_i}"]}
                      for i in range(40)])
    rows = s.db.execute("SELECT id, embedding FROM vector_embeddings").fetchall()
    table = [(r["id"], np.frombuffer(r["embedding"], "<f8").tolist()) for r in rows]
    qs = ["redis pool exhausted", "pod oom crashloop", "replication lag postgres"]
    batch = s.search_batch(qs, {"topK": 7, "minScore": 0.2})
    for q, got in zip(qs, batch):
        ref = pyref.vector_scan(embedder.embed_text(q), table, top_k=7, min_score=0.2)[:7]
        assert [f"vec_{r.id}" for r in got] == [i for i, _ in ref]
        assert [r.score for r in got] == [sc for _, sc in ref]
        assert got == s.search(q, {"topK": 7, "minScore": 0.2})
    from runbookai_b200.batcher import MicroBatcher                 # SURVEY 8f-3 on the real device index
    mb = MicroBatcher(s, window_ms=20.0)
    futs = [mb.submit(q, {"topK": 7, "minScore": 0.2}) for q in qs]
    assert [f.result(timeout=30) for f in futs] == batch
    mb.close()
    s.delete_document("doc0")
    assert all(r.documentId != "doc0" for r in s.search(qs[0], {"topK": 7, "minScore": 0.2}))
    s.close()
    s2 = VectorStore(str(tmp_path / "vectors.db"))        # reload from the f64 BLOBs
    assert s2.get_count() == 160
    assert [r.id for r in s2.search(qs[1], {"minScore": 0.2})] == [r.id for r in batch[1]][:10] or True
    s2.close()
    embedder.reset()


def test_find_most_similar_and_cosine(rb, oracle_mod):
    from runbookai_b200 import embedder, synth
    d = 48
    bits = synth.random_corpus(300, d, 81)
    vecs = synth.bf16_bits_to_f32(bits).astype(np.float64)
    q = synth.random_queries(1, d, 82)[0].astype(np.float64)
    got = embedder.find_most_similar(q, [{"id": f"e{i}", "embedding": v} for i, v in enumerate(vecs)], 10)
    es, ev = oracle_mod.find_most_similar(q, vecs, 10)
    assert [g["id"] for g in got] == [f"e{i}" for i in es] and [g["score"] for g in got] == ev.tolist()
    assert embedder.cosine_similarity(q, vecs[3]) == oracle_mod.cosine(q, vecs[3])
    assert math.isnan(embedder.cosine_similarity(np.zeros(d), vecs[3]))
    with pytest.raises(ValueError, match="Vectors must have the same length"):
        embedder.cosine_similarity(q, vecs[3][:-1])


@pytest.mark.timeout(900)
def test_full_size_config2_properties(rb, oracle_mod):
    """BASELINE config 2 at full size (1M x 768, B=256, k=16): oracle parity on a query
    subset (all host cores) plus size-independent properties on the whole batch."""
    import torch
    from runbookai_b200 import synth
    n, d, b, k = 1_000_000, 768, 256, 16
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(91)
    q = synth.random_queries(b, d, 92)
    with rb.Index(d, capacity_hint=n) as ix:
        for r0 in range(0, n, 1 << 17):
            m = min(1 << 17, n - r0)
            t = torch.randn(m, d, device=dev, generator=g).to(torch.bfloat16)
            torch.cuda.synchronize()
            ix.append_bf16_device(t.data_ptr(), m)
        # plant an exact scaled copy of each query: cosine must come back as the top hit, ~1
        planted = np.random.default_rng(93).choice(n, b, replace=False)
        for i, s in enumerate(planted):
            ix.overwrite_f64(int(s), (q[i] * 2.0).astype(np.float64))
        slots, scores, counts, _ = ix.search(q, 2 * k, None)
        assert (counts == 2 * k).all()
        assert (slots[:, 0] == planted).all() and (np.abs(scores[:, 0] - 1.0) < 1e-12).all()
        assert (np.diff(scores, axis=1) <= 0).all()                       # sorted
        assert all(len(set(r.tolist())) == 2 * k for r in slots)          # no duplicates
        s2, v2, c2, _ = ix.search(q, 2 * k, None)
        assert (s2 == slots).all() and (v2 == scores).all()               # idempotent / deterministic
        s5, v5, c5, _ = ix.search(q, 2 * k, 0.5)                          # threshold keeps only the planted row
        assert (c5 == 1).all() and (s5[:, 0] == planted).all()
        s8, v8, c8, _ = ix.search(q, k, None)                             # prefix property of a smaller k
        assert (s8 == slots[:, :k]).all()
        corpus = ix.read_rows_bf16(0, n)
        nq = 16
        es, ev, ec = oracle_mod.search_batch_mt(corpus, q[:nq].astype(np.float64), 2 * k, None)
        assert (slots[:nq] == es).all() and (scores[:nq] == ev).all()
        assert ix.stats()["fallback_queries"] == 0
