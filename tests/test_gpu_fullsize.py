"""GPU suite (-m gpu), part 2: oracle parity AT THE SIZES THE HEADLINE IS QUOTED ON, the adversarial
case for the scan's error bound, and the real NCCL path.

SURVEY.md §8(d): for N > 1M the check is a fixed 64-query subsample of the batch against the all-cores
oracle.  The corpus never exists on the host as a whole: it is generated on the device, read back from
the index chunk by chunk and handed to `oracle.search_chunked` (identical per-pair arithmetic to the
literal loop, see rbk_oracle.c "verify" variant and tests/test_oracle.py).  Nothing here reads
the reference checkout."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def rb(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    import runbookai_b200
    return runbookai_b200


def fill_random(ix, n, d, seed, dev):
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    for r0 in range(0, n, 1 << 17):
        m = min(1 << 17, n - r0)
        t = torch.randn(m, d, device=dev, generator=g).to(torch.bfloat16)
        torch.cuda.synchronize()
        ix.append_bf16_device(t.data_ptr(), m)


def check_subsample(oracle_mod, ix, n, q, k_fetch, min_score, got, nq=64):
    slots, scores, counts = got
    es, ev, ec = oracle_mod.search_chunked(ix.read_rows_bf16, n, q[:nq].astype(np.float64), k_fetch, min_score,
                                           chunk_rows=1 << 19)
    assert (counts[:nq] == ec).all()
    for b in range(nq):
        assert (slots[b, :ec[b]] == es[b, :ec[b]]).all(), (b, slots[b], es[b])
        assert (scores[b, :ec[b]] == ev[b, :ec[b]]).all(), (b, scores[b], ev[b])     # bit-exact fp64


@pytest.mark.timeout(1500)
def test_full_size_config3_oracle_subsample(rb, oracle_mod):
    """BASELINE config 3 at FULL size - 10M x 768 bf16, B=1024, k=16 (k_fetch 32), the configuration the headline
    and the roofline are quoted on: ids and fp64 scores of a 64-query subsample identical to the oracle, plus
    size-independent properties of the whole batch."""
    import torch
    from runbookai_b200 import synth
    n, d, b, k = 10_000_000, 768, 1024, 16
    dev = torch.device("cuda", 0)
    q = synth.random_queries(b, d, 301)
    with rb.Index(d, capacity_hint=n) as ix:
        fill_random(ix, n, d, 302, dev)
        slots, scores, counts, _ = ix.search(q, 2 * k, None)
        assert (counts == 2 * k).all()
        assert (np.diff(scores, axis=1) <= 0).all()                       # sorted
        assert all(len(set(r.tolist())) == 2 * k for r in slots)          # no duplicates
        assert slots.min() >= 0 and slots.max() < n
        st = ix.stats()
        assert st["fallback_queries"] == 0 and st["retry_batches"] == 0   # random data: every proof goes through
        check_subsample(oracle_mod, ix, n, q, 2 * k, None, (slots, scores, counts))
        s2, v2, c2, _ = ix.search(q, 2 * k, None)                         # deterministic
        assert (s2 == slots).all() and (v2 == scores).all()


@pytest.mark.timeout(900)
def test_config5_shape_oracle_subsample(rb, oracle_mod):
    """BASELINE config 5: the hypothesis-branch batch, 32 investigations x 8 queries against 5M x 768, k=8.  The
    8 queries of one investigation are near-duplicates of each other (same incident, re-phrased), as in real
    traffic: same neighbours, different scores."""
    import torch
    from runbookai_b200 import synth
    n, d, k = 5_000_000, 768, 8
    dev = torch.device("cuda", 0)
    base = synth.random_queries(32, d, 311)
    rng = np.random.default_rng(312)
    q = synth.bf16_round((base[:, None, :] + 0.3 * rng.standard_normal((32, 8, d))).reshape(256, d)
                         .astype(np.float32))
    with rb.Index(d, capacity_hint=n) as ix:
        fill_random(ix, n, d, 313, dev)
        planted = rng.choice(n, 32, replace=False)
        for i, s in enumerate(planted):                                   # one true neighbour per investigation
            ix.overwrite_f64(int(s), (base[i] * 1.5).astype(np.float64))
        got = ix.search(q, 2 * k, None)[:3]
        assert (got[0][:, 0] == np.repeat(planted, 8)).all()
        check_subsample(oracle_mod, ix, n, q, 2 * k, None, got)
        got5 = ix.search(q, 2 * k, 0.5)[:3]                               # the reference's default threshold
        assert (got5[2] == 1).all()
        check_subsample(oracle_mod, ix, n, q, 2 * k, 0.5, got5)
        assert ix.stats()["fallback_queries"] == 0


@pytest.mark.parametrize("d", [1536, 2048])
def test_all_positive_corpus_error_bound_and_exact_ids(rb, oracle_mod, d):
    """The adversarial case for fp32 tensor-core accumulation: an all-positive corpus and all-positive queries
    (every product has the same sign, cosines ~0.64-1, nothing cancels), at the widest dims.  (i) the scan's
    approximate scores stay inside accumulation_eps(d) = (d+8)*2^-22, the bound the exactness proof rests on;
    (ii) ids and fp64 scores are still bit-identical to the oracle - with scores this crowded most proofs fail and
    the wide rescan / exhaustive kernel must take over, which is the point."""
    from runbookai_b200 import synth
    n, b = 6000, 12
    rng = np.random.Generator(np.random.Philox(900 + d))
    corpus = synth.f32_to_bf16_bits(np.abs(rng.standard_normal((n, d), dtype=np.float32)) + 0.05)
    corpus[:500] = synth.f32_to_bf16_bits(np.full((500, d), 1.0, np.float32) +
                                          rng.uniform(0, 2 ** -6, (500, d)).astype(np.float32))  # near-constant rows
    corpus[500:1000] = synth.f32_to_bf16_bits(rng.uniform(1.0, 1.99, (500, d)).astype(np.float32))  # full mantissas
    q = synth.bf16_round(np.abs(rng.standard_normal((b, d), dtype=np.float32)) + 0.05)
    q[0] = 1.0
    q[1] = synth.bf16_round(rng.uniform(1.0, 1.99, d).astype(np.float32))
    cf = synth.bf16_bits_to_f32(corpus).astype(np.float64)
    qf = q.astype(np.float64)
    ref = (qf @ cf.T) / (np.linalg.norm(qf, axis=1)[:, None] * np.linalg.norm(cf, axis=1)[None, :])
    eps = (d + 8) * 2.0 ** -22                                           # rbk::accumulation_eps
    with rb.Index(d) as ix:
        ix.append_bf16(corpus)
        got = ix.debug_scores(q)
        err = np.abs(got - ref).max()
        assert err <= eps, (err, eps)
        assert err <= eps / 4, f"error {err:.3e} is using more than a quarter of the bound {eps:.3e}"
        for k_fetch, ms in ((10, None), (32, 0.5), (112, None)):
            slots, scores, counts, _ = ix.search(q, k_fetch, ms)
            es, ev, ec = oracle_mod.search_batch_verify(corpus, qf, k_fetch, ms)
            assert (counts == ec).all()
            assert (slots == es).all() and np.array_equal(scores, ev, equal_nan=True)


@pytest.mark.timeout(900)
def test_two_rank_nccl_sharded_parity(rb):
    """The REAL multi-GPU path: two torchrun ranks, NCCL all-gather of the packed blocks (results + exactness flags)
    + merge kernel, one host synchronisation per step; ids and fp64 scores against the oracle, with ties planted
    across the shard boundary and a duplicated-row group that forces the dirty-flag / re-answer path
    (scripts/dist_check.py).  Needs two GPUs."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    env = dict(os.environ, PYTHONPATH=str(ROOT))
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29533", str(ROOT / "scripts" / "dist_check.py")],
                         capture_output=True, text=True, env=env, timeout=800)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert '"parity": true' in res.stdout and '"parity": false' not in res.stdout
