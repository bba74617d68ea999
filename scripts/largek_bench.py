#!/usr/bin/env python
"""Large-k search on one GPU: rbk_index_search_large_f64 (k_fetch up to 4096) or, for --k above 2048,
rbk_index_search_unbounded_f64, through the host-facing call against the route both replace (exact_scores of every row,
then the threshold / stable sort / cut on the host).

    python scripts/largek_bench.py [--rows 1000000] [--dim 1536] [--batch 32] [--k 500] [--steps 10] [--warmup 3]

The default shape is the reference's default embedding width with k = 500 (k_fetch 1000).  The two routes alternate
step by step on the same card, so both numbers come from the same clocks.  Prints one JSON line with the card name and
power limit, device and end-to-end queries/s of both routes, a roofline over this path's algorithmic bytes, and a
`parity` object against the CPU oracle (ids and fp64 scores).  Writes nothing to the tree.  Corpus generation and the
oracle check are bench.py's.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402  (corpus generator, oracle parity, data-sheet peaks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--k", type=int, default=500, help="topK; the search fetches 2*k")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--old-steps", type=int, default=3,
                    help="steps of the old route (seconds each: a host sort of every row of every query)")
    ap.add_argument("--parity-budget", type=float, default=120.0,
                    help="seconds the CPU oracle may take (fewer queries beyond); 0 skips it - every old-route step "
                         "still checks the two routes agree bit for bit")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("largek_bench.py needs a CUDA device: this engine has no CPU path")
    import runbookai_b200._native as nat
    n, d, B, k_fetch = args.rows, args.dim, args.batch, 2 * args.k
    if not nat.RBK_MAX_K_FETCH < k_fetch:
        raise SystemExit(f"2*k must be above {nat.RBK_MAX_K_FETCH}")
    unbounded = k_fetch > nat.RBK_MAX_K_FETCH_LARGE
    synth, pk = bench.load_synth(), bench.peaks()
    ctx = bench.Ctx()
    ctx.world, ctx.rank, ctx.n_total, ctx.device = 1, 0, n, torch.device("cuda", 0)
    ix = nat.Index(d, 0, n)
    bench.gen_shard(ix, 0, n, d, ctx.device)
    q = synth.random_queries(B, d, bench.SEED + 1).astype(np.float64)

    class _Scores:   # hands precomputed exact scores to the mirror's host-side cut (k_fetch above the large limit)
        def __init__(self, sc):
            self.sc = sc

        def exact_scores(self, _q):
            return self.sc

    def old_route():
        res = nat._search_any_k(_Scores(ix.exact_scores(q)), q, max(k_fetch, nat.RBK_MAX_K_FETCH_LARGE + 1), None)
        return res[0][:, :k_fetch], res[1][:, :k_fetch], np.minimum(res[2], k_fetch)

    new_route = ix.search_unbounded if unbounded else ix.search_large
    for _ in range(args.warmup):
        got = new_route(q, k_fetch, None)
    old_route()
    launches0 = ix.stats()["scan_launches"]
    got = new_route(q, k_fetch, None)
    scans_per_call = ix.stats()["scan_launches"] - launches0      # 1 count + 1 emit per query group (and per 1024 queries)
    new_wall, new_dev, old_wall = [], [], []
    for i in range(args.steps):
        t0 = time.perf_counter()
        got = new_route(q, k_fetch, None)
        new_wall.append(time.perf_counter() - t0)
        new_dev.append(got[3])
        if i < args.old_steps:
            t0 = time.perf_counter()
            old = old_route()
            old_wall.append(time.perf_counter() - t0)
            if not ((old[0] == got[0]).all() and old[1].tobytes() == got[1].tobytes() and (old[2] == got[2]).all()):
                raise SystemExit("the two routes disagree")
    st = ix.stats()
    slots, scores, counts = got[0], got[1], got[2]
    parity = (bench.oracle_parity(ctx, ix, 0, n, q, k_fetch, None, (slots, scores, counts), budget_s=args.parity_budget)
              if args.parity_budget > 0 else {"skipped": "--parity-budget 0",
                                               "old_route_bit_equal_steps": len(old_wall)})
    dev_ms = float(np.median(new_dev))
    e2e_s = float(np.median(new_wall))
    old_s = float(np.median(old_wall))
    scan_bytes = scans_per_call * 2.0 * n * d    # count + emit scans of the bf16 corpus
    gather_bytes = float(counts.sum()) * d * 2    # re-rank row reads, counted at the returned rows: a lower bound
    flops = scans_per_call * 2.0 * n * d * B
    t_mem, t_tc = (scan_bytes + gather_bytes) / (pk["hbm"] * 1e9), flops / (pk["tf"] * 1e12)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "metric": "knn_queries_per_sec", "value": B / (dev_ms * 1e-3), "unit": "queries/s", "card": card,
        "config": {"n_docs": n, "dim": d, "batch": B, "k": args.k, "k_fetch": k_fetch, "dtype": "bf16",
                   "data": "synthetic", "steps": args.steps, "warmup": args.warmup,
                   "route": "search_unbounded" if unbounded else "search_large"},
        "device_ms_per_call": dev_ms,
        "e2e": {"value": B / e2e_s, "unit": "queries/s", "seconds_per_call": e2e_s},
        "old_route": {"value": B / old_s, "unit": "queries/s", "seconds_per_call": old_s, "steps": len(old_wall),
                      "what": "exact_scores (fp64 cosine of every row) + host threshold / stable sort / cut"},
        "speedup_e2e": old_s / e2e_s,
        "launches": {"scan_launches": st["scan_launches"], "kernel_launches": st["kernel_launches"],
                     "scans_per_call": scans_per_call},
        "roofline": {"bytes": scan_bytes + gather_bytes, "flops": flops, "t_min_ms": max(t_mem, t_tc) * 1e3,
                     "bound": "memory" if t_mem >= t_tc else "compute",
                     "frac_of_bound": max(t_mem, t_tc) * 1e3 / dev_ms, "peaks": pk,
                     "note": "device time of the whole call (H2D, two scans, select, re-rank, D2H)"},
        "parity": parity}), flush=True)
    ix.close()


if __name__ == "__main__":
    main()
