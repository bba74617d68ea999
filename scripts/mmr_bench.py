#!/usr/bin/env python
"""Diverse hits by maximal marginal relevance on one GPU: rbk_index_search_mmr_f64 against rbk_index_search_each_f64 at
the same fetch_k (the candidate search MMR runs first), and how many planted duplicates each puts in a top 10.

    python scripts/mmr_bench.py [--rows 1000000] [--dim 1536] [--placement device|host] [--steps 5] [--warmup 2]

The float64 rows of scripts/search_slots_bench.py (clusters of 64, made on the device from a seed), with planted
duplicates: in every planted cluster the first row is copied exactly over the next four.  Each query is a planted
cluster's first row plus a little noise, so its plain top 10 holds all five copies.  For B = 1, 32 and 1024, k = 10,
fetch_k 50 and 1000 and lambda 0.5 the two calls alternate step by step after the warm-up: median device ms of each.
Duplicate share: the hits in a top 10 that copy a row already above them, over all hits, for search_each's first 10
and for the MMR picks.  Oracle parity: for sampled queries the greedy selection of tests/mmr_oracle.py over the
search_each candidates and their rows, regenerated from the seed, against the library's picks bit for bit.  Prints
one JSON line with the card name and power limit, read in the same run.  Writes nothing to the tree.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
sys.path.insert(0, str(ROOT / "tests"))

from search_slots_bench import CLUSTER, fill   # noqa: E402

BATCHES = [1, 32, 1024]
FETCH_K = [50, 1000]
K, LAM, COPIES = 10, 0.5, 4
SEED = 11


class _Sink:
    """fill()'s target when only the host copies of some rows are wanted: the rows are made again from the seed."""

    def append_f64_device(self, ptr, n):
        pass


def dup_share(slots, counts, first_of):
    """Hits that copy a row already above them in their list, over all hits."""
    dup = hits = 0
    for b in range(len(counts)):
        seen = set()
        for s in slots[b, :counts[b]]:
            src = first_of.get(int(s), int(s))
            dup += src in seen
            seen.add(src)
            hits += 1
    return dup / max(hits, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--placement", choices=["device", "host"], default="device")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parity-queries", type=int, default=4)
    a = ap.parse_args()
    import torch
    import mmr_oracle
    from runbookai_b200 import Index
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    n_clusters = a.rows // CLUSTER
    planted = np.linspace(0, n_clusters - 1, max(BATCHES)).astype(np.int64) * CLUSTER   # each cluster's first row
    first_of = {int(p) + i: int(p) for p in planted for i in range(1, COPIES + 1)}
    rng = np.random.default_rng(5)
    res = {"card": card, "rows": a.rows, "dim": a.dim, "placement": a.placement, "k": K, "lambda": LAM,
           "planted_clusters": len(planted), "copies": COPIES, "cases": []}
    with Index(a.dim, device=0, capacity_hint=a.rows, keep_f64=True, f64_on_host=a.placement == "host") as ix:
        src = fill(ix, a.rows, a.dim, SEED, planted)
        for i in range(1, COPIES + 1):
            ix.overwrite_f64_batch(planted + i, src)
        torch.cuda.empty_cache()
        q_all = src + 0.05 * rng.standard_normal(src.shape)
        last = {}
        for B in BATCHES:
            q = q_all[:B]
            for f in FETCH_K:
                t_mmr, t_each = [], []
                for step in range(a.warmup + a.steps):
                    m = ix.search_mmr(q, K, f, LAM, None)
                    e = ix.search_each(q, [f] * B, [None] * B)
                    if step >= a.warmup:
                        t_mmr.append(m[3])
                        t_each.append(e[3])
                last[(B, f)] = (m, e)
                res["cases"].append({
                    "B": B, "fetch_k": f, "search_mmr_ms_median": round(float(np.median(t_mmr)), 3),
                    "search_each_ms_median": round(float(np.median(t_each)), 3),
                    "search_mmr_ms": [round(t, 3) for t in t_mmr], "search_each_ms": [round(t, 3) for t in t_each],
                    "dup_share_top10_plain": round(dup_share(e[0][:, :K], np.minimum(e[2], K), first_of), 4),
                    "dup_share_top10_mmr": round(dup_share(m[0], m[2], first_of), 4)})
        # oracle parity on sampled queries of the largest batch
        pick = np.linspace(0, max(BATCHES) - 1, a.parity_queries).astype(np.int64)
        parity = []
        for f in FETCH_K:
            m, e = last[(max(BATCHES), f)]
            cand = np.unique(np.concatenate([e[0][b, :e[2][b]] for b in pick]))
            rows = fill(_Sink(), a.rows, a.dim, SEED, np.unique(np.concatenate([cand, planted])))
            keep = np.unique(np.concatenate([cand, planted]))
            row_of = {int(s): rows[i] for i, s in enumerate(keep)}
            for s, p in first_of.items():
                if s in row_of:
                    row_of[s] = row_of[p]
            for b in pick:
                c = int(e[2][b])
                sl = e[0][b, :c]
                picks = mmr_oracle.select(np.stack([row_of[int(s)] for s in sl]), e[1][b, :c], K, LAM)
                ok = (m[2][b] == len(picks) and (m[0][b, :len(picks)] == sl[picks]).all()
                      and m[1][b, :len(picks)].tobytes() == e[1][b, :c][picks].tobytes())
                parity.append(bool(ok))
        res["oracle_parity"] = {"queries": len(parity), "equal": sum(parity)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
