#!/usr/bin/env python
"""Stored rows as queries on one GPU: rbk_index_search_slots_f64 against rbk_index_search_each_f64 on the host copies
of the same rows (what a caller pays today, with the embedding already in hand), and one all-neighbours pass.

    python scripts/search_slots_bench.py [--rows 1000000] [--dim 1536] [--placement device|host] [--steps 5]
                                         [--warmup 2] [--pass-k 10] [--pass-rows N]

Float64 rows in clusters of 64, made on the device from a seed; the query slots are spread over the corpus and their
rows read back once.  For B = 1, 32 and 1024 and k_fetch 20 and 1000 the two calls alternate step by step after the warm-up, and
every answer of search_slots is compared with search_each's.  Then one search_slots over the first --pass-rows slots
(default: every row) at k_fetch --pass-k: wall time, queries per second, and the pass's scan work (2 B N d
operations) over that time against the 989 TFLOP/s dense BF16 figure of NVIDIA's H100 SXM data sheet.  Prints one
JSON line with the card name and power limit, read in the same run.  Writes nothing to the tree.
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

BATCHES = [1, 32, 1024]
K_FETCH = [20, 1000]
PEAK_TFLOPS = 989.0
CLUSTER = 64


def fill(ix, rows, dim, seed, keep):
    """rows float64 rows made on the device in chunks and appended from there: clusters of CLUSTER consecutive rows,
    each a normal centre plus 0.7 times normal noise, so that a row's nearest rows are its cluster's, well apart from
    the rest, as chunks of one document are.  (Rows that are all independent normal vectors score around 0 with
    one another, too close together for any first pass to prove a top 10.)  Returns the host copies of the rows
    `keep` (sorted slots)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn((rows + CLUSTER - 1) // CLUSTER, dim, dtype=torch.float64, device="cuda", generator=g)
    chunk = max(CLUSTER, (1 << 28) // (dim * 8) // CLUSTER * CLUSTER)
    out = []
    for r0 in range(0, rows, chunk):
        n = min(chunk, rows - r0)
        x = centres[(torch.arange(r0, r0 + n, device="cuda") // CLUSTER)]
        x += 0.7 * torch.randn(n, dim, dtype=torch.float64, device="cuda", generator=g)
        mine = keep[(keep >= r0) & (keep < r0 + n)] - r0
        if len(mine):
            out.append(x[torch.as_tensor(mine, device="cuda")].cpu().numpy())
        torch.cuda.synchronize()
        ix.append_f64_device(x.data_ptr(), n)
        del x
    return np.concatenate(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--placement", choices=["device", "host"], default="device")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pass-k", type=int, default=10)
    ap.add_argument("--pass-rows", type=int, default=0, help="queries of the all-neighbours pass (0: every row)")
    a = ap.parse_args()
    import torch
    from runbookai_b200 import Index
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    slots = np.unique(np.linspace(0, a.rows - 1, max(BATCHES)).astype(np.int64))
    res = {"card": card, "rows": a.rows, "dim": a.dim, "placement": a.placement, "cases": []}
    with Index(a.dim, device=0, capacity_hint=a.rows, keep_f64=True, f64_on_host=a.placement == "host") as ix:
        q_all = fill(ix, a.rows, a.dim, 11, slots)
        torch.cuda.empty_cache()
        for B in BATCHES:
            sl, q = slots[:B], q_all[:B]
            for k in K_FETCH:
                t_slots, t_each, equal = [], [], True
                for step in range(a.warmup + a.steps):
                    s = ix.search_slots(sl, k, None)
                    e = ix.search_each(q, [k] * B, [None] * B)
                    equal &= (s[2] == e[2]).all() and (s[0] == e[0]).all() and s[1].tobytes() == e[1].tobytes()
                    if step >= a.warmup:
                        t_slots.append(s[3])
                        t_each.append(e[3])
                res["cases"].append({"B": B, "k_fetch": k, "search_slots_ms_median": round(float(np.median(t_slots)), 3),
                                     "search_each_ms_median": round(float(np.median(t_each)), 3),
                                     "search_slots_ms": [round(t, 3) for t in t_slots],
                                     "search_each_ms": [round(t, 3) for t in t_each], "answers_equal": bool(equal)})
        nq = a.pass_rows or a.rows
        torch.cuda.synchronize()
        st0 = ix.stats()
        t0 = time.perf_counter()
        s, v, c, ms = ix.search_slots(np.arange(nq, dtype=np.int64), a.pass_k, None)
        wall = time.perf_counter() - t0
        st1 = ix.stats()
        self_first = float(np.mean(s[:, 0] == np.arange(nq)))
        flop = 2.0 * nq * a.rows * a.dim
        res["all_neighbours"] = {"queries": nq, "k_fetch": a.pass_k, "wall_s": round(wall, 3),
                                 "device_s": round(ms / 1e3, 3), "queries_per_s": round(nq / wall, 1),
                                 "scan_tflops": round(flop / wall / 1e12, 1),
                                 "share_of_989_tflops": round(flop / wall / 1e12 / PEAK_TFLOPS, 3),
                                 "own_row_first": self_first,
                                 "retry_batches": st1["retry_batches"] - st0["retry_batches"],
                                 "fallback_queries": st1["fallback_queries"] - st0["fallback_queries"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
