#!/usr/bin/env python
"""Every pair of stored rows at or above a threshold on one GPU: the paged rbk_index_similar_pairs_f64 pass against the
search_slots all-neighbours pass at k = 10 over the same rows.

    python scripts/similar_pairs_bench.py [--rows 1000000] [--dim 1536] [--placements device,host]
                                          [--thresholds 0.99,0.9] [--page 33554432] [--sample 64]

Float64 rows in clusters of 64 made on the device from a seed (search_slots_bench.fill), with planted near-duplicate
pairs: every 97th row's successor is a copy with 1e-4 relative noise.  For each placement of the exact rows and each
threshold, one full paged pass: wall time, pages, pairs found, the device time of the call summed over the pages and
its scan part (the stats' last_scan_ms), the device memory the index holds after each page (its scratch grows only),
and a sample of --sample first slots checked against search_slots([a], count(), t) (slots and score bits).  Then the
all-neighbours pass at k = 10.  Last, the pairs of --oracle-rows sampled first slots (half of them planted) against
the oracle: the rows are made again from the same seed in chunks, read back, and every pair's cosine is the oracle's
(oracle.scores), cut at each threshold and sorted by (score desc, slot asc).  Prints one JSON line with the card name
and power limit, read in the same run.  Writes nothing to the tree.
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
sys.path.insert(0, str(ROOT / "scripts"))


CLUSTER = 64


def corpus_chunks(rows, dim, seed):
    """search_slots_bench.fill's rows, chunk by chunk on the device: (first row, float64 tensor)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn((rows + CLUSTER - 1) // CLUSTER, dim, dtype=torch.float64, device="cuda", generator=g)
    chunk = max(CLUSTER, (1 << 28) // (dim * 8) // CLUSTER * CLUSTER)
    for r0 in range(0, rows, chunk):
        n = min(chunk, rows - r0)
        x = centres[(torch.arange(r0, r0 + n, device="cuda") // CLUSTER)]
        x += 0.7 * torch.randn(n, dim, dtype=torch.float64, device="cuda", generator=g)
        yield r0, x


def oracle_pairs(rows, dim, seed, planted_slots, planted, queries, thresholds):
    """{(q, t): (b [n], scores [n])}: every pair (q, b > q) with the oracle's cosine >= t, in the engine's order."""
    import oracle
    dst = {p: i for i, p in enumerate(planted_slots.tolist())}

    def host_chunks():
        for r0, x in corpus_chunks(rows, dim, seed):
            h = x.cpu().numpy()
            mine = planted_slots[(planted_slots >= r0) & (planted_slots < r0 + len(h))]
            h[mine - r0] = planted[[dst[int(s)] for s in mine]]
            yield r0, h
    qv = {}
    for r0, h in host_chunks():
        for q in queries:
            if r0 <= q < r0 + len(h):
                qv[q] = h[q - r0].copy()
    hits = {q: ([], []) for q in queries}
    lo = min(thresholds)
    for r0, h in host_chunks():
        for q in queries:
            sc = oracle.scores(h, qv[q])
            with np.errstate(invalid="ignore"):
                sel = np.flatnonzero(sc >= lo)
            sel = sel[sel + r0 > q]
            hits[q][0].append(sel + r0)
            hits[q][1].append(sc[sel])
    out = {}
    for q in queries:
        b, v = np.concatenate(hits[q][0]), np.concatenate(hits[q][1])
        for t in thresholds:
            m = v >= t
            order = np.lexsort((b[m], -v[m]))
            out[(q, t)] = (b[m][order], v[m][order])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--placements", default="device,host")
    ap.add_argument("--thresholds", default="0.99,0.9")
    ap.add_argument("--page", type=int, default=1 << 25)
    ap.add_argument("--sample", type=int, default=64)
    ap.add_argument("--oracle-rows", type=int, default=8)
    a = ap.parse_args()
    import torch
    from runbookai_b200 import Index
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card, "rows": a.rows, "dim": a.dim, "runs": []}
    rng = np.random.default_rng(5)
    for placement in a.placements.split(","):
        with Index(a.dim, device=0, capacity_hint=a.rows, keep_f64=True, f64_on_host=placement == "host") as ix:
            src = np.arange(0, a.rows - 1, 97, dtype=np.int64)
            base = []
            for r0, x in corpus_chunks(a.rows, a.dim, 11):
                mine = src[(src >= r0) & (src < r0 + len(x))] - r0
                base.append(x[torch.as_tensor(mine, device="cuda")].cpu().numpy())
                torch.cuda.synchronize()
                ix.append_f64_device(x.data_ptr(), len(x))
                del x
            base = np.concatenate(base)
            planted = base * (1.0 + 1e-4 * np.random.default_rng(5).standard_normal(base.shape))
            ix.overwrite_f64_batch(src + 1, planted)
            del base
            torch.cuda.empty_cache()
            thresholds = [float(x) for x in a.thresholds.split(",")]
            picks = np.random.default_rng(9).choice(len(src), a.oracle_rows // 2, replace=False)
            oracle_q = sorted(set(src[picks].tolist()) | set(np.random.default_rng(10).choice(
                a.rows, a.oracle_rows - len(picks), replace=False).tolist()))
            engine = {}
            for t in thresholds:
                torch.cuda.synchronize()
                free_min = free0 = torch.cuda.mem_get_info()[0]
                pages, pairs, dev_ms, scan_ms, nxt = 0, 0, 0.0, 0.0, 0
                sample = []
                t0 = time.perf_counter()
                while nxt < a.rows:
                    pa, pb, ps, n2 = ix.similar_pairs(t, nxt, a.page)
                    st = ix.stats()
                    dev_ms += st["last_total_ms"]
                    scan_ms += st["last_scan_ms"]
                    free_min = min(free_min, torch.cuda.mem_get_info()[0])
                    pairs += len(pa)
                    for q in oracle_q:
                        m = pa == q
                        if m.any() or (q, t) not in engine:
                            engine[(q, t)] = (pb[m].copy(), ps[m].copy())
                    if len(pa) and len(sample) < a.sample:
                        firsts = np.unique(pa)
                        for q in rng.choice(firsts, min(len(firsts), 8), replace=False):
                            m = pa == q
                            sample.append((int(q), pb[m].copy(), ps[m].copy()))
                    nxt, pages = n2, pages + 1
                wall = time.perf_counter() - t0
                ok = True
                for q, b, s in sample:
                    sl, sv, sc, _ = ix.search_slots([q], ix.count(), t)
                    m = sl[0, :sc[0]] > q
                    ok &= bool((sl[0, :sc[0]][m] == b).all() and sv[0, :sc[0]][m].tobytes() == s.tobytes())
                res["runs"].append({"placement": placement, "min_score": t, "wall_s": round(wall, 3), "pages": pages,
                                    "pairs": pairs, "device_s": round(dev_ms / 1e3, 3),
                                    "scan_s": round(scan_ms / 1e3, 3),
                                    "rerank_and_rest_s": round((dev_ms - scan_ms) / 1e3, 3),
                                    "device_mem_held_mb": round((free0 - free_min) / 2**20, 1),
                                    "sampled_rows": len(sample), "sample_equals_search_slots": ok})
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ix.search_slots(np.arange(a.rows, dtype=np.int64), 10, None)
            res["runs"].append({"placement": placement, "all_neighbours_k10_wall_s": round(time.perf_counter() - t0, 3)})
            want = oracle_pairs(a.rows, a.dim, 11, src + 1, planted, oracle_q, thresholds)
            equal = all(engine[k][0].tolist() == want[k][0].tolist() and engine[k][1].tobytes() == want[k][1].tobytes()
                        for k in want)
            res["runs"].append({"placement": placement, "oracle_rows": oracle_q,
                                "oracle_pairs": sum(len(v[0]) for v in want.values()),
                                "oracle_equal": bool(equal)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
