#!/usr/bin/env python
"""Compaction on one GPU: what rbk_index_compact costs, and what it gives back to every search.

    python scripts/compact_bench.py [--rows 2000000] [--dim 1536] [--batch 32] [--steps 10] [--warmup 3]

Two KEEP_F64 indexes (the layout VectorStore builds) receive the same rows; about half of the rows are then deleted
in runs of 8-40 contiguous slots, the shape `KnowledgeRetriever.sync()` leaves behind when documents change.  One
index is compacted.  Reports, as one JSON line:
  * the compaction's wall time (the call is synchronous) and its bytes moved / time against the H100 data sheet's
    3.35 TB/s, counting read plus write of 2*dpad + 8*d + 12 bytes per moved row;
  * the search device time of both indexes (same live rows), alternated call by call: B queries with k_fetch 20
    (VectorStore's shape) and k_fetch 1000 (the large-k search);
  * oracle parity of both on the queries (ids and fp64 scores), with the card name and power limit.
Writes nothing to the tree.  Corpus generation is bench.py's.
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

import bench  # noqa: E402  (corpus generator, data-sheet peaks)


def deletion_runs(n: int, frac: float, seed: int) -> np.ndarray:
    """Slots to delete: runs of 8-40 contiguous slots, each run deleted with probability `frac`."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(8, 41, size=n // 8 + 1)
    starts = np.concatenate([[0], np.cumsum(lens)])
    starts = starts[starts < n]
    live = np.ones(n, dtype=bool)
    for s, ln, kill in zip(starts, lens, rng.random(len(starts)) < frac):
        if kill:
            live[s:s + ln] = False
    return np.flatnonzero(~live)


def same(a, b) -> bool:
    return (a[0] == b[0]).all() and a[1].tobytes() == b[1].tobytes() and (a[2] == b[2]).all()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--delete", type=float, default=0.5, help="fraction of the deletion runs applied")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("compact_bench.py needs a CUDA device: this engine has no CPU path")
    import oracle
    import runbookai_b200._native as nat
    n, d, B = args.rows, args.dim, args.batch
    synth, pk = bench.load_synth(), bench.peaks()
    dev = torch.device("cuda", 0)
    plain = nat.Index(d, 0, n, keep_f64=True)
    packed = nat.Index(d, 0, n, keep_f64=True)
    bench.gen_shard(plain, 0, n, d, dev)
    bench.gen_shard(packed, 0, n, d, dev)
    torch.cuda.empty_cache()
    dead = deletion_runs(n, args.delete, bench.SEED + 7)
    plain.tombstone(dead)
    packed.tombstone(dead)
    q = synth.random_queries(B, d, bench.SEED + 1).astype(np.float64)
    before = {k: packed.search_any_k(q, k, None)[:3] for k in (20, 1000)}

    t0 = time.perf_counter()
    old_to_new = packed.compact()
    compact_s = time.perf_counter() - t0
    live = old_to_new >= 0
    moved = int((live & (old_to_new != np.arange(n))).sum())
    dpad = -(-d // 64) * 64
    row_bytes = 2 * dpad + 8 * d + 12
    moved_bytes = 2.0 * moved * row_bytes                   # read + write
    assert packed.size() == packed.count() == plain.count() == int(live.sum())

    timing = {}
    for k in (20, 1000):
        fn = {"plain": (lambda q_, k_=k: plain.search_any_k(q_, k_, None)),
              "compacted": (lambda q_, k_=k: packed.search_any_k(q_, k_, None))}
        for _ in range(args.warmup):
            for f in fn.values():
                f(q)
        ms = {name: [] for name in fn}
        res = {}
        for _ in range(args.steps):
            for name, f in fn.items():                      # alternated call by call: same clocks for both
                res[name] = f(q)
                ms[name].append(res[name][3])               # device time of the whole call (CUDA events)
        p, c = res["plain"][:3], res["compacted"][:3]
        renumber = lambda r: (np.where(r[0] >= 0, old_to_new[np.maximum(r[0], 0)], -1), r[1], r[2])  # noqa: E731
        med = {name: float(np.median(v)) for name, v in ms.items()}
        timing[f"k_fetch_{k}"] = {"plain_ms": med["plain"], "compacted_ms": med["compacted"],
                                  "speedup": med["plain"] / med["compacted"],
                                  "plain_equals_compacted_through_map": bool(same(renumber(p), c)),
                                  "same_index_before_equals_after_through_map": bool(same(renumber(before[k]), c))}

    # oracle parity: the plain index against the oracle over its rows with the tombstones, the compacted one against
    # the oracle over its own (fewer) rows
    t0 = time.perf_counter()
    parity = {}
    for k in (20, 1000):
        ref_p = oracle.search_chunked(plain.read_rows_bf16, n, q, k, None, live=live.astype(np.uint8))
        ref_c = oracle.search_chunked(packed.read_rows_bf16, packed.size(), q, k, None)
        got_p = plain.search_any_k(q, k, None)[:3]
        got_c = packed.search_any_k(q, k, None)[:3]
        parity[f"k_fetch_{k}"] = {"plain": bool(same(got_p, ref_p)), "compacted": bool(same(got_c, ref_c))}
    parity["queries"] = B
    parity["seconds"] = time.perf_counter() - t0
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "metric": "compaction", "card": card,
        "config": {"rows": n, "dim": d, "batch": B, "deleted": int(len(dead)), "live": int(live.sum()),
                   "keep_f64": True, "steps": args.steps, "warmup": args.warmup},
        "compact": {"seconds": compact_s, "moved_rows": moved, "bytes_moved": moved_bytes,
                    "tb_per_s": moved_bytes / compact_s / 1e12, "frac_of_hbm_peak": moved_bytes / compact_s / (pk["hbm"] * 1e9),
                    "peaks": pk, "note": "wall time of the synchronous call, including the D2H of old_to_new"},
        "search_device_ms": timing, "parity": parity}), flush=True)
    plain.close()
    packed.close()


if __name__ == "__main__":
    main()
