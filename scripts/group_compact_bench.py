#!/usr/bin/env python
"""Compaction of a device group: what rbk_group_compact costs, and what it gives back to every search.

    python scripts/group_compact_bench.py [--gpus G] [--rows-per-gpu 1000000] [--dim 1536] [--batch 32]
                                          [--steps 10] [--warmup 3]

One KEEP_F64 group (the layout VectorStore builds) over G GPUs (all visible by default) receives about rows-per-gpu
rows per GPU; about half of them are then deleted in runs of 8-40 contiguous slots, the shape
`KnowledgeRetriever.sync()` leaves behind when documents change, and the group is compacted.  Reports, as one JSON
line:
  * the wall time of the synchronous call;
  * the rows and bytes that change device and that stay on their device, from the block-cyclic layout the copy plan
    follows (a row whose slot changes is staged once and copied once: 2*dpad + 8*d + 12 bytes);
  * the search device time before and after (B queries, k_fetch 20 and 1000), and whether the answers after equal
    those before through old_to_new;
  * the card name, power limit and GPU count, read in the same run.
Writes nothing to the tree.  Corpus generation is bench.py's (bf16-rounded N(0,1) rows, generated on the device).
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

import bench  # noqa: E402  (corpus seed, synth)
from scripts.compact_bench import deletion_runs, same  # noqa: E402

BLOCK = 4096


def fill(g, n: int, d: int, device):
    """bench.gen_shard's corpus, through the host (a group appends host rows)."""
    import torch
    gen = torch.Generator(device=device)
    for c in range(-(-n // bench.GEN_CHUNK)):
        gen.manual_seed(bench.SEED * 1_000_003 + c)
        t = torch.randn(bench.GEN_CHUNK, d, device=device, generator=gen, dtype=torch.float32).to(torch.bfloat16)
        rows = t[:min(bench.GEN_CHUNK, n - c * bench.GEN_CHUNK)].view(torch.int16).cpu().numpy().view(np.uint16)
        g.append_bf16(rows)
        del t


def timed(fn, q, warmup: int, steps: int):
    for _ in range(warmup):
        fn(q)
    ms, res = [], None
    for _ in range(steps):
        res = fn(q)
        ms.append(res[3])                                   # device time of the whole call (CUDA events)
    return float(np.median(ms)), res[:3]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=0, help="GPUs in the group (0: all visible)")
    ap.add_argument("--rows-per-gpu", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--delete", type=float, default=0.5, help="fraction of the deletion runs applied")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("group_compact_bench.py needs a CUDA device: this engine has no CPU path")
    import runbookai_b200._native as nat
    G = args.gpus or torch.cuda.device_count()
    n, d, B = args.rows_per_gpu * G, args.dim, args.batch
    synth = bench.load_synth()
    g = nat.Group(d, list(range(G)), n, keep_f64=True)
    fill(g, n, d, torch.device("cuda", 0))
    torch.cuda.empty_cache()
    dead = deletion_runs(n, args.delete, bench.SEED + 7)
    g.tombstone(dead)
    q = synth.random_queries(B, d, bench.SEED + 1).astype(np.float64)
    searches = {20: lambda q_: g.search(q_, 20, None), 1000: lambda q_: g.search_large(q_, 1000, None)}
    before = {k: timed(f, q, args.warmup, args.steps) for k, f in searches.items()}

    t0 = time.perf_counter()
    old_to_new = g.compact()
    compact_s = time.perf_counter() - t0
    live = old_to_new >= 0
    assert g.size() == g.count() == int(live.sum())
    old = np.flatnonzero(live & (old_to_new != np.arange(n)))
    new = old_to_new[old]
    between = int(((old // BLOCK) % G != (new // BLOCK) % G).sum())
    dpad = -(-d // 64) * 64
    row_bytes = 2 * dpad + 8 * d + 12

    timing = {}
    for k, f in searches.items():
        ms, got = timed(f, q, args.warmup, args.steps)
        b_ms, b_got = before[k]
        renumbered = (np.where(b_got[0] >= 0, old_to_new[np.maximum(b_got[0], 0)], -1), b_got[1], b_got[2])
        timing[f"k_fetch_{k}"] = {"before_ms": b_ms, "after_ms": ms, "speedup": b_ms / ms,
                                  "after_equals_before_through_map": bool(same(renumbered, got))}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "metric": "group_compaction", "card": card, "gpus": G,
        "config": {"rows": n, "dim": d, "batch": B, "deleted": int(len(dead)), "live": int(live.sum()),
                   "keep_f64": True, "steps": args.steps, "warmup": args.warmup},
        "compact": {"seconds": compact_s, "moved_rows": int(len(old)), "rows_between_devices": between,
                    "rows_within_a_device": int(len(old)) - between, "bytes_between_devices": between * row_bytes,
                    "bytes_within_a_device": (int(len(old)) - between) * row_bytes,
                    "note": "wall time of the synchronous call, including old_to_new"},
        "search_device_ms": timing}), flush=True)
    g.close()


if __name__ == "__main__":
    main()
