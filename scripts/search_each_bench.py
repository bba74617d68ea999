#!/usr/bin/env python
"""One micro-batcher window of mixed callers on one GPU: the strategy of a batcher without per-query parameters (one
search at the largest small k and the lowest threshold, cut again on the host, plus a large-k search of its own for
every caller whose k_fetch exceeds the scan's) against ONE rbk_index_search_each_f64 at every caller's own k_fetch and
min_score.

    python scripts/search_each_bench.py [--rows 1000000] [--dim 1536] [--rows-kind f64|bf16] [--placement device|host]
                                        [--steps 5] [--warmup 2]

The window is drawn from the reference's limits (search_knowledge 5, hooks / CLI 10, Agent.run 20, infra-context 50,
knowledge-context 1000; k_fetch = 2 * limit): k_fetch 10, 20, 40, 100, 2000.  The two strategies alternate step by step
after the warm-up, on the same card and clocks.  Prints one JSON line: the card name and power limit (read in the same
run), the median device time of each strategy (the sum of its calls' device times), their scan launches per window,
and whether every caller's answer is the same under both.  Writes nothing to the tree.
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

WINDOW_K = [10, 20, 40, 100, 10, 20, 2000, 2000, 2000]
WINDOW_MIN = [0.02, None, 0.03, 0.0, None, 0.05, 0.0, None, 0.01]


def fill(ix, rows, dim, kind, seed):
    """rows random rows made on the device in chunks (normal float64, or their bf16 copies), appended from there."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    chunk = max(1, (1 << 28) // (dim * 8))
    for r0 in range(0, rows, chunk):
        n = min(chunk, rows - r0)
        x = torch.randn(n, dim, dtype=torch.float64, device="cuda", generator=g)
        if kind == "bf16":
            x = x.to(torch.bfloat16).contiguous()
            torch.cuda.synchronize()
            ix.append_bf16_device(x.data_ptr(), n)
        else:
            torch.cuda.synchronize()
            ix.append_f64_device(x.data_ptr(), n)
        del x


def split_strategy(ix, q, ks, mins):
    """One shared search for the callers the scan can serve (largest k, lowest threshold), each re-cut on the host; a
    search_any_k of its own for every other caller."""
    small = [b for b in range(len(q)) if ks[b] <= 112]
    big = [b for b in range(len(q)) if ks[b] > 112]
    out, ms = {}, 0.0
    if small:
        lo = [m for m in (mins[b] for b in small)]
        floor = None if any(m is None for m in lo) else min(lo)
        s, v, c, t = ix.search(q[small], max(ks[b] for b in small), floor)
        ms += t
        for i, b in enumerate(small):
            n = int(c[i])
            keep = np.ones(n, bool) if mins[b] is None else v[i, :n] >= mins[b]
            out[b] = (s[i, :n][keep][:ks[b]], v[i, :n][keep][:ks[b]])
    for b in big:
        s, v, c, t = ix.search_any_k(q[b:b + 1], ks[b], mins[b])
        ms += t
        out[b] = (s[0, :c[0]], v[0, :c[0]])
    return out, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--rows-kind", choices=["f64", "bf16"], default="f64")
    ap.add_argument("--placement", choices=["device", "host"], default="device",
                    help="where the float64 exact rows live (f64 rows only)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    from runbookai_b200 import Index
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    kw = {} if a.rows_kind == "bf16" else {"keep_f64": True, "f64_on_host": a.placement == "host"}
    rng = np.random.default_rng(7)
    q = rng.standard_normal((len(WINDOW_K), a.dim))
    with Index(a.dim, device=0, capacity_hint=a.rows, **kw) as ix:
        fill(ix, a.rows, a.dim, a.rows_kind, 11)
        torch.cuda.empty_cache()
        t_split, t_each, equal = [], [], True
        launches = {}
        for step in range(a.warmup + a.steps):
            s0 = ix.stats()["scan_launches"]
            ref, ms_split = split_strategy(ix, q, WINDOW_K, WINDOW_MIN)
            s1 = ix.stats()["scan_launches"]
            slots, scores, counts, ms_each = ix.search_each(q, WINDOW_K, WINDOW_MIN)
            s2 = ix.stats()["scan_launches"]
            launches = {"split": s1 - s0, "search_each": s2 - s1}
            for b in range(len(q)):
                n = int(counts[b])
                es, ev = ref[b]
                equal &= len(es) == n and (slots[b, :n] == es).all() and scores[b, :n].tobytes() == ev.tobytes()
            if step >= a.warmup:
                t_split.append(ms_split)
                t_each.append(ms_each)
    print(json.dumps({
        "card": card, "rows": a.rows, "dim": a.dim, "rows_kind": a.rows_kind,
        "placement": a.placement if a.rows_kind == "f64" else "device",
        "window_k_fetch": WINDOW_K, "window_min_score": WINDOW_MIN,
        "split_ms_median": round(float(np.median(t_split)), 3), "search_each_ms_median": round(float(np.median(t_each)), 3),
        "split_ms": [round(t, 3) for t in t_split], "search_each_ms": [round(t, 3) for t in t_each],
        "scan_launches_per_window": launches, "answers_equal": bool(equal)}))


if __name__ == "__main__":
    main()
