#!/usr/bin/env python
"""How far one GPU's index grows, what each growth step costs, and what trim() gives back.

    python scripts/growth_bench.py [--dim 1536] [--reserve-mb 256] [--max-rows 0]

One KEEP_F64 index on the device tier (the layout VectorStore builds) is created without a capacity hint and loaded
with float64 rows from the host in 64 MB slices, exactly as VectorStore loads its sidecar, until an append fails with
RBK_ENOMEM.  A torch tensor of --reserve-mb is held during the load and released afterwards, so that the compaction
below has room for its scratch; both builds being compared hold the same reserve.  Then every other row is deleted,
the index is compacted and trimmed (a build without trim stops after the load).  Reports, as one JSON line:
  * the rows reached and the capacity at the failure;
  * every growth step: the capacity before and after, and the wall time of the append that grew (the call is
    synchronous up to its last copy), next to the median time of an append that did not grow;
  * the free device memory trim() returned, the drop in storage_bytes() and the difference (the chunk slack);
  * the card name and power limit.
Writes nothing to the tree.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--reserve-mb", type=int, default=256)
    ap.add_argument("--max-rows", type=int, default=0, help="stop here instead of at RBK_ENOMEM (0: no limit)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("growth_bench.py needs a CUDA device: this engine has no CPU path")
    import runbookai_b200._native as nat
    d = args.dim
    step = max(1, (64 << 20) // (d * 8))                       # vector_store.py's sidecar slice
    rows = np.random.default_rng(5).standard_normal((step, d))
    reserve = torch.empty(args.reserve_mb << 20, dtype=torch.uint8, device="cuda")
    ix = nat.Index(d, 0, keep_f64=True)
    growth, plain_ms = [], []
    stop = "max_rows"
    t_load = time.perf_counter()
    while not args.max_rows or ix.size() < args.max_rows:
        before = ix.storage_bytes()[0]
        t0 = time.perf_counter()
        try:
            ix.append_f64(rows)
        except nat.RbkError as e:
            if e.status != nat.RBK_ENOMEM:
                raise
            stop = "RBK_ENOMEM: " + str(e)
            break
        ms = (time.perf_counter() - t0) * 1e3
        after = ix.storage_bytes()[0]
        if after != before:
            growth.append({"rows": ix.size(), "storage_gb_before": before / 1e9, "storage_gb_after": after / 1e9,
                           "append_ms": ms})
        else:
            plain_ms.append(ms)
    load_s = time.perf_counter() - t_load
    reached, storage_full = ix.size(), ix.storage_bytes()[0]
    del reserve
    torch.cuda.empty_cache()

    trim = None
    if hasattr(ix, "trim") and hasattr(nat.lib, "rbk_index_trim"):   # a build without trim stops at the load
        ix.tombstone(np.arange(0, reached, 2))
        ix.compact()
        torch.cuda.synchronize()
        free0, stored0 = torch.cuda.mem_get_info()[0], ix.storage_bytes()[0]
        t0 = time.perf_counter()
        ix.trim()
        trim_ms = (time.perf_counter() - t0) * 1e3
        free1, stored1 = torch.cuda.mem_get_info()[0], ix.storage_bytes()[0]
        trim = {"seconds": trim_ms / 1e3, "live_rows": ix.size(), "storage_gb_before": stored0 / 1e9,
                "storage_gb_after": stored1 / 1e9, "free_gb_returned": (free1 - free0) / 1e9,
                "returned_minus_storage_drop_gb": ((free1 - free0) - (stored0 - stored1)) / 1e9}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,memory.total", "--format=csv,noheader",
                           "-i", "0"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "metric": "index_growth", "card": card,
        "config": {"dim": d, "keep_f64": True, "tier": "device", "slice_rows": step, "reserve_mb": args.reserve_mb},
        "rows_reached": reached, "storage_gb_at_stop": storage_full / 1e9, "stop": stop, "load_seconds": load_s,
        "growth_steps": growth,
        "median_append_ms_without_growth": float(np.median(plain_ms)) if plain_ms else None,
        "trim": trim}), flush=True)
    ix.close()


if __name__ == "__main__":
    main()
