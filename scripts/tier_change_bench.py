#!/usr/bin/env python
"""Changing the storage tier of a loaded KEEP_F64 index in place (rbk_index_set_tier): what each transition costs.

    python scripts/tier_change_bench.py [--rows 1000000] [--dim 1536] [--past-ceiling]

One KEEP_F64 index of arbitrary float64 rows (N(0,1), not bf16-representable; 12 GB of float64 at the defaults, on the
device and, after the first move, in pinned host memory) goes through the four single-flag transitions
    device/bf16 -> host/bf16 -> device/bf16 -> device/fp16 -> device/bf16.
For each one the JSON line reports the wall time of set_tier() (it is synchronous), the effective rate (the float64 bytes
moved over PCIe for a placement change; the float64 bytes read for a scan change), storage_bytes() before and after, and
a 64-query oracle parity check (ids and fp64 scores; the float64 oracle answers the queries once, on all host threads)
of the index after it.  The card name and power limit are read
in the same run (read-only nvidia-smi queries).

--past-ceiling (about 100 GB of host RAM): a second device-tier index is filled in 64 MB slices until an append fails
with RBK_ENOMEM, moved to host memory, and filled on past the old ceiling; then moving it back must fail with
RBK_ENOMEM and leave it as it was.  Reports the rows at each point and the time of the move.  Writes nothing to the
tree.
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

SEED = 0x5EED0007
CHUNK = 16384


def card_info() -> dict:
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def rows_at(i0: int, n: int, d: int) -> np.ndarray:
    """Rows [i0, i0 + n) of the corpus, generated per chunk so that the host never holds it all."""
    out = np.empty((n, d))
    for c0 in range(0, n, CHUNK):
        m = min(CHUNK, n - c0)
        out[c0:c0 + m] = np.random.default_rng([SEED, (i0 + c0) // CHUNK]).standard_normal((m, d))
    return out


def oracle_answers(oracle, corpus: np.ndarray, nq: int = 64, k: int = 20):
    """64 queries near corpus rows and the float64 oracle's answers to them (one query per host thread)."""
    from concurrent.futures import ThreadPoolExecutor
    rng = np.random.default_rng(SEED + 1)
    q = corpus[rng.choice(len(corpus), nq, replace=False)] + 0.3 * rng.standard_normal((nq, corpus.shape[1]))
    with ThreadPoolExecutor(oracle.host_threads()) as ex:
        ref = list(ex.map(lambda b: oracle.search(corpus, q[b], k, None), range(nq)))
    return q, k, ref


def parity(ix, q, k, ref) -> dict:
    slots, scores, counts, _ = ix.search(q, k, None)
    bad = 0
    for b, (es, ev) in enumerate(ref):
        ok = counts[b] == len(es) and (slots[b, :len(es)] == es).all() and scores[b, :len(es)].tobytes() == ev.tobytes()
        bad += not ok
    return {"queries": len(q), "k_fetch": k, "mismatches": bad}


def transitions(args, rb, oracle) -> list[dict]:
    n, d = args.rows, args.dim
    corpus = rows_at(0, n, d)
    q, k, ref = oracle_answers(oracle, corpus)
    out = []
    with rb.Index(d, capacity_hint=n, keep_f64=True) as ix:
        for i0 in range(0, n, CHUNK):
            ix.append_f64(corpus[i0:i0 + CHUNK])
        del corpus
        f64_bytes = n * d * 8
        out.append({"transition": "none (device/bf16 as loaded)", "parity": parity(ix, q, k, ref)})
        for name, kw in (("device->host", {"f64_on_host": True}), ("host->device", {"f64_on_host": False}),
                         ("bf16->fp16", {"scan_f16": True}), ("fp16->bf16", {"scan_f16": False})):
            before = ix.storage_bytes()
            t0 = time.perf_counter()
            ix.set_tier(**kw)
            sec = time.perf_counter() - t0
            out.append({"transition": name, "seconds": round(sec, 3), "f64_bytes": f64_bytes,
                        "effective_gb_per_s": round(f64_bytes / sec / 1e9, 2),
                        "storage_bytes_before": list(before), "storage_bytes_after": list(ix.storage_bytes()),
                        "flags_after": ix.flags, "parity": parity(ix, q, k, ref)})
    return out


def past_ceiling(args, rb) -> dict:
    d = args.dim
    slice_rows = max(1, (64 << 20) // (d * 8))
    res = {}
    with rb.Index(d, keep_f64=True) as ix:
        n = 0
        while True:
            try:
                ix.append_f64(rows_at(n, slice_rows, d))
            except rb.RbkError as e:
                if e.status != rb._native.RBK_ENOMEM:
                    raise
                break
            n += slice_rows
        res["device_ceiling_rows"] = ix.size()
        res["device_capacity_bytes"] = list(ix.storage_bytes())
        t0 = time.perf_counter()
        ix.set_tier(f64_on_host=True)
        res["move_to_host_seconds"] = round(time.perf_counter() - t0, 3)
        target = int(ix.size() * 1.25)
        while ix.size() < target:
            ix.append_f64(rows_at(ix.size(), slice_rows, d))
        res["rows_after_move"] = ix.size()
        res["storage_bytes_after"] = list(ix.storage_bytes())
        before = (ix.flags, ix.storage_bytes(), ix.size())
        try:
            ix.set_tier(f64_on_host=False)
            res["move_back"] = "accepted (unexpected)"
        except rb.RbkError as e:
            res["move_back"] = {"status": e.status, "message": str(e),
                                "unchanged": before == (ix.flags, ix.storage_bytes(), ix.size())}
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--past-ceiling", action="store_true")
    args = ap.parse_args()
    import oracle
    import runbookai_b200 as rb
    result = {"card": card_info(), "rows": args.rows, "dim": args.dim, "transitions": transitions(args, rb, oracle)}
    if args.past_ceiling:
        result["past_ceiling"] = past_ceiling(args, rb)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
