#!/usr/bin/env python
"""Float64 rows on the GPU or in pinned host memory (RBK_INDEX_F64_ON_HOST): what each placement costs.

    python scripts/host_rows_bench.py [--rows 1000000] [--dim 1536] [--steps 10] [--warmup 3]

Two KEEP_F64 indexes (the layout VectorStore builds) receive the same arbitrary float64 rows (N(0,1), not
bf16-representable; about 12 GB of pinned host memory at the defaults), one with its float64 rows on the device, one
with them in pinned host memory.  A tie group of 150 copies of one row is planted so that one query must take the
exhaustive fallback.  Reports, as one JSON line:
  * the card name, power limit and PCIe link (read-only nvidia-smi queries);
  * the pinned host-to-device cudaMemcpy rate measured in the same run: the ceiling for reads of host rows;
  * storage_bytes() of both indexes;
  * search device time of both tiers, alternated call by call: B in {1, 32, 256} at k_fetch 20, and B = 32 at
    k_fetch 1000 (large-k), with the host-row bytes each search read and that rate against the copy rate;
  * the append (host float64 source) and compaction (half of the rows deleted in runs of 8-40 slots, as in
    compact_bench.py) time of both tiers, the forced exhaustive-fallback query and one exact_scores call;
  * oracle parity of every query of both indexes (ids and fp64 scores) and bit-equality between the tiers.
Writes nothing to the tree.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from compact_bench import deletion_runs  # noqa: E402

SEED = 0x5EED0004
TIES = 150


def same(a, b) -> bool:
    return all(x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def card_info() -> dict:
    q = "name,power.limit,pcie.link.gen.current,pcie.link.gen.max,pcie.link.width.current,pcie.link.width.max"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def h2d_rate_gbs(torch, mb: int = 1024, reps: int = 10) -> float:
    """Pinned host -> device cudaMemcpy, GB/s (1e9 bytes), median of `reps` copies of `mb` MiB."""
    src = torch.empty(mb << 20, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(mb << 20, dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dst.copy_(src, non_blocking=True)
    rates = []
    for _ in range(reps):
        e0.record()
        dst.copy_(src, non_blocking=True)
        e1.record()
        e1.synchronize()
        rates.append(src.numel() / (e0.elapsed_time(e1) * 1e-3) / 1e9)
    return float(np.median(rates))


def oracle_answers(oracle, corpus, q, ks, live=None):
    """(slots, scores, counts) per k for every query, from the f64 oracle, one query per thread (ctypes drops the
    GIL)."""
    kmax = max(ks)

    def one(b):
        return oracle.search(corpus, q[b], kmax, None, live=live)

    with ThreadPoolExecutor(max_workers=oracle.host_threads()) as ex:
        res = list(ex.map(one, range(len(q))))
    out = {}
    for k in ks:
        s = np.full((len(q), k), -1, np.int64)
        v = np.full((len(q), k), np.nan)
        c = np.zeros(len(q), np.int32)
        for b, (es, ev) in enumerate(res):
            m = min(k, len(es))
            s[b, :m], v[b, :m], c[b] = es[:m], ev[:m], m
        out[k] = (s, v, c)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("host_rows_bench.py needs a CUDA device: this engine has no CPU path")
    import oracle
    import runbookai_b200._native as nat
    n, d = args.rows, args.dim
    rng = np.random.default_rng(SEED)
    corpus = rng.standard_normal((n, d))
    tie_rows = rng.choice(n, TIES, replace=False)
    corpus[tie_rows] = corpus[tie_rows[0]]
    q = corpus[rng.choice(n, 256, replace=False)] + 0.5 * rng.standard_normal((256, d))
    q_tie = corpus[tie_rows[0]][None, :] * 1.5

    copy_gbs = h2d_rate_gbs(torch)
    tiers = {"device": nat.Index(d, 0, n, keep_f64=True), "host": nat.Index(d, 0, n, keep_f64=True, f64_on_host=True)}
    append_s = {}
    for name, ix in tiers.items():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.append_f64(corpus)
        torch.cuda.synchronize()
        append_s[name] = time.perf_counter() - t0
    storage = {name: dict(zip(("device_bytes", "pinned_host_bytes"), ix.storage_bytes())) for name, ix in tiers.items()}
    per_row = {name: (s["device_bytes"] / n, s["pinned_host_bytes"] / n) for name, s in storage.items()}

    shapes = [(1, 20), (32, 20), (256, 20), (32, 1000)]
    timing, results = {}, {}
    for B, k in shapes:
        def call(ix, B=B, k=k):
            return ix.search(q[:B], k, None) if k <= nat.RBK_MAX_K_FETCH else ix.search_large(q[:B], k, None)
        for _ in range(args.warmup):
            for ix in tiers.values():
                call(ix)
        ms = {name: [] for name in tiers}
        retry0 = tiers["host"].stats()["retry_batches"]
        for _ in range(args.steps):
            for name, ix in tiers.items():              # alternated call by call: same clocks for both
                r = call(ix)
                ms[name].append(r[3])
                results[(name, B, k)] = r[:3]
        med = {name: float(np.median(v)) for name, v in ms.items()}
        if k <= nat.RBK_MAX_K_FETCH:
            # k' rows per query, and k' = 128 once more for a batch whose proof failed and was rescanned
            kp = min(128, -(-(k + 16) // 16) * 16)
            retried = (tiers["host"].stats()["retry_batches"] - retry0) / args.steps
            host_bytes = int(B * (kp + 128 * retried) * 8 * d)
            note = f"k' = {kp} rows per query; {retried:.2f} wide rescans (k' = 128) per call"
        else:
            host_bytes = B * k * 8 * d
            note = "lower bound: k_fetch rows per query (the re-rank reads every emitted candidate, at least k_fetch)"
        timing[f"B{B}_k{k}"] = {
            "device_tier_ms": med["device"], "host_tier_ms": med["host"], "host_over_device": med["host"] / med["device"],
            "host_row_bytes": host_bytes, "host_row_bytes_note": note,
            "host_row_gbs_over_whole_call": host_bytes / (med["host"] * 1e-3) / 1e9,
            "share_of_copy_rate": host_bytes / (med["host"] * 1e-3) / 1e9 / copy_gbs,
            "tiers_bit_equal": bool(same(results[("device", B, k)], results[("host", B, k)]))}

    # forced exhaustive fallback: 150 tied rows, k_fetch 20 (the retry with k' = 128 cannot hold them)
    fallback = {}
    for name, ix in tiers.items():
        st0 = ix.stats()
        r = ix.search(q_tie, 20, None)
        st1 = ix.stats()
        fallback[name] = {"ms": r[3], "fallback_queries": st1["fallback_queries"] - st0["fallback_queries"],
                          "retry_batches": st1["retry_batches"] - st0["retry_batches"], "result": r[:3]}
    # the k > 4096 route: the exact cosine of every row (one query)
    exact = {}
    for name, ix in tiers.items():
        t0 = time.perf_counter()
        exact[name] = ix.exact_scores(q[:1])
        exact[f"{name}_s"] = time.perf_counter() - t0

    t0 = time.perf_counter()
    ref = oracle_answers(oracle, corpus, np.concatenate([q, q_tie]), (20, 1000))
    oracle_s = time.perf_counter() - t0
    parity = {}
    for name in tiers:
        ok = True
        for B, k in shapes:
            ok &= same(results[(name, B, k)], tuple(x[:B] for x in ref[k]))
        ok &= same(fallback[name]["result"], tuple(x[256:] for x in ref[20]))
        parity[name] = bool(ok)
    parity["queries"] = 257
    parity["oracle_seconds"] = oracle_s
    parity["fallback_tiers_bit_equal"] = bool(same(fallback["device"]["result"], fallback["host"]["result"]))
    parity["exact_scores_tiers_bit_equal"] = bool(exact["device"].tobytes() == exact["host"].tobytes())

    # compaction: half of the rows deleted in document-sized runs
    dead = deletion_runs(n, 0.5, SEED + 7)
    compact_s, maps = {}, {}
    for name, ix in tiers.items():
        ix.tombstone(dead)
        t0 = time.perf_counter()
        maps[name] = ix.compact()
        compact_s[name] = time.perf_counter() - t0
    after = {name: ix.search(q[:32], 20, None)[:3] for name, ix in tiers.items()}

    print(json.dumps({
        "metric": "host_rows", "card": card_info(),
        "config": {"rows": n, "dim": d, "rows_kind": "N(0,1) float64", "steps": args.steps, "warmup": args.warmup,
                   "tie_group": TIES},
        "pinned_h2d_copy_gbs": copy_gbs,
        "storage_bytes": storage, "bytes_per_row": per_row,
        "device_bytes_ratio": storage["device"]["device_bytes"] / storage["host"]["device_bytes"],
        "append_seconds": append_s,
        "append_rows_per_s": {name: n / s for name, s in append_s.items()},
        "search_device_ms": timing,
        "fallback_query": {name: {k: v for k, v in f.items() if k != "result"} for name, f in fallback.items()},
        "exact_scores_one_query_s": {name: exact[f"{name}_s"] for name in tiers},
        "compaction": {"deleted": int(len(dead)), "seconds": compact_s,
                       "maps_equal": bool(maps["device"].tobytes() == maps["host"].tobytes()),
                       "tiers_bit_equal_after": bool(same(after["device"], after["host"]))},
        "parity": parity}), flush=True)
    for ix in tiers.values():
        ix.close()


if __name__ == "__main__":
    main()
