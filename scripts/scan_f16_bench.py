#!/usr/bin/env python
"""The fp16 scan (RBK_INDEX_SCAN_F16) against the default bf16 scan of float64-backed indexes.

    python scripts/scan_f16_bench.py [--rows 1000000] [--dim 1536] [--steps 5] [--big-rows 5000000] [--big-dim 768]

Reports, as one JSON line:
  * the card name and power limit (read-only nvidia-smi queries);
  * for each float64 placement (device, pinned host): a bf16-tier and an fp16-tier KEEP_F64 index fed the same
    arbitrary float64 rows (N(0,1), --rows x --dim), queries = a corpus row + 0.05 noise (the near-tied case of
    DESIGN.md §7); B in {1, 32, 256} at k_fetch 20 and 1000, the two tiers alternated call by call: median device ms,
    and the retry_batches / fallback_queries added per call; oracle parity of every answer (ids and fp64 score bytes);
  * the append time of each index (host float64 source) and the ingest kernels alone (device float64 source);
  * the scan kernel time at --big-rows x --big-dim (device tier, B = 1024, k_fetch 20), from the scan timing events
    (stats scan_ms_total / scans_timed): one index at a time (two do not fit), built bf16, fp16, bf16, fp16 from the
    same rows.
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

SEED = 0x5EED0016


def card_info() -> dict:
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def oracle_answers(oracle, corpus, q, k):
    def one(b):
        return oracle.search(corpus, q[b], k, None)

    with ThreadPoolExecutor(max_workers=oracle.host_threads()) as ex:
        return list(ex.map(one, range(len(q))))


def parity(ans, want) -> bool:
    slots, scores, counts = ans[:3]
    k = slots.shape[1]
    for b, (es, ev) in enumerate(want):
        m = min(k, len(es))
        if counts[b] != m or not (slots[b, :m] == es[:m]).all() or scores[b, :m].tobytes() != ev[:m].tobytes():
            return False
    return True


def counters(ix):
    st = ix.stats()
    return st["retry_batches"], st["fallback_queries"], st["scan_ms_total"], st["scans_timed"]


def search(ix, q, k):
    return ix.search(q, k, None) if k <= 112 else ix.search_large(q, k, None)


def placement_run(nat, want, corpus, q, placement, steps, torch):
    d = corpus.shape[1]
    tiers = {}
    out = {"append_s": {}, "ingest_kernels_ms": {}}
    for name, f16 in (("bf16", False), ("f16", True)):
        ix = nat.Index(d, 0, len(corpus), keep_f64=True, f64_on_host=placement == "host", scan_f16=f16)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.append_f64(corpus)
        torch.cuda.synchronize()
        out["append_s"][name] = time.perf_counter() - t0
        tiers[name] = ix
    # the ingest kernels alone: 65 536 device-resident float64 rows into a fresh index of each tier, CUDA events
    chunk = torch.from_numpy(corpus[:65536]).cuda()
    torch.cuda.synchronize()
    for name, f16 in (("bf16", False), ("f16", True)):
        times = []
        for _ in range(3):
            with nat.Index(d, 0, 65536, keep_f64=True, f64_on_host=placement == "host", scan_f16=f16) as ix:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ix.set_stream(torch.cuda.current_stream().cuda_stream)
                e0.record()
                ix.append_f64_device(chunk.data_ptr(), len(chunk))
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
        out["ingest_kernels_ms"][name] = float(np.median(times))
    del chunk
    res = {}
    for k in (20, 1000):
        for B in (1, 32, 256):
            key = f"B{B}_k{k}"
            res[key] = {}
            ms = {n: [] for n in tiers}
            dr = {n: [] for n in tiers}
            df = {n: [] for n in tiers}
            ok = {n: True for n in tiers}
            sub = [want[k][b] for b in range(B)]
            for step in range(steps + 1):
                for name, ix in tiers.items():       # alternated call by call
                    r0, f0, _, _ = counters(ix)
                    ans = search(ix, q[:B], k)
                    r1, f1, _, _ = counters(ix)
                    if step == 0:
                        ok[name] = parity(ans, sub)
                        continue                       # warm-up
                    ms[name].append(ans[3])
                    dr[name].append(r1 - r0)
                    df[name].append(f1 - f0)
            print(f"{placement} {key} done", file=sys.stderr, flush=True)
            for name in tiers:
                res[key][name] = {"device_ms": float(np.median(ms[name])), "retry_per_call": float(np.mean(dr[name])),
                                  "fallback_per_call": float(np.mean(df[name])), "oracle_parity": ok[name]}
    for ix in tiers.values():
        ix.close()
    out["search"] = res
    return out


def big_scan(nat, torch, n, d, steps):
    """Scan kernel ms at n x d, B = 1024: bf16, fp16, bf16, fp16 indexes built one at a time from the same rows."""
    chunk = 250000
    out = {"bf16": [], "f16": []}
    q = torch.randn(1024, d, dtype=torch.float64, generator=torch.Generator().manual_seed(3)).numpy()
    for name, f16 in (("bf16", False), ("f16", True), ("bf16", False), ("f16", True)):
        with nat.Index(d, 0, n, keep_f64=True, scan_f16=f16) as ix:
            g = torch.Generator(device="cuda").manual_seed(7)
            for first in range(0, n, chunk):
                t = torch.randn(min(chunk, n - first), d, dtype=torch.float64, device="cuda", generator=g)
                torch.cuda.synchronize()
                ix.append_f64_device(t.data_ptr(), len(t))
                del t
            ix.search(q, 20, None)                   # warm-up
            _, _, s0, n0 = counters(ix)
            for _ in range(steps):
                ix.search(q, 20, None)
            _, _, s1, n1 = counters(ix)
            out[name].append((s1 - s0) / max(1, n1 - n0))
            print(f"big scan {name}: {out[name][-1]:.3f} ms", file=sys.stderr, flush=True)
    return {k: [round(x, 3) for x in v] for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--big-rows", type=int, default=5_000_000)
    ap.add_argument("--big-dim", type=int, default=768)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("scan_f16_bench.py needs a CUDA device: this engine has no CPU path")
    import oracle
    import runbookai_b200._native as nat
    rng = np.random.default_rng(SEED)
    corpus = rng.standard_normal((args.rows, args.dim))
    q = corpus[rng.choice(args.rows, 256, replace=False)] + 0.05 * rng.standard_normal((256, args.dim))
    report = {"card": card_info(), "rows": args.rows, "dim": args.dim, "steps": args.steps}
    want = {k: oracle_answers(oracle, corpus, q, k) for k in (20, 1000)}
    print("oracle done", file=sys.stderr, flush=True)
    for placement in ("device", "host"):
        report[placement] = placement_run(nat, want, corpus, q, placement, args.steps, torch)
    del corpus
    if args.big_rows > 0:
        report["scan_ms_big"] = {"rows": args.big_rows, "dim": args.big_dim, "B": 1024,
                                 **big_scan(nat, torch, args.big_rows, args.big_dim, args.steps)}
    print(json.dumps(report))


if __name__ == "__main__":
    main()
