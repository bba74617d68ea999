#!/usr/bin/env python
"""Float32 exact rows (RBK_INDEX_KEEP_F32) and split float32 rows (RBK_INDEX_KEEP_F32_SPLIT) against float64 ones
(RBK_INDEX_KEEP_F64): what the narrower rows save.

    python scripts/f32_rows_bench.py [--rows 1000000] [--dim 1536] [--steps 5] [--warmup 2]

Six indexes receive the same float32-exact rows (N(0,1) drawn as float32, widened to float64; about 21 GB of pinned
host memory at the defaults): KEEP_F64, KEEP_F32 and KEEP_F32_SPLIT, each with its exact rows on the device and in
pinned host memory (RBK_INDEX_F64_ON_HOST).  A tie group of 150 copies of one row is planted so that one query must take
the exhaustive fallback.  Reports, as one JSON line:
  * the card name, power limit and PCIe link (read-only nvidia-smi queries);
  * storage_bytes() of all six indexes;
  * the append time of each from a host float64 source (the float32 widths: with the float32-exactness check);
  * search device time, the three widths alternated call by call, on each tier: B in {1, 32, 256} x k_fetch in
    {20, 1000};
  * the forced exhaustive-fallback query and one exact_scores query on each index;
  * the wall time of in-place set_tier changes of the device-tier KEEP_F64 index: F64 -> F32, F32 -> split,
    split -> F32, F32 -> F64 and F64 -> split;
  * bit-equality of every answer between the widths, and oracle parity (ids and fp64 scores) of 64 queries.
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

SEED = 0x5EED0032
TIES = 150
CHECKED = 64   # queries checked against the oracle


def same(a, b) -> bool:
    return all(x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def card_info() -> dict:
    q = "name,power.limit,pcie.link.gen.current,pcie.link.width.current"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def oracle_answers(oracle, corpus, q, ks):
    kmax = max(ks)
    with ThreadPoolExecutor(max_workers=oracle.host_threads()) as ex:
        res = list(ex.map(lambda b: oracle.search(corpus, q[b], kmax, None), range(len(q))))
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


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("f32_rows_bench.py needs a CUDA device: this engine has no CPU path")
    import oracle
    import runbookai_b200._native as nat
    n, d = args.rows, args.dim
    rng = np.random.default_rng(SEED)
    corpus = rng.standard_normal((n, d), dtype=np.float32).astype(np.float64)   # float32-exact float64 values
    tie_rows = rng.choice(n, TIES, replace=False)
    corpus[tie_rows] = corpus[tie_rows[0]]
    q = corpus[rng.choice(n, 256, replace=False)] + 0.5 * rng.standard_normal((256, d))
    q_tie = corpus[tie_rows[0]][None, :] * 1.5

    widths = ("f64", "f32", "f32_split")
    names = [(t, w) for t in ("device", "host") for w in widths]
    ix = {(t, w): nat.Index(d, 0, n, keep_f64=w == "f64", keep_f32=w == "f32", keep_f32_split=w == "f32_split",
                            f64_on_host=t == "host")
          for t, w in names}
    append_s = {}
    for key in names:
        _, append_s[f"{key[0]}_{key[1]}"] = timed(torch, lambda key=key: ix[key].append_f64(corpus))
    storage = {f"{t}_{w}": dict(zip(("device_bytes", "pinned_host_bytes"), ix[(t, w)].storage_bytes()))
               for t, w in names}
    per_row = {k: (s["device_bytes"] / n, s["pinned_host_bytes"] / n) for k, s in storage.items()}

    shapes = [(B, k) for k in (20, 1000) for B in (1, 32, 256)]
    timing, results = {}, {}
    for tier in ("device", "host"):
        for B, k in shapes:
            def call(x, B=B, k=k):
                return x.search(q[:B], k, None) if k <= nat.RBK_MAX_K_FETCH else x.search_large(q[:B], k, None)
            for _ in range(args.warmup):
                for w in widths:
                    call(ix[(tier, w)])
            ms = {w: [] for w in widths}
            for _ in range(args.steps):
                for w in widths:                           # alternated call by call: same clocks for all three
                    r = call(ix[(tier, w)])
                    ms[w].append(r[3])
                    results[(tier, w, B, k)] = r[:3]
            med = {w: float(np.median(v)) for w, v in ms.items()}
            timing[f"{tier}_B{B}_k{k}"] = {
                "f64_ms": med["f64"], "f32_ms": med["f32"], "f32_split_ms": med["f32_split"],
                "f64_over_f32": med["f64"] / med["f32"], "f32_over_split": med["f32"] / med["f32_split"],
                "bit_equal": bool(all(same(results[(tier, "f64", B, k)], results[(tier, w, B, k)]) for w in widths))}

    fallback, exact = {}, {}
    for key in names:
        x = ix[key]
        st0 = x.stats()
        r = x.search(q_tie, 20, None)
        st1 = x.stats()
        fallback[key] = {"ms": r[3], "fallback_queries": st1["fallback_queries"] - st0["fallback_queries"],
                         "result": r[:3]}
        exact[key], exact[key + ("s",)] = timed(torch, lambda x=x: x.exact_scores(q[:1]))

    t0 = time.perf_counter()
    ref = oracle_answers(oracle, corpus, np.concatenate([q[:CHECKED], q_tie]), (20, 1000))
    oracle_s = time.perf_counter() - t0
    parity = {}
    for key in names:
        ok = True
        for B, k in shapes:
            m = min(B, CHECKED)
            ok &= same(tuple(x[:m] for x in results[(key[0], key[1], B, k)]), tuple(x[:m] for x in ref[k]))
        ok &= same(fallback[key]["result"], tuple(x[CHECKED:] for x in ref[20]))
        parity[f"{key[0]}_{key[1]}"] = bool(ok)
    parity["queries"] = CHECKED + 1
    parity["oracle_seconds"] = oracle_s
    parity["fallback_widths_bit_equal"] = {t: bool(all(same(fallback[(t, "f64")]["result"], fallback[(t, w)]["result"])
                                                       for w in widths)) for t in ("device", "host")}
    parity["exact_scores_widths_bit_equal"] = {t: bool(all(exact[(t, "f64")].tobytes() == exact[(t, w)].tobytes()
                                                           for w in widths)) for t in ("device", "host")}

    # in place, on the device tier: the KEEP_F64 index through every width and back
    x = ix[("device", "f64")]
    for k in list(ix):
        if k != ("device", "f64"):
            ix.pop(k).close()                                     # room for old + new exact rows
    before = x.search(q[:32], 20, None)[:3]
    set_tier = {"flags_after": [], "storage_after": [], "answers_bit_equal": True}
    for src, dst in (("f64", "f32"), ("f32", "f32_split"), ("f32_split", "f32"), ("f32", "f64"), ("f64", "f32_split")):
        _, set_tier[f"{src}_to_{dst}_s"] = timed(torch, lambda dst=dst: x.set_tier(exact_rows=dst))
        set_tier["flags_after"].append(x.flags)
        set_tier["storage_after"].append(x.storage_bytes())
        set_tier["answers_bit_equal"] &= bool(same(before, x.search(q[:32], 20, None)[:3]))
    x.close()

    print(json.dumps({
        "metric": "f32_rows", "card": card_info(),
        "config": {"rows": n, "dim": d, "rows_kind": "N(0,1) float32, widened to float64", "steps": args.steps,
                   "warmup": args.warmup, "tie_group": TIES},
        "storage_bytes": storage, "bytes_per_row": per_row,
        "append_seconds": append_s,
        "search_device_ms": timing,
        "fallback_query": {f"{t}_{w}": {k: v for k, v in f.items() if k != "result"} for (t, w), f in fallback.items()},
        "exact_scores_one_query_s": {f"{t}_{w}": exact[(t, w, "s")] for t, w in names},
        "set_tier": set_tier,
        "parity": parity}), flush=True)


if __name__ == "__main__":
    main()
