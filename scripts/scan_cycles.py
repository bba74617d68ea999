#!/usr/bin/env python
"""Where a tile's cycles go in the fused scan: the RBK_SCAN_CYCLE_STATS probe at bench.py's shapes.

    python scripts/scan_cycles.py --out DIR [--workloads cfg3,cfg5] [--launches 5]

Builds the library with -DRBK_SCAN_CYCLE_STATS into a temporary copy of the package (the tree's own library is never
replaced), then, per workload, generates bench.py's corpus and queries in a child process and runs one warm-up search
and `--launches` searches.  After each search it reads (and clears) the probe's sums with `rbk_scan_cycle_stats`, and
writes DIR/scan_cycles.json: per workload and launch the raw sums of each wgmma warpgroup, and the median over the
launches of each bucket per (tile, warpgroup), in SM cycles.  `unit` is the whole main loop (full + mma + handoff +
tile_end; pace and refill are parts of handoff).  `fetch` is per blocked `full` wait, not per tile: the cycles from
the slot's TMA issue to the wait's return, with `fetch_waits` such waits per tile.  Each launch also carries the probe kernel's time (CUDA events, `last_scan_ms`) and the SM clock the
two imply (`unit` cycles per CTA over that time): compare that time with bench.py's `kernel_ms` of the default build
to see how far the probe's clock reads moved the kernel.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import shutil
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
BUCKETS = ("full", "mma", "handoff", "pace", "refill", "tile_end", "fetch")
LAPS = ("full", "mma", "handoff", "tile_end")      # contiguous: they sum to the main loop
FIELDS = BUCKETS + ("tiles", "units", "fetch_waits", "refills")


def build_probe(pkg_dir: Path) -> Path:
    """A copy of the package's Python files with a probe build of the library next to them."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("rbk_build", ROOT / "runbookai_b200" / "build.py")
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    dst = pkg_dir / "runbookai_b200"
    (dst / "lib").mkdir(parents=True)
    for f in (ROOT / "runbookai_b200").glob("*.py"):
        shutil.copy2(f, dst / f.name)
    lib = dst / "lib" / "librbk_knn.so"
    cmd = [build._nvcc(), "-DRBK_SCAN_CYCLE_STATS", *build.NVCC_FLAGS,
           *[str(build.CSRC / s) for s in build.SOURCES], "-o", str(lib)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise SystemExit("nvcc failed:\n" + res.stdout + res.stderr)
    return lib


def read_sums(lib) -> dict:
    """{mode: {"wg1": {field: sum}, "wg2": ...}} for the modes that ran since the last read."""
    n = 3 * 2 * len(FIELDS)
    buf = (ctypes.c_ulonglong * n)()
    if lib.rbk_scan_cycle_stats(buf) != n:
        raise SystemExit("rbk_scan_cycle_stats failed")
    out = {}
    for mode in range(3):
        recs = {}
        for wg in range(2):
            base = (mode * 2 + wg) * len(FIELDS)
            recs[f"wg{wg + 1}"] = dict(zip(FIELDS, buf[base:base + len(FIELDS)]))
        if recs["wg1"]["tiles"]:
            out[mode] = recs
    return out


def child(pkg_root: str, workload: str, launches: int) -> None:
    sys.path.insert(0, pkg_root)            # the probe build, ahead of the tree's package
    import runbookai_b200                   # noqa: F401
    from runbookai_b200 import _native, Index
    sys.path.insert(1, str(ROOT))
    import bench
    import torch
    lib = _native.lib
    lib.rbk_scan_cycle_stats.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)]
    lib.rbk_scan_cycle_stats.restype = ctypes.c_int
    n, d, B, k, _ = bench.WORKLOADS[workload]
    q = bench.load_synth().random_queries(B, d, bench.SEED + 1)
    recs = []
    with Index(d, device=0, capacity_hint=n) as ix:
        bench.gen_shard(ix, 0, n, d, torch.device("cuda", 0))
        ix.search(q, 2 * k, None)           # warm-up
        read_sums(lib)
        for _ in range(launches):
            s0 = ix.stats()["scans_timed"]
            ix.search(q, 2 * k, None)
            st = ix.stats()
            for mode, r in read_sums(lib).items():
                recs.append({"mode": mode, "n_ks": -(-d // 64), "scans": int(st["scans_timed"] - s0),
                             "last_scan_ms": float(st["last_scan_ms"]), **r})
    print(json.dumps(recs), flush=True)


def per_tile(rec: dict) -> dict:
    """Cycles per (tile, warpgroup), both warpgroups averaged, and each warpgroup's own where they differ by role."""
    w1, w2 = rec["wg1"], rec["wg2"]
    tiles = w1["tiles"] + w2["tiles"]
    res = {b: (w1[b] + w2[b]) / tiles for b in LAPS}
    res["unit"] = sum(res[b] for b in LAPS)
    for name, w in (("wg1", w1), ("wg2", w2)):
        for b in ("full", "handoff", "pace", "refill"):
            res[f"{b}_{name}"] = w[b] / w["tiles"]
        res[f"refills_{name}"] = w["refills"] / w["tiles"]
        res[f"fetch_waits_{name}"] = w["fetch_waits"] / w["tiles"]
    waits = w1["fetch_waits"] + w2["fetch_waits"]
    res["fetch_per_blocked_wait"] = (w1["fetch"] + w2["fetch"]) / waits if waits else 0.0
    # the SM clock that this many cycles per CTA in the probe kernel's event time implies
    unit_per_cta = sum(w1[b] + w2[b] for b in LAPS) / (w1["units"] + w2["units"])
    res["implied_sm_mhz"] = unit_per_cta / (rec["last_scan_ms"] * 1e3)
    res["scan_ms"] = rec["last_scan_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for scan_cycles.json")
    ap.add_argument("--workloads", default="cfg3,cfg5")
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--child", nargs=3, metavar=("PKG_ROOT", "WORKLOAD", "LAUNCHES"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.child[0], args.child[1], int(args.child[2]))
        return
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                           "-i", "0"], capture_output=True, text=True).stdout.strip()
    result = {"card": card, "workloads": {}}
    with tempfile.TemporaryDirectory(prefix="rbk_scan_cycles_") as tmp:
        build_probe(Path(tmp))
        for wl in args.workloads.split(","):
            res = subprocess.run([sys.executable, __file__, "--out", args.out, "--child", tmp, wl,
                                  str(args.launches)], capture_output=True, text=True)
            if res.returncode != 0:
                raise SystemExit(f"{wl}: the probe run failed\n{res.stdout[-4000:]}\n{res.stderr[-4000:]}")
            recs = json.loads(res.stdout.strip().splitlines()[-1])
            # top-k' launches of a single scan per search (a search that rescans has no single kernel time)
            tiles = [per_tile(r) for r in recs if r["mode"] == 0 and r["scans"] == 1]
            med = {b: statistics.median(t[b] for t in tiles) for b in tiles[0]} if tiles else None
            result["workloads"][wl] = {"launches": recs, "per_tile_median": med}
            print(json.dumps({"workload": wl, "card": card, "n_ks": recs[0]["n_ks"] if recs else None,
                              "per_tile_median": med}), flush=True)
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "scan_cycles.json").write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
