"""Scan-kernel time for one query block (B <= 128) over 1M x 768 rows: how close do the HBM-bound small batches get to
the HBM bandwidth (3350 GB/s, NVIDIA's H100 SXM data sheet)?"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from runbookai_b200 import Index, synth  # noqa: E402

n, d, k = 1_000_000, 768, 32
dev = torch.device("cuda", 0)
ix = Index(d, capacity_hint=n)
g = torch.Generator(device=dev).manual_seed(7)
for r0 in range(0, n, 1 << 18):
    m = min(1 << 18, n - r0)
    t = torch.randn(m, d, device=dev, generator=g).to(torch.bfloat16)
    torch.cuda.synchronize()
    ix.append_bf16_device(t.data_ptr(), m)
for b in (1, 8, 64, 128):
    q = torch.from_numpy(synth.random_queries(b, d, 8)).to(dev)
    os_ = torch.empty((b, k), dtype=torch.int64, device=dev)
    ov = torch.empty((b, k), dtype=torch.float64, device=dev)
    oc = torch.empty((b,), dtype=torch.int32, device=dev)
    res = []
    for _ in range(12):
        ix.search_device(q.data_ptr(), b, k, None, os_.data_ptr(), ov.data_ptr(), oc.data_ptr())
        res.append(ix.stats()["last_scan_ms"])
    best = min(res[2:])
    print(json.dumps({"B": b, "rows": n, "scan_ms_min": round(best, 4), "scan_ms_med": round(float(np.median(res[2:])), 4),
                      "gbs": round(2.0 * n * d / best / 1e6), "frac_of_hbm_peak": round(2.0 * n * d / best / 1e6 / 3350.0, 3)}), flush=True)
ix.close()
