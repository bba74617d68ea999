"""K3 ingest throughput: convert_rows_kernel (f64 -> bf16, bf16 copy) and row_norms_kernel at BASELINE scale,
device-resident sources (the PCIe hop is not the kernel).  Prints one JSON line per case with CUDA-event times;
use torch.profiler for the per-kernel launch list.

    python scripts/ingest_bench.py [rows] [dim]
"""
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from runbookai_b200 import Index  # noqa: E402

PEAK = 3350.0   # GB/s, HBM3 bandwidth in NVIDIA's H100 SXM data sheet


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 4_000_000
    d = int(sys.argv[2]) if len(sys.argv) > 2 else 768
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(dev)
    torch.cuda.set_stream(st)
    for kind in ("f64", "bf16"):
        src = torch.randn(n, d, device=dev, dtype=torch.float32)
        src = src.to(torch.float64) if kind == "f64" else src.to(torch.bfloat16)
        for rep in range(3):
            ix = Index(d, device=0, capacity_hint=n)
            ix.set_stream(st.cuda_stream)
            fn = ix.append_f64_device if kind == "f64" else ix.append_bf16_device
            ms = timed(lambda: fn(src.data_ptr(), n))
            ix.close()
        elem = 8 if kind == "f64" else 2
        # convert: read elem*N*d, write 2*N*d; norms: read 2*N*d (+ 12 bytes/row out)
        bytes_ = (elem + 2 + 2) * n * d + 12 * n
        print(json.dumps({"case": f"append_{kind}_device", "rows": n, "dim": d, "ms": ms,
                          "algorithmic_bytes": bytes_, "gbs": bytes_ / ms / 1e6, "frac_of_hbm_peak": bytes_ / ms / 1e6 / PEAK}),
              flush=True)
        del src


if __name__ == "__main__":
    main()
