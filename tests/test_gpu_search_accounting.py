"""GPU suite (-m gpu): the exact per-call change of every rbk_stats counter, for each search path of one index.

The counters say what a call did on the device: searches and queries answered, scan and kernel launches, scans
timed, graph replays, wide retries and exhaustive fallbacks.  Each case below makes one call and compares the
counters' change (and the last_* values after it) with the values the engine has always produced.  That includes the
call that first captures the small-batch graph, whose scan counts twice: once while it is captured, once when it
is replayed.

`python tests/test_gpu_search_accounting.py` prints the measured table as JSON."""
import json
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

COUNTERS = ("searches", "queries", "fallback_queries", "scan_launches", "kernel_launches", "retry_batches",
            "scans_timed", "graph_replays")
LAST = ("last_kprime", "last_ring_stages")

# (counter deltas in COUNTERS order, then LAST values) per case
EXPECTED = {
    "graph_capture":         [1, 4, 0, 2, 6, 0, 0, 1, 32, 4],
    "graph_replay":          [1, 4, 0, 1, 3, 0, 0, 1, 32, 4],
    "graph_f64_capture":     [1, 4, 0, 2, 6, 0, 0, 1, 32, 4],
    "graph_then_retry":      [2, 2, 0, 4, 12, 1, 2, 1, 128, 4],
    "general_1_sub_batch":   [1, 200, 0, 1, 3, 0, 1, 0, 48, 4],
    "general_2_sub_batches": [1, 1098, 1, 4, 12, 1, 4, 0, 128, 4],
    "search_device":         [1, 33, 0, 1, 3, 0, 1, 0, 48, 4],
    "search_device_async":   [1, 33, 0, 1, 3, 0, 1, 0, 48, 4],
    "retry":                 [1, 200, 0, 2, 6, 1, 2, 0, 128, 4],
    "retry_and_fallback":    [1, 200, 1, 2, 8, 1, 2, 0, 128, 4],
    "large_1_sub_batch":     [1, 8, 0, 2, 6, 0, 2, 0, 500, 4],
    "large_2_sub_batches":   [1, 1098, 0, 4, 11, 0, 4, 0, 200, 4],
    "debug_scores":          [0, 0, 0, 1, 2, 0, 1, 0, 32, 4],
    "empty_small":           [1, 4, 0, 0, 1, 0, 0, 0, 32, 0],
    "empty_general":         [1, 200, 0, 0, 1, 0, 0, 0, 48, 0],
    "empty_large":           [1, 8, 0, 0, 1, 0, 0, 0, 500, 0],
}


def _measure():
    import torch
    from runbookai_b200 import Index, synth

    n, d = 20_000, 128
    corpus = synth.random_corpus(n, d, 31)
    q = synth.random_queries(1100, d, 32)
    rng = np.random.default_rng(33)
    dup = rng.choice(n, 270, replace=False)
    corpus[dup[:200]] = synth.f32_to_bf16_bits(q[0] * 0.5)    # 200 exact ties > 128 candidates: retry, then fallback
    corpus[dup[200:]] = synth.f32_to_bf16_bits(q[1] * 0.25)   # 70 exact ties: the wide retry proves them
    plain = q[2:]

    def snap(ix):
        torch.cuda.synchronize()   # every timed scan has finished: stats() folds them all in
        return ix.stats()

    out = {}

    def case(name, ix, call):
        a = snap(ix)
        call()
        b = snap(ix)
        out[name] = [b[c] - a[c] for c in COUNTERS] + [b[c] for c in LAST]

    def device_call(ix, B, k, asynchronous):
        qd = torch.from_numpy(np.ascontiguousarray(plain[:B])).cuda()
        s = torch.empty((B, k), dtype=torch.int64, device="cuda")
        v = torch.empty((B, k), dtype=torch.float64, device="cuda")
        c = torch.empty(B, dtype=torch.int32, device="cuda")
        f = torch.empty(B, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        if asynchronous:
            return lambda: ix.search_device_async(qd.data_ptr(), B, k, None, s.data_ptr(), v.data_ptr(),
                                                  c.data_ptr(), f.data_ptr())
        return lambda: ix.search_device(qd.data_ptr(), B, k, None, s.data_ptr(), v.data_ptr(), c.data_ptr())

    with Index(d) as ix:
        ix.append_bf16(corpus)
        case("graph_capture", ix, lambda: ix.search(plain[:4], 10, 0.5))
        case("graph_replay", ix, lambda: ix.search(plain[:4], 10, 0.5))
        case("graph_f64_capture", ix, lambda: ix.search(plain[:4].astype(np.float64), 10, None))
        case("graph_then_retry", ix, lambda: ix.search(q[1:2], 20, None))
        case("general_1_sub_batch", ix, lambda: ix.search(plain[:200], 20, None))
        # 1098 queries: two sub-batches, and one random query meets the 200 tied rows near its 20th hit
        case("general_2_sub_batches", ix, lambda: ix.search(plain[:1098], 20, None))
        case("search_device", ix, device_call(ix, 33, 20, False))
        case("search_device_async", ix, device_call(ix, 33, 20, True))
        case("retry", ix, lambda: ix.search(np.concatenate([q[1:2], plain[:199]]), 20, None))
        case("retry_and_fallback", ix, lambda: ix.search(np.concatenate([q[0:2], plain[:198]]), 20, 0.5))
        case("large_1_sub_batch", ix, lambda: ix.search_large(plain[:8].astype(np.float64), 500, None))
        case("large_2_sub_batches", ix, lambda: ix.search_large(plain[:1098].astype(np.float64), 200, None))
        case("debug_scores", ix, lambda: ix.debug_scores(plain[:3]))
    with Index(d) as ix:
        case("empty_small", ix, lambda: ix.search(plain[:4], 10, 0.5))
        case("empty_general", ix, lambda: ix.search(plain[:200], 20, None))
        case("empty_large", ix, lambda: ix.search_large(plain[:8].astype(np.float64), 500, None))
    return out


def test_search_accounting(native):
    import torch
    assert torch.cuda.is_available(), "run -m gpu on a GPU box"
    got = _measure()
    assert got == EXPECTED


if __name__ == "__main__":
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    print(json.dumps(_measure()))
