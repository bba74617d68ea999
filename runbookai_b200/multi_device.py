"""One corpus over several GPUs from ONE host process (SURVEY §8e, the deployment RunbookAI itself would
use: a single Node process, no torchrun).

`MultiDeviceIndex` has the `_native.Index` surface, so it drops into `VectorStore(index_factory=...)`:
one `rbk_index` per device, rows dealt out block-cyclically (global slot s lives on device
(s // block) % G), every search fanned out to all devices on host threads (the C ABI call releases the
GIL; each index runs on its own stream) and the G exact per-device lists merged on the host by
(score desc, global slot asc).  Block-cyclic instead of contiguous blocks because this index GROWS
(`addChunks` at sync time): no device needs to know the final corpus size, and load stays balanced.
Within a device local order == global order, so every per-device list is already in the reference's
tie-break order and the merge is an ordinary k-way merge of exact results - nothing is approximated.

The one-process-per-GPU path (`sharded.py`, NCCL all-gather + merge kernel) is what `bench.py` measures;
this module is host glue over the same C ABI calls.
"""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor
from typing import Callable, Sequence

import numpy as np

from ._native import RBK_EDIM, DimensionError, Index


class MultiDeviceIndex:
    def __init__(self, dim: int, devices: Sequence[int], capacity_hint: int = 0, keep_f64: bool = False,
                 block: int = 4096, index_factory: Callable | None = None, keep_f32: bool = False,
                 keep_f32_split: bool = False):
        if not devices:
            raise ValueError("devices must name at least one GPU")
        make = index_factory or (lambda d, dev: Index(d, device=dev, capacity_hint=-(-capacity_hint // len(devices)),
                                                      keep_f64=keep_f64, keep_f32=keep_f32,
                                                      keep_f32_split=keep_f32_split))
        self.dim = dim
        self.devices = list(devices)
        self.block = int(block)
        self.parts = [make(dim, dev) for dev in self.devices]
        self._n = 0                                   # global slots handed out
        self._pool = ThreadPoolExecutor(max_workers=len(self.parts), thread_name_prefix="rbk-dev")

    # ------------------------------------------------------------------ slot arithmetic
    def _locate(self, slots: np.ndarray):
        """global slot -> (device index, local slot)."""
        s = np.asarray(slots, dtype=np.int64)
        blk = s // self.block
        G = len(self.parts)
        return blk % G, (blk // G) * self.block + s % self.block

    def _global(self, g: int, local: np.ndarray) -> np.ndarray:
        """local slot on device g -> global slot (-1 stays -1)."""
        l = np.asarray(local, dtype=np.int64)
        out = ((l // self.block) * len(self.parts) + g) * self.block + l % self.block
        return np.where(l < 0, -1, out)

    # ------------------------------------------------------------------ mutation
    def _append(self, rows: np.ndarray, how: str) -> int:
        if rows.ndim != 2 or rows.shape[1] != self.dim:
            raise DimensionError(RBK_EDIM, "Vectors must have the same length")
        first = self._n
        i = 0
        while i < rows.shape[0]:                      # one call per run of rows that share a block
            s = self._n
            take = min(self.block - s % self.block, rows.shape[0] - i)
            g = (s // self.block) % len(self.parts)
            local = getattr(self.parts[g], how)(rows[i:i + take])
            assert local == self._locate(np.array([s]))[1][0], "device index out of step with the slot map"
            self._n += take
            i += take
        return first

    def append_f64(self, rows) -> int:
        return self._append(np.ascontiguousarray(rows, dtype=np.float64).reshape(-1, self.dim), "append_f64")

    def append_f32(self, rows) -> int:
        return self._append(np.ascontiguousarray(rows, dtype=np.float32).reshape(-1, self.dim), "append_f32")

    def append_bf16(self, rows_u16) -> int:
        return self._append(np.ascontiguousarray(rows_u16, dtype=np.uint16).reshape(-1, self.dim), "append_bf16")

    def overwrite_f64(self, slot: int, row) -> None:
        g, l = self._locate(np.array([slot]))
        self.parts[int(g[0])].overwrite_f64(int(l[0]), row)

    def tombstone(self, slots) -> None:
        s = np.asarray(slots, dtype=np.int64)
        g, l = self._locate(s)
        for d in range(len(self.parts)):
            m = g == d
            if m.any():
                self.parts[d].tombstone(l[m])

    def clear(self) -> None:
        for p in self.parts:
            p.clear()
        self._n = 0

    def count(self) -> int:
        return sum(p.count() for p in self.parts)

    def size(self) -> int:
        return self._n

    def close(self) -> None:
        for p in self.parts:
            p.close()
        self._pool.shutdown(wait=False)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ------------------------------------------------------------------ search
    def search(self, queries, k_fetch: int, min_score: float | None = 0.5):
        """Same contract as Index.search: (global slots [B,k], fp64 scores [B,k], counts [B], device_ms = max)."""
        q = np.asarray(queries)
        if q.ndim == 1:
            q = q[None, :]
        if q.shape[1] != self.dim:
            raise DimensionError(RBK_EDIM, "Vectors must have the same length")
        # any k: every device answers on the GPU (Index.search_any_k: the scan, the large-k or the unbounded search)
        res = list(self._pool.map(lambda p: getattr(p, "search_any_k", p.search)(q, k_fetch, min_score), self.parts))
        B, G = q.shape[0], len(self.parts)
        slots = np.concatenate([self._global(g, r[0]) for g, r in enumerate(res)], axis=1)      # [B, G*k]
        scores = np.concatenate([r[1] for r in res], axis=1)
        valid = slots >= 0
        # (score desc, slot asc); unused entries (slot -1, score NaN) sort last
        key_score = np.where(valid, -scores, np.inf)
        key_slot = np.where(valid, slots, np.iinfo(np.int64).max)
        order = np.lexsort((key_slot, key_score), axis=1)[:, :k_fetch]
        out_s = np.take_along_axis(slots, order, axis=1)
        out_v = np.take_along_axis(scores, order, axis=1)
        counts = np.minimum(valid.sum(axis=1), k_fetch).astype(np.int32)
        tail = np.arange(k_fetch)[None, :] >= counts[:, None]
        out_s[tail] = -1
        out_v[tail] = np.nan
        return out_s, out_v, counts, max(r[3] for r in res)

    search_any_k = search

    def stats(self) -> dict:
        per = [p.stats() for p in self.parts]
        out = {k: sum(s[k] for s in per) for k in ("searches", "queries", "fallback_queries", "scan_launches",
                                                   "kernel_launches", "retry_batches") if k in per[0]}
        out["devices"] = len(per)
        return out
