"""Query micro-batcher (SURVEY.md §8f-3).

The reference issues knowledge queries one at a time (`InvestigationOrchestrator` awaits each
`search_knowledge` call in turn, src/agent/investigation-orchestrator.ts:975-997; the agent's
`ParallelToolExecutor` runs at most 5 tool calls concurrently, src/agent/parallel-executor.ts:32-35).
One GPU pass over the corpus costs the same for 1 query as for 128, so concurrent callers
(several investigations in one process, the Slack gateway, hypothesis branches) should share a
pass: this class coalesces `search()` calls that arrive within a short window into ONE
device call, and hands every caller exactly what its own `search()` would have returned.  On an
index with `search_each` that call is ONE search at every caller's own k_fetch = 2*topK and minScore,
large callers included (a caller whose 2*topK is not an integer in [1, 4096] still goes through
`VectorStore.search` alone: its own error, or a result that would make every row of the shared one
that wide); on any other index object the shared pass fetches for the most demanding
caller at the lowest minScore and each caller's own cut is re-applied on the host, while callers
whose 2*topK exceeds the scan's candidate lists take `VectorStore.search` on their own.

    batcher = MicroBatcher(store, window_ms=2.0, max_batch=256)
    fut = batcher.submit("redis pool exhausted", {"topK": 5})     # concurrent.futures.Future
    chunks = batcher.search("redis pool exhausted", {"topK": 5})  # blocking convenience
"""
from __future__ import annotations

import queue
import threading
import time
from concurrent.futures import Future

import numpy as np

from . import embedder as _emb
from ._native import RBK_EDIM, RBK_MAX_K_FETCH, RBK_MAX_K_FETCH_LARGE, DimensionError
from .vector_store import NOT_CONFIGURED, VectorStore, js_or


def _shareable(k_fetch) -> bool:
    """A k_fetch one search_each call can carry for everybody: an integer in [1, RBK_MAX_K_FETCH_LARGE]."""
    return isinstance(k_fetch, (int, np.integer)) and not isinstance(k_fetch, bool) and \
        1 <= k_fetch <= RBK_MAX_K_FETCH_LARGE


class MicroBatcher:
    def __init__(self, store: VectorStore, window_ms: float = 2.0, max_batch: int = 256):
        self.store = store
        self.window = window_ms / 1000.0
        self.max_batch = max_batch
        self._q: queue.Queue = queue.Queue()
        self._stop = threading.Event()
        self._close_lock = threading.Lock()
        self.batches = 0          # device passes issued
        self.served = 0           # queries answered
        self._thread = threading.Thread(target=self._run, name="rbk-microbatcher", daemon=True)
        self._thread.start()

    # ------------------------------------------------------------------ public
    def submit(self, query: str, options: dict | None = None) -> Future:
        fut: Future = Future()
        with self._close_lock:
            if self._stop.is_set():
                raise RuntimeError("batcher closed")
            self._q.put((query, dict(options or {}), fut))
        return fut

    def search(self, query: str, options: dict | None = None):
        return self.submit(query, options).result()

    def close(self) -> None:
        """Stop the worker.  Requests still queued are failed with `batcher closed` (nobody is left waiting for a
        result that will never come); submit() after close raises."""
        with self._close_lock:
            self._stop.set()
            self._q.put(None)
        self._thread.join(timeout=5)
        while True:
            try:
                item = self._q.get_nowait()
            except queue.Empty:
                break
            if item is not None and not item[2].done():
                item[2].set_exception(RuntimeError("batcher closed"))

    # ------------------------------------------------------------------ worker
    def _run(self) -> None:
        while not self._stop.is_set():
            item = self._q.get()
            if item is None:
                continue
            batch = [item]
            deadline = time.monotonic() + self.window
            while len(batch) < self.max_batch:
                left = deadline - time.monotonic()
                if left <= 0:
                    break
                try:
                    nxt = self._q.get(timeout=left)
                except queue.Empty:
                    break
                if nxt is None:
                    break
                batch.append(nxt)
            self._serve(batch)

    def _serve(self, batch) -> None:
        try:
            if not _emb.is_embedder_configured():
                raise RuntimeError(NOT_CONFIGURED)
            st = self.store
            if getattr(st._index, "search_each", None) is not None:
                alone = [b for b in batch if not _shareable(2 * js_or(b[1].get("topK"), b[1].get("top_k"), 10))]
                for q_, o_, f_ in alone:
                    try:
                        f_.set_result(st.search(q_, o_))
                    except Exception as exc:
                        f_.set_exception(exc)
                    self.served += 1
                batch = [b for b in batch if b not in alone]
                if batch:
                    self._serve_each(batch)
                return
            # callers that want more than the scan's candidate lists hold (topK > 56) take the large-k path of
            # VectorStore.search on their own; everybody else shares one device pass
            big = [b for b in batch if 2 * js_or(b[1].get("topK"), b[1].get("top_k"), 10) > RBK_MAX_K_FETCH]
            for q_, o_, f_ in big:
                try:
                    f_.set_result(st.search(q_, o_))
                except Exception as exc:
                    f_.set_exception(exc)
                self.served += 1
            batch = [b for b in batch if b not in big]
            if not batch:
                return
            qvec = np.asarray(_emb.embed_texts([b[0] for b in batch]), dtype=np.float64)
            # one device pass: fetch enough for the most demanding caller, strictest-common threshold = the
            # LOWEST minScore; each caller's own cut and threshold are re-applied below (S4, S5, S7)
            top_ks = [js_or(o.get("topK"), o.get("top_k"), 10) for _, o, _ in batch]
            mins = [js_or(o.get("minScore"), o.get("min_score"), 0.5) for _, o, _ in batch]
            k_fetch = 2 * max(top_ks)
            with st._st.lock:   # state checks, scan and slot -> id lookup against the same table (the index may be shared)
                if st._index is None or not st._ids:
                    for _, _, f in batch:
                        f.set_result([])
                    return
                if st._ragged or qvec.shape[1] != st._index.dim:
                    raise DimensionError(RBK_EDIM, "Vectors must have the same length")
                slots, scores, counts, _ = st._index.search(qvec, k_fetch, min(mins))
                picked = []
                for i in range(len(batch)):
                    n = int(counts[i])
                    keep = scores[i, :n] >= mins[i]                  # this caller's `>= minScore`
                    s_i, v_i = slots[i, :n][keep][: 2 * top_ks[i]], scores[i, :n][keep][: 2 * top_ks[i]]
                    picked.append(([st._ids[int(s)] for s in s_i], v_i))
            self.batches += 1
            for i, (_, o, fut) in enumerate(batch):
                ids_i, v_i = picked[i]
                fut.set_result(st._hydrate(ids_i, v_i, top_ks[i], o.get("typeFilter") or o.get("type_filter"),
                                           o.get("serviceFilter") or o.get("service_filter")))
                self.served += 1
        except Exception as exc:  # every waiter gets the error its own search() would have raised
            for _, _, f in batch:
                if not f.done():
                    f.set_exception(exc)

    def _serve_each(self, batch) -> None:
        """The whole window in one index.search_each: caller i at its own k_fetch = 2*topK and minScore, so its row is
        exactly its own search()'s device answer (vector-store.ts:207-221) and only the hydration is left."""
        st = self.store
        qvec = np.asarray(_emb.embed_texts([b[0] for b in batch]), dtype=np.float64)
        top_ks = [js_or(o.get("topK"), o.get("top_k"), 10) for _, o, _ in batch]
        mins = [js_or(o.get("minScore"), o.get("min_score"), 0.5) for _, o, _ in batch]
        with st._st.lock:   # state checks, scan and slot -> id lookup against the same table (the index may be shared)
            if st._index is None or not st._ids:
                for _, _, f in batch:
                    f.set_result([])
                return
            if st._ragged or qvec.shape[1] != st._index.dim:
                raise DimensionError(RBK_EDIM, "Vectors must have the same length")
            slots, scores, counts, _ = st._index.search_each(qvec, [2 * k for k in top_ks], mins)
            picked = [([st._ids[int(s)] for s in slots[i, :counts[i]]], scores[i, :counts[i]]) for i in range(len(batch))]
        self.batches += 1
        for i, (_, o, fut) in enumerate(batch):
            ids_i, v_i = picked[i]
            fut.set_result(st._hydrate(ids_i, v_i, top_ks[i], o.get("typeFilter") or o.get("type_filter"),
                                       o.get("serviceFilter") or o.get("service_filter")))
            self.served += 1
