"""Host mirror of src/knowledge/retriever/index.ts (`KnowledgeRetriever`, `createRetriever`) — the object the
CLI, the MCP server and the agent actually call — wired to the GPU path (SURVEY §8f-1 / f-2).

The reference's retriever only knows the FTS store and its `sync()` never embeds anything, so the vector
store stays empty unless something else fills it.  This variant keeps the reference surface
(`sync() -> {added, updated}`, `search(query, {typeFilter, serviceFilter, limit}) -> RetrievedKnowledge`,
`getRunbooksForService`, counts, `close`) and
  * searches through `HybridRetriever` (FTS5 + the device index + RRF) when an embedder is configured,
    through the FTS store alone otherwise (the reference behaviour);
  * in `sync()` mirrors every upserted document into the vector store: its old vectors are tombstoned
    (`deleteDocument`) and its chunks embedded and appended in one `addChunks` call; once enough slots are dead
    the vector store is compacted (`VectorStore.compact`), so repeated syncs do not grow the device index.
Loading documents from disk / Confluence / ... (src/knowledge/sources) is out of scope: `sources` are
callables returning document dicts in the reference's KnowledgeDocument shape.
"""
from __future__ import annotations

import os
from typing import Callable, Iterable, Sequence

from . import embedder as _emb
from .fts_store import KnowledgeStore
from .hybrid_search import HybridRetriever

_COMPACT_MIN_DEAD = 4096   # sync() compacts the vector store from this many tombstoned slots (and >= size() / 4)
_BUCKET = {"runbook": "runbooks", "postmortem": "postmortems", "architecture": "architecture",
           "known_issue": "knownIssues"}


def _bucket(chunks) -> dict:
    """retriever/index.ts:100-123."""
    out = {"runbooks": [], "postmortems": [], "architecture": [], "knownIssues": []}
    for c in chunks:
        if c.type in _BUCKET:
            out[_BUCKET[c.type]].append(c)
    return out


class KnowledgeRetriever:
    def __init__(self, config: dict, device: int | None = None, vector_store=None, scan_f16: bool | None = None,
                 exact_rows: str | None = None):
        """config: {storePath, sources: [callable(since) -> iterable of documents], vectorStorePath?}
        (retriever/index.ts:19-39).  scan_f16: the vector store's scan precision (see VectorStore; None:
        RUNBOOK_KNN_SCAN_F16).  exact_rows: the vector store's exact-row width (see VectorStore; None:
        RUNBOOK_KNN_EXACT_ROWS)."""
        self.config = config
        d = os.path.dirname(config["storePath"])
        if d:
            os.makedirs(d, exist_ok=True)
        self.store = KnowledgeStore(config["storePath"])
        self.initialized = False
        self._hybrid: HybridRetriever | None = None
        if _emb.is_embedder_configured() or vector_store is not None:
            self._hybrid = HybridRetriever({"storePath": config["storePath"],
                                            "vectorStorePath": config.get("vectorStorePath")
                                            or os.path.join(d or ".", "vectors.db")},
                                           fts_store=self.store, device=device, scan_f16=scan_f16,
                                           exact_rows=exact_rows)
            if vector_store is not None:       # tests inject a store built on the CPU stand-in index
                if self._hybrid.vector_store is not None:
                    self._hybrid.vector_store.close()
                self._hybrid.vector_store = vector_store

    @property
    def vector_store(self):
        return self._hybrid.vector_store if self._hybrid else None

    # ------------------------------------------------------------------ sync
    def sync(self) -> dict:
        """retriever/index.ts:44-70, plus the mirror into the vector store."""
        added = updated = 0
        for source in self.config.get("sources", []):
            since = getattr(source, "last_sync_time", None)
            for doc in source(since):
                if self.store.has_document(doc["id"]):
                    updated += 1
                else:
                    added += 1
                self.store.upsert_document(doc)
                self._mirror(doc)
        self._reclaim()
        self.initialized = True
        return {"added": added, "updated": updated}

    def _reclaim(self) -> None:
        """Every mirrored update tombstones the document's old chunks, so a long-running process would otherwise
        keep their device memory and scan time for good.  Once the dead slots reach a quarter of all slots (and at
        least _COMPACT_MIN_DEAD - below that they cost less than the call) the vector store is compacted, then
        trimmed, so the freed slots' device memory goes back too (growing again later maps memory, it copies
        nothing).  A single-GPU index and a device group are reclaimed alike; an index without `compact` is skipped."""
        vs = self.vector_store
        ix = vs._index if vs is not None else None
        if ix is None or getattr(ix, "compact", None) is None:
            return
        size = ix.size()
        dead = size - ix.count()
        if dead >= _COMPACT_MIN_DEAD and 4 * dead >= size:
            vs.compact()
            vs.trim()

    def _mirror(self, doc: dict) -> None:
        vs = self.vector_store
        if vs is None or not _emb.is_embedder_configured():
            return
        if vs.has_document(doc["id"]):
            vs.delete_document(doc["id"])          # stale chunk ids must not survive an update
        chunks = [{"chunk": {"id": ch["id"], "documentId": doc["id"], "content": ch["content"],
                             "sectionTitle": ch.get("sectionTitle")},
                   "documentTitle": doc["title"], "type": doc["type"], "services": doc.get("services", [])}
                  for ch in doc.get("chunks", [])]
        if chunks:
            vs.add_chunks(chunks)

    def ensure_initialized(self) -> None:
        """retriever/index.ts:75-80."""
        if not self.initialized and self.store.get_document_count() == 0:
            self.sync()
        self.initialized = True

    # ------------------------------------------------------------------ search
    def search(self, query: str, options: dict | None = None) -> dict:
        """retriever/index.ts:85-126: `limit || 20` chunks, bucketed by document type."""
        o = options or {}
        self.ensure_initialized()
        limit = o.get("limit") or 20
        if self._hybrid is not None and self._hybrid.has_vector_search():
            chunks = self._hybrid.search(query, {"topK": limit, "typeFilter": o.get("typeFilter"),
                                                 "serviceFilter": o.get("serviceFilter")})
        else:
            chunks = self.store.search(query, {"typeFilter": o.get("typeFilter"),
                                               "serviceFilter": o.get("serviceFilter"), "limit": limit})
        return _bucket(chunks)

    def get_runbooks_for_service(self, service_name: str) -> dict:
        """retriever/index.ts:131-136."""
        return self.search(service_name, {"typeFilter": ["runbook"], "serviceFilter": [service_name]})

    def get_document_count(self) -> int:
        return self.store.get_document_count()

    def get_document_counts_by_type(self) -> dict:
        return self.store.get_document_counts_by_type()

    def close(self) -> None:
        if self._hybrid is not None:
            self._hybrid.close()        # closes the FTS store and drops this retriever's reference on the index
        else:
            self.store.close()

    ensureInitialized, getRunbooksForService = ensure_initialized, get_runbooks_for_service
    getDocumentCount, getDocumentCountsByType = get_document_count, get_document_counts_by_type


def create_retriever(base_dir: str = ".runbook", sources: Sequence[Callable[[object], Iterable[dict]]] = (),
                     device: int | None = None) -> KnowledgeRetriever:
    """retriever/index.ts:170-191 (`${baseDir}/knowledge.db`); the vector store is `${baseDir}/vectors.db`
    (vector-store.ts:338-341), one shared device index per process."""
    return KnowledgeRetriever({"storePath": os.path.join(base_dir, "knowledge.db"),
                               "vectorStorePath": os.path.join(base_dir, "vectors.db"), "sources": list(sources)},
                              device=device)


createRetriever = create_retriever
