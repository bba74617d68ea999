"""Host mirror of src/knowledge/retriever/hybrid-search.ts (SURVEY.md §8f row f-1).

RRF and the mode dispatch stay on the host exactly as in the reference; the vector leg is
the GPU-backed VectorStore.  The FTS leg is any object with the KnowledgeStore.search
signature (sqlite.ts:125-209 is SQLite FTS5/BM25 — out of scope for the kernel work); a
minimal one is in fts_store.py.
"""
from __future__ import annotations

from dataclasses import replace
from typing import Sequence

from . import embedder as _emb
from .vector_store import RetrievedChunk, VectorStore, create_vector_store, js_or


def reciprocal_rank_fusion(fts_results: Sequence[RetrievedChunk], vector_results: Sequence[RetrievedChunk],
                           top_k: int, rrf_k: float = 60, fts_weight: float = 0.4,
                           vector_weight: float = 0.6) -> list[RetrievedChunk]:
    """hybrid-search.ts:106-151 (S12): score(id) = sum w/(k + i + 1); FTS list first."""
    scores: dict[str, list] = {}   # insertion-ordered, like the JS Map
    for results, w in ((fts_results, fts_weight), (vector_results, vector_weight)):
        for i, chunk in enumerate(results):
            rrf = w * (1 / (rrf_k + i + 1))
            ent = scores.get(chunk.id)
            if ent is not None:
                ent[1] += rrf
            else:
                scores[chunk.id] = [chunk, rrf]
    fused = list(scores.values())
    fused.sort(key=lambda e: -e[1])   # stable
    return [replace(c, score=s) for c, s in fused[:top_k]]


class HybridRetriever:
    def __init__(self, config: dict, fts_store=None, device: int | None = None, scan_f16: bool | None = None,
                 exact_rows: str | None = None):
        """hybrid-search.ts:27-42."""
        self.config = {"ftsWeight": 0.4, "vectorWeight": 0.6, "rrf_k": 60}
        self.config.update({k: v for k, v in config.items() if v is not None})
        if fts_store is None:
            from .fts_store import KnowledgeStore
            fts_store = KnowledgeStore(config["storePath"])
        self.fts_store = fts_store
        self.vector_store: VectorStore | None = None
        if _emb.is_embedder_configured():
            vector_path = config.get("vectorStorePath") or config["storePath"].replace(".db", "_vectors.db", 1)
            self.vector_store = create_vector_store(vector_path.replace("/vectors.db", "", 1), device,
                                                    scan_f16=scan_f16, exact_rows=exact_rows)  # :39-40 quirk

    def has_vector_search(self) -> bool:
        return self.vector_store is not None and _emb.is_embedder_configured()   # :47-49

    def search(self, query: str, options: dict | None = None, **kw) -> list[RetrievedChunk]:
        """hybrid-search.ts:54-100."""
        o = dict(options or {})
        o.update(kw)
        top_k = js_or(o.get("topK"), 10)
        mode = o.get("mode") or ("hybrid" if self.has_vector_search() else "fts")
        tf, sf = o.get("typeFilter"), o.get("serviceFilter")
        if mode == "fts" or not self.has_vector_search():
            return self.fts_store.search(query, {"typeFilter": tf, "serviceFilter": sf, "limit": top_k})
        if mode == "vector" and self.vector_store:
            return self.vector_store.search(query, {"topK": top_k, "typeFilter": tf, "serviceFilter": sf})
        fts = self.fts_store.search(query, {"typeFilter": tf, "serviceFilter": sf, "limit": top_k * 2})
        vec = self.vector_store.search(query, {"topK": top_k * 2, "typeFilter": tf, "serviceFilter": sf})
        return reciprocal_rank_fusion(fts, vec, top_k, self.config["rrf_k"], self.config["ftsWeight"],
                                      self.config["vectorWeight"])

    def search_by_type(self, query: str, options: dict | None = None) -> dict:
        """hybrid-search.ts:156-193."""
        o = options or {}
        results = self.search(query, {"topK": o.get("topK") or 20, "serviceFilter": o.get("serviceFilter")})
        out = {"runbooks": [], "postmortems": [], "architecture": [], "knownIssues": []}
        key = {"runbook": "runbooks", "postmortem": "postmortems", "architecture": "architecture",
               "known_issue": "knownIssues"}
        for c in results:
            if c.type in key:
                out[key[c.type]].append(c)
        return out

    def get_runbooks_for_service(self, service_name: str):
        return self.search(f"runbook for {service_name}",
                           {"topK": 5, "typeFilter": ["runbook"], "serviceFilter": [service_name]})

    def find_similar_incidents(self, description: str):
        return self.search(description, {"topK": 5, "typeFilter": ["postmortem", "known_issue"]})

    def get_architecture_context(self, services: Sequence[str]):
        return self.search(f"architecture dependencies {' '.join(services)}",
                           {"topK": 5, "typeFilter": ["architecture"], "serviceFilter": list(services)})

    def close(self) -> None:
        self.fts_store.close()
        if self.vector_store:
            self.vector_store.close()

    hasVectorSearch, searchByType = has_vector_search, search_by_type
    getRunbooksForService, findSimilarIncidents = get_runbooks_for_service, find_similar_incidents
    getArchitectureContext = get_architecture_context


def create_hybrid_retriever(base_dir: str = ".runbook", **kw) -> HybridRetriever:
    """hybrid-search.ts:240-245."""
    return HybridRetriever({"storePath": f"{base_dir}/knowledge.db", "vectorStorePath": f"{base_dir}/vectors.db"}, **kw)


createHybridRetriever = create_hybrid_retriever
