"""Minimal host mirror of the FTS leg used by HybridRetriever: KnowledgeStore.search
(src/knowledge/store/sqlite.ts:125-209) and upsertDocument (:76-120), same SQLite schema
(:20-68), FTS5/BM25 inside SQLite.  Out of the kernel scope (SURVEY.md §2): it exists so
the hybrid path (SURVEY §8f-1) can be exercised end to end; nothing here touches the GPU.
"""
from __future__ import annotations

import json
import re
import sqlite3

from .vector_store import RetrievedChunk, js_or

SCHEMA = """
      CREATE TABLE IF NOT EXISTS documents (
        id TEXT PRIMARY KEY, type TEXT NOT NULL, title TEXT NOT NULL, content TEXT NOT NULL,
        services TEXT, tags TEXT, symptoms TEXT, severity_relevance TEXT, source_url TEXT,
        author TEXT, created_at TEXT, updated_at TEXT, last_validated TEXT
      );
      CREATE TABLE IF NOT EXISTS chunks (
        id TEXT PRIMARY KEY, document_id TEXT NOT NULL, content TEXT NOT NULL, section_title TEXT,
        chunk_type TEXT, line_start INTEGER, line_end INTEGER,
        FOREIGN KEY (document_id) REFERENCES documents(id)
      );
      CREATE INDEX IF NOT EXISTS idx_documents_type ON documents(type);
      CREATE INDEX IF NOT EXISTS idx_documents_services ON documents(services);
      CREATE INDEX IF NOT EXISTS idx_chunks_document_id ON chunks(document_id);
      CREATE VIRTUAL TABLE IF NOT EXISTS chunks_fts USING fts5(
        content, section_title, content='chunks', content_rowid='rowid'
      );
      CREATE TRIGGER IF NOT EXISTS chunks_ai AFTER INSERT ON chunks BEGIN
        INSERT INTO chunks_fts(rowid, content, section_title) VALUES (NEW.rowid, NEW.content, NEW.section_title);
      END;
      CREATE TRIGGER IF NOT EXISTS chunks_ad AFTER DELETE ON chunks BEGIN
        INSERT INTO chunks_fts(chunks_fts, rowid, content, section_title)
        VALUES('delete', OLD.rowid, OLD.content, OLD.section_title);
      END;
"""


class KnowledgeStore:
    def __init__(self, db_path: str):
        self.db = sqlite3.connect(db_path)
        self.db.row_factory = sqlite3.Row
        self.db.executescript(SCHEMA)

    def upsert_document(self, doc: dict) -> None:
        """sqlite.ts:76-120."""
        with self.db:
            self.db.execute(
                "INSERT OR REPLACE INTO documents (id, type, title, content, services, tags, symptoms, "
                "severity_relevance, source_url, author, created_at, updated_at, last_validated) "
                "VALUES (?, ?, ?, ?, ?, ?, ?, ?, ?, ?, ?, ?, ?)",
                (doc["id"], doc["type"], doc["title"], doc.get("content", ""), json.dumps(doc.get("services", [])),
                 json.dumps(doc.get("tags", [])), json.dumps(doc.get("symptoms") or []),
                 json.dumps(doc.get("severityRelevance", [])), doc.get("sourceUrl"), doc.get("author"),
                 doc.get("createdAt"), doc.get("updatedAt"), doc.get("lastValidated")))
            self.db.execute("DELETE FROM chunks WHERE document_id = ?", (doc["id"],))
            for ch in doc.get("chunks", []):
                self.db.execute(
                    "INSERT INTO chunks (id, document_id, content, section_title, chunk_type, line_start, line_end) "
                    "VALUES (?, ?, ?, ?, ?, ?, ?)",
                    (ch["id"], doc["id"], ch["content"], ch.get("sectionTitle"), ch.get("chunkType"),
                     ch.get("lineStart"), ch.get("lineEnd")))

    def search(self, query, options: dict | None = None) -> list[RetrievedChunk]:
        """sqlite.ts:125-209."""
        o = options or {}
        limit = js_or(o.get("limit"), 10)
        safe = query if isinstance(query, str) else str(query or "")
        type_filter = [t for t in (o.get("typeFilter") or []) if isinstance(t, str)]
        service_filter = [s for s in (o.get("serviceFilter") or []) if isinstance(s, str)]
        terms = " OR ".join(f'"{t}"*' for t in re.split(r"\s+", safe) if len(t) > 2)   # :139-143
        if not terms:
            return []                                                                   # :145-147
        sql = ("SELECT c.id, c.document_id, c.content, c.section_title, c.chunk_type, d.title, d.type, d.services, "
               "d.source_url, bm25(chunks_fts) as score FROM chunks_fts JOIN chunks c ON chunks_fts.rowid = c.rowid "
               "JOIN documents d ON c.document_id = d.id WHERE chunks_fts MATCH ?")
        params: list = [terms]
        if type_filter:
            sql += f" AND d.type IN ({','.join('?' * len(type_filter))})"
            params += type_filter
        if service_filter:
            sql += " AND (" + " OR ".join("d.services LIKE ?" for _ in service_filter) + ")"
            params += [f'%"{s}"%' for s in service_filter]
        sql += " ORDER BY score LIMIT ?"
        params.append(limit)
        try:
            rows = self.db.execute(sql, params).fetchall()
        except sqlite3.OperationalError:
            return []   # FTS5 syntax error from an odd token: the reference would throw; callers swallow it
        return [RetrievedChunk(id=r["id"], documentId=r["document_id"], title=r["section_title"] or r["title"],
                               content=r["content"], type=r["type"], services=json.loads(r["services"] or "[]"),
                               score=abs(r["score"]), sourceUrl=r["source_url"] or None) for r in rows]

    def has_document(self, doc_id: str) -> bool:
        """`getDocument(id) !== null` (sqlite.ts:261-265)."""
        return self.db.execute("SELECT 1 FROM documents WHERE id = ?", (doc_id,)).fetchone() is not None

    def get_document_count(self) -> int:
        """sqlite.ts:313-317."""
        return self.db.execute("SELECT COUNT(*) FROM documents").fetchone()[0]

    def get_document_counts_by_type(self) -> dict:
        """sqlite.ts:233-255."""
        counts = {t: 0 for t in ("runbook", "postmortem", "architecture", "ownership", "known_issue", "environment",
                                 "playbook", "faq")}
        for r in self.db.execute("SELECT type, COUNT(*) AS count FROM documents GROUP BY type"):
            if r["type"] in counts:
                counts[r["type"]] = r["count"]
        return counts

    def close(self) -> None:
        self.db.close()

    upsertDocument, hasDocument = upsert_document, has_document
    getDocumentCount, getDocumentCountsByType = get_document_count, get_document_counts_by_type
