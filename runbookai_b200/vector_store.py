"""Host mirror of src/knowledge/store/vector-store.ts with the scan on the GPU.

Same SQLite schema and f64-LE BLOB codec (vector-store.ts:34-88), same public surface
(search / addChunk(s) / deleteDocument / getCount / hasDocument / clear / close,
createVectorStore), same quirks (S4 `||` defaults, S7 2*topK over-fetch, S8 filters after
the cut, S9 final stable re-sort).  The only thing that changed is the hot loop
(:207-221): `for (const [id, embedding] of this.embeddings) ... sort ... slice` is one
`rbk_index_search_*` call on a device-resident bf16 index.  The in-RAM
`Map<string, number[]>` becomes (a) the device index and (b) the slot <-> id table kept
here.  Steps a4 (SQL fetch, filters, final cut, vector-store.ts:223-279) stay on the host.

The reference's methods are async only because of embedText (network); this mirror is
synchronous and adds the batched entry point `search_batch` the reference lacks.

Shared index (SURVEY §8f-2).  The reference builds a VectorStore - and re-parses every BLOB into the
Map - at each createRetriever() call site (e.g. hook-handlers.ts:329-337 opens and closes one per hook).
With the corpus on a GPU that would be an upload per call, so `shared=True` (the default of
create_vector_store) keeps ONE device index and slot table per (real path of the db, device) in this
process, reference-counted: the first opener loads it, later openers attach in O(1), the last close()
frees it.  Instances sharing an index see each other's mutations at once (the reference's copies only
converge at the next reload); each instance still owns its SQLite connection.

Reload sidecar (SURVEY §8f-2).  The reference re-parses every BLOB of the table at every construction
(vector-store.ts:56-66).  Next to `<db>` this mirror keeps `<db>.rbk`: the same float64 rows in rowid order as ONE
contiguous little-endian matrix plus the id table, stamped with a fingerprint of the table (row count and highest
rowid - every mutation the reference's code can make, INSERT OR REPLACE / DELETE, moves one of the two).  A matching
sidecar is memory-mapped and handed to `rbk_index_append_f64` in 64 MB slices: no SQL scan of the BLOBs, no per-row
Python, no intermediate copy.  A missing or stale sidecar falls back to the BLOBs (the source of truth) and is
rewritten at close().  RUNBOOK_KNN_SIDECAR=0 turns it off.
"""
from __future__ import annotations

import hashlib
import json
import os
import sqlite3
import struct
import threading
from dataclasses import asdict, dataclass, field
from typing import Sequence

import numpy as np

from . import embedder as _emb
from ._native import RBK_EDIM, RBK_MAX_K_FETCH, DimensionError, Index

SCHEMA = """
      CREATE TABLE IF NOT EXISTS vector_embeddings (
        id TEXT PRIMARY KEY,
        chunk_id TEXT NOT NULL,
        document_id TEXT NOT NULL,
        embedding BLOB NOT NULL,
        content TEXT NOT NULL,
        title TEXT,
        type TEXT NOT NULL,
        services TEXT,
        created_at TEXT DEFAULT CURRENT_TIMESTAMP
      );

      CREATE INDEX IF NOT EXISTS idx_vector_document_id ON vector_embeddings(document_id);
      CREATE INDEX IF NOT EXISTS idx_vector_type ON vector_embeddings(type);
"""
NOT_CONFIGURED = "Embedder not configured. Set OPENAI_API_KEY."
SIDECAR_MAGIC = b"RBKVEC1\0"
# magic, version, dim, rows, table count, max rowid, generation (PRAGMA user_version), hash of the table's tail,
# bytes of the id table
_SIDECAR_HDR = struct.Struct("<8sIIQQQQQQ")
_SIDECAR_VERSION = 2
_TAIL_ROWS = 64


@dataclass
class RetrievedChunk:
    """src/knowledge/types.ts:250-259."""
    id: str
    documentId: str
    title: str
    content: str
    type: str
    services: list[str] = field(default_factory=list)
    score: float = 0.0
    sourceUrl: str | None = None

    def to_dict(self) -> dict:
        d = asdict(self)
        if d["sourceUrl"] is None:
            del d["sourceUrl"]
        return d


def float_array_to_buffer(arr) -> bytes:
    """vector-store.ts:71-77 (writeDoubleLE per element)."""
    return np.asarray(arr, dtype="<f8").tobytes()


def buffer_to_float_array(buf: bytes) -> np.ndarray:
    """vector-store.ts:82-88."""
    return np.frombuffer(buf, dtype="<f8")


class _IndexState:
    """What replaces the reference's `embeddings: Map<string, number[]>`: the device index plus the
    slot <-> id table.  One per VectorStore, or one per (db path, device) when shared."""

    def __init__(self, key=None):
        self.key = key                       # registry key, None = private
        self.refs = 1
        self.loaded = False
        self.lock = threading.RLock()        # serialises mutation / table reads across sharing instances
        self.index: Index | None = None
        self.ids: list[str | None] = []      # slot -> id (None = deleted)
        self.slot_of: dict[str, int] = {}    # live id -> slot  (the reference's Map keys)
        self.bad_ids: set[str] = set()       # ids whose stored vector has another length: while any is in the
        #                                      Map the reference's search throws (S2); deleting / re-setting it heals


_SHARED: dict[tuple[str, int], _IndexState] = {}
_SHARED_LOCK = threading.Lock()


def shared_index_count() -> int:
    """Device indexes currently kept alive by the per-path registry (introspection / tests)."""
    with _SHARED_LOCK:
        return len(_SHARED)


class VectorStore:
    def __init__(self, db_path: str, device: int | None = None, index_factory=None, shared: bool = False,
                 f64_on_host: bool | None = None):
        # index_factory(dim, device) -> object with the _native.Index surface; tests inject a
        # CPU stand-in to exercise the host logic where there is no GPU
        # keep_f64: the reference stores float64 embeddings; keep them so the re-rank is exact for any input.
        # f64_on_host (None: RUNBOOK_KNN_F64_ON_HOST=1 enables): those float64 rows live in pinned host memory instead
        # of on the GPU - the same answers, about 5x the rows per GPU at d = 1536, host RAM and PCIe reads in the
        # re-rank instead.  A shared index keeps the placement of the instance that created it.
        if f64_on_host is None:
            f64_on_host = os.environ.get("RUNBOOK_KNN_F64_ON_HOST", "0") == "1"
        self.f64_on_host = on_host = bool(f64_on_host)
        self._index_factory = index_factory or (
            lambda dim, dev: Index(dim, device=dev, keep_f64=True, f64_on_host=on_host))
        # one connection, usable from the micro-batcher's worker thread too; serialised by a lock
        self.db = sqlite3.connect(db_path, check_same_thread=False)
        self.db.row_factory = sqlite3.Row
        self._db_lock = threading.RLock()
        self.device = int(os.environ.get("RUNBOOK_KNN_DEVICE", "0")) if device is None else device
        self._closed = False
        self._db_path = db_path
        self._sidecar = (db_path != ":memory:" and not db_path.startswith("file:")
                         and os.environ.get("RUNBOOK_KNN_SIDECAR", "1") != "0")
        self.loaded_from_sidecar = False
        self._init_schema()
        if shared and db_path != ":memory:" and not db_path.startswith("file:"):
            key = (os.path.realpath(db_path), self.device)
            with _SHARED_LOCK:
                st = _SHARED.get(key)
                if st is None:
                    st = _SHARED[key] = _IndexState(key)
                else:
                    st.refs += 1
            self._st = st
        else:
            self._st = _IndexState()
        with self._st.lock:                  # a second opener waits for the first one's load
            if not self._st.loaded:
                try:
                    self._load_embeddings()
                    self._st.loaded = True
                except BaseException:
                    # a half-built shared state must not be found by the next opener: drop it, the device index and
                    # the connection, then let the caller see the error (e.g. cudaMalloc failed mid-append)
                    st = self._st
                    if st.key is not None:
                        with _SHARED_LOCK:
                            st.refs -= 1
                            if _SHARED.get(st.key) is st:
                                _SHARED.pop(st.key, None)
                    if st.index is not None:
                        try:
                            st.index.close()
                        finally:
                            st.index = None
                    st.ids.clear()
                    st.slot_of.clear()
                    st.bad_ids.clear()
                    self._closed = True
                    self.db.close()
                    raise

    # the state lives in self._st so that instances on the same db can share it
    @property
    def _index(self):
        return self._st.index

    @_index.setter
    def _index(self, v):
        self._st.index = v

    @property
    def _ids(self):
        return self._st.ids

    @property
    def _slot_of(self):
        return self._st.slot_of

    @property
    def _ragged(self) -> bool:
        """`Vectors must have the same length` is thrown exactly while a mismatched embedding is in the Map."""
        return bool(self._st.bad_ids)

    # ------------------------------------------------------------------ setup
    def _init_schema(self) -> None:
        self.db.executescript(SCHEMA)

    def _ensure_index(self, dim: int) -> Index:
        if self._index is None:
            self._index = self._index_factory(dim, self.device)
        return self._index

    # ------------------------------------------------------------------ reload sidecar
    def _fingerprint(self) -> tuple[int, int, int, int]:
        """What a sidecar must match to be used: row count, highest rowid, the generation counter this class bumps
        inside every mutating transaction (`PRAGMA user_version`: in the database header, transactional, unused by
        the reference), and a hash of the ids and BLOBs of the last rows by rowid.  Count and rowid alone are not
        enough: SQLite hands the rowid of a deleted LAST row out again, so re-embedding the newest chunk leaves both
        unchanged.  The tail hash covers writers that do not know about the counter (the unpatched reference on the
        same file), whose inserts and replacements land at the tail."""
        r = self.db.execute("SELECT COUNT(*), COALESCE(MAX(rowid), 0) FROM vector_embeddings").fetchone()
        gen = int(self.db.execute("PRAGMA user_version").fetchone()[0])
        h = hashlib.blake2b(digest_size=8)
        for row in self.db.execute("SELECT id, embedding FROM vector_embeddings ORDER BY rowid DESC LIMIT ?",
                                   (_TAIL_ROWS,)):
            h.update(row["id"].encode("utf-8"))
            h.update(b"\0")
            h.update(row["embedding"])
        return int(r[0]), int(r[1]), gen, int.from_bytes(h.digest(), "little")

    def _bump_generation(self) -> None:
        """Inside the caller's transaction: the table is about to differ from every sidecar written so far."""
        gen = int(self.db.execute("PRAGMA user_version").fetchone()[0])
        self.db.execute(f"PRAGMA user_version = {(gen + 1) & 0x7FFFFFFF}")

    def _load_sidecar(self) -> bool:
        """Bulk-load from `<db>.rbk` if it describes the table as it is now."""
        path = self._db_path + ".rbk"
        try:
            with open(path, "rb") as f:
                hdr = f.read(_SIDECAR_HDR.size)
                if len(hdr) != _SIDECAR_HDR.size:
                    return False
                magic, ver, dim, n, count, max_rowid, gen, tail, id_bytes = _SIDECAR_HDR.unpack(hdr)
                if (magic != SIDECAR_MAGIC or ver != _SIDECAR_VERSION or n != count
                        or (count, max_rowid, gen, tail) != self._fingerprint()):
                    return False
                off = (_SIDECAR_HDR.size + id_bytes + 63) // 64 * 64
                if os.path.getsize(path) != off + n * dim * 8:
                    return False
                ids = f.read(id_bytes).decode("utf-8").split("\n") if n else []
            if len(ids) != n:
                return False
            if n == 0:
                return True
            mm = np.memmap(path, dtype="<f8", mode="r", offset=off, shape=(n, dim))
            ix = self._ensure_index(dim)
            step = max(1, (64 << 20) // (dim * 8))
            for r0 in range(0, n, step):
                first = ix.append_f64(mm[r0:r0 + step])          # straight from the page cache to the device
                if first != r0:
                    raise RuntimeError("slot numbering out of step while loading the sidecar")
            for i, vid in enumerate(ids):
                self._slot_of[vid] = i
                self._ids.append(vid)
            del mm
            self.loaded_from_sidecar = True
            return True
        except (OSError, ValueError, UnicodeDecodeError):
            return False

    def save_sidecar(self) -> bool:
        """Write `<db>.rbk` for the table as it is now (called by close() when missing or stale).  Rows of differing
        length (S2) cannot be one matrix: no sidecar then."""
        if not self._sidecar:
            return False
        with self._db_lock:
            count, max_rowid, gen, tail = self._fingerprint()
            cur = self.db.execute("SELECT id, embedding FROM vector_embeddings ORDER BY rowid")
            first = cur.fetchone()
            dim = len(first["embedding"]) // 8 if first else 0
            tmp = self._db_path + ".rbk.tmp"
            with open(tmp, "wb") as f:
                rows = ([first] if first else [])
                id_list = []
                # the matrix offset depends on the size of the id table, which is only known after the scan: stream
                # the BLOBs to a scratch file once, then write header + ids and append the scratch file
                blobs_path = tmp + ".rows"
                with open(blobs_path, "wb") as bf:
                    while rows:
                        for r in rows:
                            if len(r["embedding"]) != dim * 8 or "\n" in r["id"]:
                                bf.close()
                                os.remove(blobs_path)
                                f.close()
                                os.remove(tmp)
                                return False
                            id_list.append(r["id"])
                            bf.write(r["embedding"])
                        rows = cur.fetchmany(4096)
                idb = "\n".join(id_list).encode("utf-8")
                f.seek(0)
                f.write(_SIDECAR_HDR.pack(SIDECAR_MAGIC, _SIDECAR_VERSION, dim, len(id_list), count, max_rowid, gen, tail,
                                          len(idb)))
                f.write(idb)
                f.write(b"\0" * ((_SIDECAR_HDR.size + len(idb) + 63) // 64 * 64 - _SIDECAR_HDR.size - len(idb)))
                with open(blobs_path, "rb") as bf:
                    while True:
                        buf = bf.read(64 << 20)
                        if not buf:
                            break
                        f.write(buf)
                os.remove(blobs_path)
            os.replace(tmp, self._db_path + ".rbk")
        return True

    def _sidecar_is_current(self) -> bool:
        try:
            with open(self._db_path + ".rbk", "rb") as f:
                hdr = f.read(_SIDECAR_HDR.size)
            magic, ver, _, _, count, max_rowid, gen, tail, _ = _SIDECAR_HDR.unpack(hdr)
            return (magic == SIDECAR_MAGIC and ver == _SIDECAR_VERSION
                    and (count, max_rowid, gen, tail) == self._fingerprint())
        except (OSError, struct.error):
            return False

    def _load_embeddings(self) -> None:
        """vector-store.ts:56-66: every row, in rowid order, into the (device) index."""
        if self._sidecar and self._load_sidecar():
            return
        rows = self.db.execute("SELECT id, embedding FROM vector_embeddings").fetchall()
        if not rows:
            return
        dim = len(rows[0]["embedding"]) // 8
        good = [r for r in rows if len(r["embedding"]) == dim * 8]
        self._st.bad_ids.update(r["id"] for r in rows if len(r["embedding"]) != dim * 8)
        ix = self._ensure_index(dim)
        step = max(1, (32 << 20) // (dim * 8))
        for r0 in range(0, len(good), step):
            blob = b"".join(r["embedding"] for r in good[r0:r0 + step])
            first = ix.append_f64(np.frombuffer(blob, dtype="<f8").reshape(-1, dim))
            for i, r in enumerate(good[r0:r0 + step]):   # the slot the ENGINE assigned, not a private count
                while len(self._ids) < first + i:
                    self._ids.append(None)
                self._slot_of[r["id"]] = first + i
                self._ids.append(r["id"])

    # ------------------------------------------------------------------ mutation
    def _set(self, vid: str, embedding) -> None:
        """`this.embeddings.set(id, embedding)` (vector-store.ts:129,178)."""
        e = np.asarray(embedding, dtype=np.float64)
        ix = self._ensure_index(e.shape[0])
        slot = self._slot_of.get(vid)
        if e.shape[0] != ix.dim:
            # the reference stores it and throws on every search until the id is deleted or re-set correctly
            # (deviation, tie order only: once re-set correctly the id is appended as a new key here, while the
            # reference's Map kept the key's original position all along)
            self._st.bad_ids.add(vid)
            if slot is not None:          # the old, well-formed vector is no longer in the Map either
                self._slot_of.pop(vid, None)
                self._ids[slot] = None
                ix.tombstone([slot])
            return
        self._st.bad_ids.discard(vid)
        if slot is not None:
            ix.overwrite_f64(slot, e)     # existing key keeps its Map position (S9b)
        else:
            self._slot_of[vid] = ix.append_f64(e[None, :])
            self._ids.append(vid)

    _INSERT = """
      INSERT OR REPLACE INTO vector_embeddings
      (id, chunk_id, document_id, embedding, content, title, type, services)
      VALUES (?, ?, ?, ?, ?, ?, ?, ?)
    """

    def add_chunk(self, chunk: dict, document_title: str, type: str, services: Sequence[str]) -> None:
        """vector-store.ts:93-130."""
        if not _emb.is_embedder_configured():
            raise RuntimeError(NOT_CONFIGURED)
        text = "\n\n".join(p for p in [document_title, chunk.get("sectionTitle"), chunk["content"]] if p)
        embedding = _emb.embed_text(text)
        vid = f"vec_{chunk['id']}"
        with self._st.lock, self._db_lock:
            with self.db:
                self.db.execute(self._INSERT, (vid, chunk["id"], chunk["documentId"],
                                               float_array_to_buffer(embedding), chunk["content"],
                                               chunk.get("sectionTitle") or document_title, type,
                                               json.dumps(list(services), separators=(",", ":"))))
                self._bump_generation()   # after the first statement: inside the transaction it opened
            self._set(vid, embedding)

    def add_chunks(self, chunks: Sequence[dict]) -> None:
        """vector-store.ts:135-183.  chunks: [{chunk, documentTitle, type, services}]."""
        if not _emb.is_embedder_configured():
            raise RuntimeError(NOT_CONFIGURED)
        texts = ["\n\n".join(p for p in [c["documentTitle"], c["chunk"].get("sectionTitle"), c["chunk"]["content"]]
                             if p) for c in chunks]
        embeddings = _emb.embed_texts(texts)
        with self._st.lock, self._db_lock:
            self._add_embedded(chunks, embeddings)

    def _add_embedded(self, chunks, embeddings) -> None:
        with self.db:  # one transaction
            for c, e in zip(chunks, embeddings):
                ch = c["chunk"]
                self.db.execute(self._INSERT, (f"vec_{ch['id']}", ch["id"], ch["documentId"],
                                               float_array_to_buffer(e), ch["content"],
                                               ch.get("sectionTitle") or c["documentTitle"], c["type"],
                                               json.dumps(list(c["services"]), separators=(",", ":"))))
            if chunks:
                self._bump_generation()
        self._set_many([(f"vec_{c['chunk']['id']}", e) for c, e in zip(chunks, embeddings)])

    def _set_many(self, items) -> None:
        """`this.embeddings.set(id, e)` for every item in order (vector-store.ts:178), as TWO engine calls: the
        re-sets of ids already in the Map in one `overwrite_f64_batch` (a re-embedded document: one host round trip,
        not one per chunk), the new ids in one `append_f64`.  Same final Map as the sequential sets: an existing key
        keeps its position, new keys are appended in order of first appearance, the last value of a key wins."""
        items = [(v, np.asarray(e, dtype=np.float64)) for v, e in items]
        if not items:
            return
        dim = self._index.dim if self._index is not None else items[0][1].shape[0]
        if any(e.ndim != 1 or e.shape[0] != dim for _, e in items):
            for v, e in items:            # a wrong-length vector in the batch: the careful path, one by one
                self._set(v, e)
            return
        ix = self._ensure_index(dim)
        last: dict[str, np.ndarray] = {}
        fresh: list[str] = []
        for v, e in items:
            if v not in self._slot_of and v not in last:
                fresh.append(v)
            last[v] = e
        again = [v for v in last if v in self._slot_of]
        if again:
            ix.overwrite_f64_batch([self._slot_of[v] for v in again], np.stack([last[v] for v in again]))
        if fresh:
            first = ix.append_f64(np.stack([last[v] for v in fresh]))
            for i, v in enumerate(fresh):
                self._slot_of[v] = first + i
                while len(self._ids) < first + i:
                    self._ids.append(None)
                self._ids.append(v)
        self._st.bad_ids.difference_update(last)

    def delete_document(self, document_id: str) -> None:
        """vector-store.ts:285-297."""
        with self._st.lock, self._db_lock:
            self._delete_document(document_id)

    def _delete_document(self, document_id: str) -> None:
        rows = self.db.execute("SELECT id FROM vector_embeddings WHERE document_id = ?", (document_id,)).fetchall()
        slots = []
        for r in rows:
            self._st.bad_ids.discard(r["id"])
            s = self._slot_of.pop(r["id"], None)
            if s is not None:
                self._ids[s] = None
                slots.append(s)
        if slots and self._index is not None:
            self._index.tombstone(slots)
        with self.db:
            self.db.execute("DELETE FROM vector_embeddings WHERE document_id = ?", (document_id,))
            self._bump_generation()

    def compact(self) -> int:
        """Give the slots of deleted rows back (the reference's `Map.delete` frees its entry; a tombstone does not):
        the device index moves its live rows down in Map order and the slot <-> id table follows its old_to_new map.
        Returns the number of slots reclaimed.  An index without `compact` (a device group) is left as it is.  The
        SQLite table, the reload sidecar (which describes the table, not slots) and `bad_ids` do not change.  Holds
        the state lock, like every search, so no search maps its slots through a half-updated table."""
        with self._st.lock:
            ix = self._index
            fn = getattr(ix, "compact", None)
            if fn is None:
                return 0
            before = ix.size()
            old_to_new = fn()
            ids: list[str | None] = [None] * ix.size()
            for s, vid in enumerate(self._ids):
                if vid is None:
                    continue
                new = int(old_to_new[s])
                if new < 0:
                    raise RuntimeError(f"compaction dropped the live slot {s} ({vid})")
                ids[new] = vid
                self._slot_of[vid] = new
            self._ids[:] = ids
            return before - ix.size()

    def trim(self) -> None:
        """Give the device memory of reclaimed slots back: the index's capacity drops to what its rows need and its
        scratch buffers are released (after compact() or clear()).  No slot moves and no answer changes.  An index
        without `trim` is left as it is.  Holds the state lock, like compact()."""
        with self._st.lock:
            fn = getattr(self._index, "trim", None)
            if fn is not None:
                fn()

    def get_count(self) -> int:
        """vector-store.ts:302-307."""
        return self.db.execute("SELECT COUNT(*) as count FROM vector_embeddings").fetchone()["count"]

    def has_document(self, document_id: str) -> bool:
        """vector-store.ts:312-317."""
        return self.db.execute("SELECT COUNT(*) as count FROM vector_embeddings WHERE document_id = ?",
                               (document_id,)).fetchone()["count"] > 0

    def clear(self) -> None:
        """vector-store.ts:322-325."""
        with self._st.lock, self._db_lock:
            with self.db:
                self.db.execute("DELETE FROM vector_embeddings")
                self._bump_generation()
            self._ids.clear()
            self._slot_of.clear()
            self._st.bad_ids.clear()
            if self._index is not None:
                self._index.clear()

    def close(self) -> None:
        """vector-store.ts:330-332.  The device index goes with the LAST instance that shares it."""
        if self._closed:
            return
        self._closed = True
        if self._sidecar:
            try:
                if not self._sidecar_is_current():
                    self.save_sidecar()
            except (OSError, sqlite3.Error):
                pass                      # the sidecar is an accelerator, never a reason to fail a close()
        self.db.close()
        st = self._st
        if st.key is not None:
            with _SHARED_LOCK:
                st.refs -= 1
                last = st.refs == 0
                if last:
                    _SHARED.pop(st.key, None)
        else:
            last = True
        if last:
            with st.lock:
                if st.index is not None:
                    st.index.close()
                    st.index = None

    # ------------------------------------------------------------------ search
    def search(self, query: str, options: dict | None = None, **kw) -> list[RetrievedChunk]:
        """vector-store.ts:188-280."""
        return self.search_batch([query], options, **kw)[0]

    def search_batch(self, queries: Sequence[str], options: dict | None = None, **kw) -> list[list[RetrievedChunk]]:
        """B queries in one device pass (what `B sequential search() calls` cost the reference)."""
        o = dict(options or {})
        o.update(kw)
        if not _emb.is_embedder_configured():
            raise RuntimeError(NOT_CONFIGURED)                       # :197-199
        top_k = o.get("topK") or o.get("top_k") or 10                # :201  (0/None -> 10)
        min_score = o.get("minScore") or o.get("min_score") or 0.5   # :202  (0/None -> 0.5)
        type_filter = o.get("typeFilter") or o.get("type_filter")
        service_filter = o.get("serviceFilter") or o.get("service_filter")
        q = np.asarray(_emb.embed_texts(list(queries)) if len(queries) > 1 else [_emb.embed_text(queries[0])],
                       dtype=np.float64)                              # :205
        with self._st.lock:   # the slot table must be the one the scan ran against
            if self._index is None or not self._ids:
                return [[] for _ in queries]
            if self._ragged or q.shape[1] != self._index.dim:
                raise DimensionError(RBK_EDIM, "Vectors must have the same length")   # embedder.ts:170
            # :207-221 — scan, `>= minScore`, stable sort desc, first 2*topK: one device call
            # (2*topK beyond the scan's candidate lists - limit: 50 / 1000 call sites, infra-context.ts:229,
            # knowledge-context.ts:150 - takes the exact-scores path: same answer, one fp64 pass per query)
            search = getattr(self._index, "search_any_k", None) if 2 * top_k > RBK_MAX_K_FETCH else None
            slots, scores, counts, _ = (search or self._index.search)(q, 2 * top_k, min_score)
            ids = [[self._ids[int(s)] for s in slots[b, :counts[b]]] for b in range(len(queries))]
        return [self._hydrate(ids[b], scores[b, :counts[b]], top_k, type_filter, service_filter)
                for b in range(len(queries))]

    def _hydrate(self, top_ids, scores, top_k, type_filter, service_filter) -> list[RetrievedChunk]:
        """vector-store.ts:223-279 (a4): stays on the host."""
        pairs = [(i, float(sc)) for i, sc in zip(top_ids, scores) if i is not None]   # None: deleted meanwhile
        top_ids = [i for i, _ in pairs]
        if not top_ids:
            return []                                                 # :223-225
        sql = ("SELECT id, chunk_id, document_id, content, title, type, services FROM vector_embeddings "
               f"WHERE id IN ({','.join('?' * len(top_ids))})")
        params: list = list(top_ids)
        if type_filter:
            sql += f" AND type IN ({','.join('?' * len(type_filter))})"   # :237-241
            params += list(type_filter)
        with self._db_lock:
            rows = self.db.execute(sql, params).fetchall()
        score_map = dict(pairs)
        results: list[RetrievedChunk] = []
        for row in rows:
            services = json.loads(row["services"] or "[]")
            if service_filter and not any(s in services for s in service_filter):   # :261-264
                continue
            results.append(RetrievedChunk(id=row["chunk_id"], documentId=row["document_id"], title=row["title"] or "",
                                          content=row["content"], type=row["type"], services=services,
                                          score=score_map.get(row["id"]) or 0))
        results.sort(key=lambda r: -r.score)                          # :278 (stable, like V8)
        return results[:top_k]                                        # :279

    # reference spellings
    addChunk, addChunks, deleteDocument = add_chunk, add_chunks, delete_document
    getCount, hasDocument = get_count, has_document


def create_vector_store(base_dir: str = ".runbook", device: int | None = None, index_factory=None,
                        shared: bool | None = None) -> VectorStore:
    """vector-store.ts:338-341.  shared (default on; RUNBOOK_KNN_SHARED_INDEX=0 turns it off): call sites
    that build and close a store per use attach to the process-wide index of that db instead of re-uploading."""
    if shared is None:
        shared = os.environ.get("RUNBOOK_KNN_SHARED_INDEX", "1") != "0"
    return VectorStore(f"{base_dir}/vectors.db", device, index_factory, shared=shared)


createVectorStore = create_vector_store
