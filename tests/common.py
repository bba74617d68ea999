"""Shared helpers for the parity tests (test infrastructure; may use the oracle)."""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np

GOLDEN = Path(__file__).parent / "golden" / "knn_golden.json"


def load_golden():
    g = json.loads(GOLDEN.read_text())
    for c in g["cases"]:
        c["query_f64"] = np.array([float.fromhex(x) for x in c["query"]], dtype=np.float64)
        c["rows_f64"] = np.array([[float.fromhex(x) for x in r] for r in c["rows"]], dtype=np.float64)
        c["scan_scores_f64"] = np.array([float.fromhex(x) for x in c["scan_scores"]], dtype=np.float64)
        c["fms_scores_f64"] = np.array([float.fromhex(x) for x in c["fms_scores"]], dtype=np.float64)
    return g


def group_devices(n):
    """A device list for an n-member group: one GPU each when the machine has n (the NCCL exchange), else n members
    co-located on GPU 0 (the copy exchange), so every G > 1 path runs on a one-GPU machine too."""
    import torch
    return list(range(n)) if torch.cuda.device_count() >= n else [0] * n


class OracleIndex:
    """CPU stand-in with the _native.Index surface, backed by the oracle.  Lets the CPU
    suite exercise the host logic (VectorStore, sharded merge) without a GPU.  Rows are
    rounded to bf16 like the device index."""

    def __init__(self, dim, device=0, capacity_hint=0):
        from runbookai_b200 import synth
        self._synth = synth
        self.dim = dim
        self.rows = np.zeros((0, dim), dtype=np.uint16)
        self.live = np.zeros((0,), dtype=np.uint8)
        self.slot_base = 0

    def _bits(self, rows):
        return self._synth.f32_to_bf16_bits(np.asarray(rows, dtype=np.float64).astype(np.float32))

    def append_f64(self, rows):
        rows = np.asarray(rows, dtype=np.float64).reshape(-1, self.dim)
        first = self.rows.shape[0]
        self.rows = np.concatenate([self.rows, self._bits(rows)])
        self.live = np.concatenate([self.live, np.ones(rows.shape[0], dtype=np.uint8)])
        return first

    def append_bf16(self, bits):
        first = self.rows.shape[0]
        self.rows = np.concatenate([self.rows, np.asarray(bits, dtype=np.uint16)])
        self.live = np.concatenate([self.live, np.ones(len(bits), dtype=np.uint8)])
        return first

    def overwrite_f64(self, slot, row):
        self.calls = getattr(self, "calls", 0) + 1
        self.rows[slot] = self._bits(np.asarray(row)[None, :])[0]

    def overwrite_f64_batch(self, slots, rows):
        """rbk_index_overwrite_f64_batch: one call; a slot named twice takes its last row."""
        self.calls = getattr(self, "calls", 0) + 1
        rows = np.asarray(rows, dtype=np.float64).reshape(-1, self.dim)
        for s, r in zip(slots, rows):
            self.rows[int(s)] = self._bits(r[None, :])[0]

    def tombstone(self, slots):
        self.live[np.asarray(slots, dtype=np.int64)] = 0

    def clear(self):
        self.rows = self.rows[:0]
        self.live = self.live[:0]

    def set_slot_base(self, b):
        self.slot_base = b

    def size(self):
        return self.rows.shape[0]

    def count(self):
        return int(self.live.sum())

    def close(self):
        pass

    def search(self, queries, k_fetch, min_score=0.5):
        import oracle
        q = np.asarray(queries, dtype=np.float64)
        if q.ndim == 1:
            q = q[None, :]
        if q.shape[1] != self.dim:
            from runbookai_b200._native import RBK_EDIM, DimensionError
            raise DimensionError(RBK_EDIM, "Vectors must have the same length")
        B = q.shape[0]
        slots = np.full((B, k_fetch), -1, dtype=np.int64)
        scores = np.full((B, k_fetch), np.nan)
        counts = np.zeros(B, dtype=np.int32)
        for b in range(B):
            s, v = oracle.search(self.rows, q[b], k_fetch, min_score, live=self.live)
            counts[b] = len(s)
            slots[b, :len(s)] = s + self.slot_base
            scores[b, :len(s)] = v
        return slots, scores, counts, 0.0


class HashEmbedder:
    """Deterministic offline embedder (the reference calls OpenAI over HTTPS): bf16-exact
    vectors derived from a hash of the text; texts sharing words get similar vectors."""

    def __init__(self, dim=64):
        self.dim = dim

    def _word(self, w):
        import hashlib
        seed = int.from_bytes(hashlib.md5(w.encode()).digest()[:8], "little")
        return np.random.Generator(np.random.Philox(seed)).standard_normal(self.dim)

    def embed_text(self, text):
        from runbookai_b200 import synth
        words = [w for w in text.lower().split() if w]
        v = np.sum([self._word(w) for w in words], axis=0) if words else np.zeros(self.dim)
        return synth.bf16_round(v).astype(np.float64).tolist()

    def embed_texts(self, texts):
        return [self.embed_text(t) for t in texts]
