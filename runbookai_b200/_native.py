"""ctypes binding of include/rbk_knn.h — the same symbols the N-API addon binds.

There is no fallback of any kind: if librbk_knn.so is missing this module raises at
import, and if there is no CUDA device every index operation raises RbkError(RBK_ECUDA).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

LIB_PATH = Path(__file__).resolve().parent / "lib" / "librbk_knn.so"

RBK_OK, RBK_EINVAL, RBK_ENOMEM, RBK_ECUDA, RBK_ENCCL, RBK_EDIM, RBK_ENOTF32 = range(7)
RBK_MAX_K_FETCH = 112
RBK_MAX_K_FETCH_LARGE = 4096
RBK_INDEX_KEEP_F64 = 1
RBK_INDEX_F64_ON_HOST = 2
RBK_INDEX_ROWS_ON_HOST = RBK_INDEX_F64_ON_HOST
RBK_INDEX_KEEP_F32 = 64
RBK_INDEX_KEEP_F32_SPLIT = 128
RBK_INDEX_SCAN_F16 = 16

# every symbol include/rbk_knn.h declares (tests check the .so exports all of them)
SYMBOLS = [
    "rbk_abi_version", "rbk_last_error", "rbk_index_create", "rbk_index_create_ex", "rbk_index_destroy", "rbk_index_set_stream",
    "rbk_index_set_slot_base", "rbk_index_append_f64", "rbk_index_append_f32", "rbk_index_append_bf16",
    "rbk_index_append_bf16_device", "rbk_index_append_f64_device", "rbk_index_overwrite_f64", "rbk_index_overwrite_f64_batch", "rbk_index_tombstone", "rbk_index_compact", "rbk_index_clear", "rbk_index_trim",
    "rbk_index_count", "rbk_index_size", "rbk_index_dim", "rbk_index_storage_bytes", "rbk_index_read_rows_bf16", "rbk_index_read_rows_f16", "rbk_index_search_f64",
    "rbk_index_search_f32", "rbk_index_search_large_f64", "rbk_index_search_unbounded_f64", "rbk_index_exact_scores_f64", "rbk_index_search_device", "rbk_index_search_device_async", "rbk_merge_topk_device",
    "rbk_packed_block_bytes", "rbk_packed_flags_offset",
    "rbk_merge_topk_packed_device", "rbk_index_stats",
    "rbk_index_debug_scores_f32",
    "rbk_group_create", "rbk_group_destroy", "rbk_group_append_f64", "rbk_group_append_f32", "rbk_group_append_bf16",
    "rbk_group_overwrite_f64_batch", "rbk_group_tombstone", "rbk_group_clear", "rbk_group_compact", "rbk_group_trim", "rbk_group_count", "rbk_group_size",
    "rbk_group_devices", "rbk_group_member", "rbk_group_redone_batches", "rbk_group_search_f32", "rbk_group_search_f64",
    "rbk_group_search_large_f64", "rbk_group_search_unbounded_f64",
    "rbk_index_flags", "rbk_index_set_tier", "rbk_group_set_tier",
    "rbk_index_search_each_f64", "rbk_group_search_each_f64",
    "rbk_index_search_slots_f64", "rbk_group_search_slots_f64",
    "rbk_index_similar_pairs_f64", "rbk_group_similar_pairs_f64",
    "rbk_index_search_mmr_f64", "rbk_group_search_mmr_f64",
]


class RbkError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(message)
        self.status = status


class DimensionError(RbkError, ValueError):
    """'Vectors must have the same length' (embedder.ts:169-171)."""


class NotFloat32Error(RbkError, ValueError):
    """RBK_ENOTF32: a keep_f32 index (or group) was given a float64 value that no float32 holds exactly; nothing was
    written.  Widen the index (set_tier(exact_rows="f64")) and repeat the call to store it."""


class RbkStats(C.Structure):
    _fields_ = [
        ("searches", C.c_int64), ("queries", C.c_int64), ("fallback_queries", C.c_int64),
        ("scan_launches", C.c_int64), ("kernel_launches", C.c_int64), ("last_scan_ms", C.c_float),
        ("last_total_ms", C.c_float), ("last_kprime", C.c_int32), ("sm_count", C.c_int32),
        ("last_ring_stages", C.c_int32), ("retry_batches", C.c_int32),
        ("scan_ms_total", C.c_double), ("scans_timed", C.c_int64), ("graph_replays", C.c_int64),
    ]


def _load() -> C.CDLL:
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m runbookai_b200.build` "
            "(or __graft_entry__.build()).  This engine has no CPU or library fallback.")
    lib = C.CDLL(str(LIB_PATH))
    vp, i32, i64, f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    lib.rbk_abi_version.restype = C.c_int
    lib.rbk_last_error.restype = C.c_char_p
    lib.rbk_index_create.argtypes = [i32, i32, i64, C.POINTER(vp)]
    lib.rbk_index_create_ex.argtypes = [i32, i32, i64, C.c_uint32, C.POINTER(vp)]
    lib.rbk_index_destroy.argtypes = [vp]
    lib.rbk_index_destroy.restype = None
    lib.rbk_index_set_stream.argtypes = [vp, vp]
    lib.rbk_index_set_slot_base.argtypes = [vp, i64]
    for n in ("rbk_index_append_f64", "rbk_index_append_f32", "rbk_index_append_bf16",
              "rbk_index_append_bf16_device", "rbk_index_append_f64_device"):
        getattr(lib, n).argtypes = [vp, vp, i64, C.POINTER(i64)]
    lib.rbk_index_overwrite_f64.argtypes = [vp, i64, vp]
    lib.rbk_index_overwrite_f64_batch.argtypes = [vp, vp, i64, vp]
    lib.rbk_index_tombstone.argtypes = [vp, vp, i64]
    lib.rbk_index_compact.argtypes = [vp, vp, i64]
    lib.rbk_index_clear.argtypes = [vp]
    lib.rbk_index_trim.argtypes = [vp]
    for n in ("rbk_index_count", "rbk_index_size"):
        getattr(lib, n).argtypes = [vp]
        getattr(lib, n).restype = i64
    lib.rbk_index_dim.argtypes = [vp]
    lib.rbk_index_dim.restype = i32
    lib.rbk_index_storage_bytes.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    lib.rbk_index_read_rows_bf16.argtypes = [vp, i64, i64, vp]
    lib.rbk_index_read_rows_f16.argtypes = [vp, i64, i64, vp]
    for n in ("rbk_index_search_f64", "rbk_index_search_f32", "rbk_index_search_large_f64",
              "rbk_index_search_unbounded_f64"):
        getattr(lib, n).argtypes = [vp, vp, i32, i32, i32, f64, vp, vp, vp, C.POINTER(C.c_float)]
    lib.rbk_index_search_device.argtypes = [vp, vp, i32, i32, f64, vp, vp, vp]
    lib.rbk_index_exact_scores_f64.argtypes = [vp, vp, i32, i32, vp]
    lib.rbk_index_search_device_async.argtypes = [vp, vp, i32, i32, f64, vp, vp, vp, vp]
    lib.rbk_merge_topk_device.argtypes = [i32, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.rbk_packed_block_bytes.argtypes = [i32, i32]
    lib.rbk_packed_block_bytes.restype = i64
    lib.rbk_packed_flags_offset.argtypes = [i32, i32]
    lib.rbk_packed_flags_offset.restype = i64
    lib.rbk_merge_topk_packed_device.argtypes = [i32, vp, i32, i32, i32, vp, vp, vp, vp, vp]
    lib.rbk_index_stats.argtypes = [vp, C.POINTER(RbkStats)]
    lib.rbk_group_create.argtypes = [i32, vp, i32, i64, C.c_uint32, C.POINTER(vp)]
    lib.rbk_group_destroy.argtypes = [vp]
    lib.rbk_group_destroy.restype = None
    for n in ("rbk_group_append_f64", "rbk_group_append_f32", "rbk_group_append_bf16"):
        getattr(lib, n).argtypes = [vp, vp, i64, C.POINTER(i64)]
    lib.rbk_group_overwrite_f64_batch.argtypes = [vp, vp, i64, vp]
    lib.rbk_group_tombstone.argtypes = [vp, vp, i64]
    lib.rbk_group_clear.argtypes = [vp]
    lib.rbk_group_compact.argtypes = [vp, vp, i64]
    lib.rbk_group_trim.argtypes = [vp]
    for n in ("rbk_group_count", "rbk_group_size", "rbk_group_redone_batches"):
        getattr(lib, n).argtypes = [vp]
        getattr(lib, n).restype = i64
    lib.rbk_group_devices.argtypes = [vp]
    lib.rbk_group_devices.restype = i32
    lib.rbk_group_member.argtypes = [vp, i32]
    lib.rbk_group_member.restype = vp
    for n in ("rbk_group_search_f32", "rbk_group_search_f64", "rbk_group_search_large_f64",
              "rbk_group_search_unbounded_f64"):
        getattr(lib, n).argtypes = [vp, vp, i32, i32, i32, f64, vp, vp, vp, C.POINTER(C.c_float)]
    for n in ("rbk_index_search_each_f64", "rbk_group_search_each_f64"):
        getattr(lib, n).argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp, C.POINTER(C.c_float)]
    for n in ("rbk_index_search_slots_f64", "rbk_group_search_slots_f64"):
        getattr(lib, n).argtypes = [vp, vp, i32, vp, vp, vp, vp, vp, C.POINTER(C.c_float)]
    for n in ("rbk_index_similar_pairs_f64", "rbk_group_similar_pairs_f64"):
        getattr(lib, n).argtypes = [vp, f64, i64, i64, vp, vp, vp, C.POINTER(i64), C.POINTER(i64),
                                    C.POINTER(C.c_float)]
    for n in ("rbk_index_search_mmr_f64", "rbk_group_search_mmr_f64"):
        getattr(lib, n).argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_float)]
    lib.rbk_index_debug_scores_f32.argtypes = [vp, vp, i32, vp]
    lib.rbk_index_flags.argtypes = [vp]
    lib.rbk_index_flags.restype = C.c_uint32
    lib.rbk_index_set_tier.argtypes = [vp, C.c_uint32]
    lib.rbk_group_set_tier.argtypes = [vp, C.c_uint32]
    return lib


lib = _load()


def check(status: int) -> None:
    if status == RBK_OK:
        return
    msg = (lib.rbk_last_error() or b"").decode("utf-8", "replace")
    if status == RBK_EDIM:
        raise DimensionError(status, msg)
    if status == RBK_ENOTF32:
        raise NotFloat32Error(status, msg)
    raise RbkError(status, msg)


def ptr(a: np.ndarray | None):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _index_flags(keep_f64: bool, f64_on_host: bool, scan_f16: bool = False, keep_f32: bool = False,
                 keep_f32_split: bool = False) -> int:
    """f64_on_host or scan_f16 without a keep bit, or several keep bits, are passed through: the library rejects them
    with its own message."""
    return ((RBK_INDEX_KEEP_F64 if keep_f64 else 0) | (RBK_INDEX_KEEP_F32 if keep_f32 else 0)
            | (RBK_INDEX_KEEP_F32_SPLIT if keep_f32_split else 0)
            | (RBK_INDEX_F64_ON_HOST if f64_on_host else 0) | (RBK_INDEX_SCAN_F16 if scan_f16 else 0))


_EXACT_ROWS = {"f64": RBK_INDEX_KEEP_F64, "f32": RBK_INDEX_KEEP_F32, "f32_split": RBK_INDEX_KEEP_F32_SPLIT}
_KEEP_BITS = RBK_INDEX_KEEP_F64 | RBK_INDEX_KEEP_F32 | RBK_INDEX_KEEP_F32_SPLIT


def exact_rows_of(flags: int) -> str | None:
    """'f64' / 'f32' / 'f32_split' for an index keeping float64 / float32 / split float32 exact rows, None for one
    without."""
    flags = int(flags)
    for name, bit in _EXACT_ROWS.items():
        if flags & bit:
            return name
    return None


def _tier_flags(current: int, f64_on_host, scan_f16, exact_rows=None) -> int:
    """The flag set of a tier change from the current one: None keeps a setting; exact_rows 'f64' / 'f32' sets the
    keep bit even on an index without exact rows, which the library then refuses with its own message)."""
    flags = int(current)
    if exact_rows is not None:
        if exact_rows not in _EXACT_ROWS:
            raise ValueError(f"exact_rows must be 'f64', 'f32', 'f32_split' or None, not {exact_rows!r}")
        flags = (flags & ~_KEEP_BITS) | _EXACT_ROWS[exact_rows]
    for value, bit, name in ((f64_on_host, RBK_INDEX_F64_ON_HOST, "f64_on_host"),
                             (scan_f16, RBK_INDEX_SCAN_F16, "scan_f16")):
        if value is None:
            continue
        if not isinstance(value, (bool, np.bool_)):
            raise TypeError(f"{name} must be a bool or None, not {type(value).__name__}")
        flags = flags | bit if value else flags & ~bit
    return flags


def _search_large(fn, h, queries, k_fetch: int, min_score):
    q = np.ascontiguousarray(np.atleast_2d(np.asarray(queries, dtype=np.float64)))
    B = q.shape[0]
    slots = np.empty((B, k_fetch), dtype=np.int64)
    scores = np.empty((B, k_fetch), dtype=np.float64)
    counts = np.empty((B,), dtype=np.int32)
    ms = C.c_float(0)
    ms_arg = -np.inf if min_score is None else float(min_score)
    check(fn(h, ptr(q), B, q.shape[1], k_fetch, ms_arg, ptr(slots), ptr(scores), ptr(counts), C.byref(ms)))
    return slots, scores, counts, ms.value


def _search_each(fn, h, queries, k_fetch, min_score):
    """rbk_*_search_each_f64: k_fetch [B] ints >= 1, min_score [B] floats or None (-inf, as in search()).  Returns
    (slots int64 [B, K], scores float64 [B, K], counts int32 [B], device_ms) with K = max(k_fetch); row b is what
    search_unbounded(queries[b], k_fetch[b], min_score[b]) returns, padded with -1 / NaN to K entries."""
    q = np.ascontiguousarray(np.atleast_2d(np.asarray(queries, dtype=np.float64)))
    B = q.shape[0]
    k32, m, K = _cuts(B, k_fetch, min_score)
    slots = np.empty((B, K), dtype=np.int64)
    scores = np.empty((B, K), dtype=np.float64)
    counts = np.empty((B,), dtype=np.int32)
    ms = C.c_float(0)
    check(fn(h, ptr(q), B, q.shape[1], ptr(k32), ptr(m), ptr(slots), ptr(scores), ptr(counts), C.byref(ms)))
    return slots, scores, counts, ms.value


def _cuts(B: int, k_fetch, min_score):
    """The int32 k_fetch [B], float64 min_score [B] and largest k of a search_each or search_slots call."""
    k = np.ascontiguousarray(np.asarray(k_fetch, dtype=np.int64).reshape(-1))
    ms_list = list(min_score) if np.ndim(min_score) else [min_score] * B
    m = np.ascontiguousarray([-np.inf if v is None else float(v) for v in ms_list], dtype=np.float64)
    if k.shape[0] != B or m.shape[0] != B:
        raise ValueError(f"k_fetch and min_score need one entry per query ({B}), not {k.shape[0]} and {m.shape[0]}")
    if (k < 1).any() or (k > np.iinfo(np.int32).max).any():
        raise RbkError(RBK_EINVAL, "every k_fetch must be in [1, 2^31 - 1]")
    k32 = k.astype(np.int32)
    return k32, m, (int(k32.max()) if B else 0)


def _search_slots(fn, h, slots, k_fetch, min_score):
    """rbk_*_search_slots_f64: the stored rows of global slots [B] as the queries; k_fetch and min_score (None = -inf)
    one per query or one for all.  Returns what _search_each returns for the host copies of those rows."""
    sl = np.ascontiguousarray(np.asarray(slots, dtype=np.int64).reshape(-1))
    B = sl.shape[0]
    k32, m, K = _cuts(B, np.full(B, k_fetch) if np.ndim(k_fetch) == 0 else k_fetch, min_score)
    out_slots = np.empty((B, K), dtype=np.int64)
    scores = np.empty((B, K), dtype=np.float64)
    counts = np.empty((B,), dtype=np.int32)
    ms = C.c_float(0)
    check(fn(h, ptr(sl), B, ptr(k32), ptr(m), ptr(out_slots), ptr(scores), ptr(counts), C.byref(ms)))
    return out_slots, scores, counts, ms.value


def _per_query(B: int, v, name: str, dtype):
    """A scalar or one value per query as a contiguous array [B] of dtype (None = -inf, for min_score)."""
    vals = list(v) if np.ndim(v) else [v] * B
    if len(vals) != B:
        raise ValueError(f"{name} needs one entry per query ({B}), not {len(vals)}")
    if dtype == np.int32:
        a = np.asarray(vals, dtype=np.int64).reshape(-1)
        if (np.abs(a) > np.iinfo(np.int32).max).any():
            raise RbkError(RBK_EINVAL, f"every {name} must fit an int32")
        return np.ascontiguousarray(a, dtype=np.int32)
    return np.ascontiguousarray([-np.inf if x is None else float(x) for x in vals], dtype=np.float64)


def _search_mmr(fn, h, queries, k, fetch_k, lambda_mult, min_score):
    """rbk_*_search_mmr_f64: k, fetch_k, lambda_mult and min_score (None = -inf) one per query or one for all; the
    library checks them.  Returns (slots int64 [B, K], scores float64 [B, K], counts int32 [B], device_ms) with
    K = max(k): row b holds query b's picks in selection order with their relevance, then -1 / NaN."""
    q = np.ascontiguousarray(np.atleast_2d(np.asarray(queries, dtype=np.float64)))
    B = q.shape[0]
    k32 = _per_query(B, k, "k", np.int32)
    f32 = _per_query(B, fetch_k, "fetch_k", np.int32)
    lam = _per_query(B, lambda_mult, "lambda_mult", np.float64)
    m = _per_query(B, min_score, "min_score", np.float64)
    K = int(max(k32.max(), 0)) if B else 0
    slots = np.empty((B, K), dtype=np.int64)
    scores = np.empty((B, K), dtype=np.float64)
    counts = np.empty((B,), dtype=np.int32)
    ms = C.c_float(0)
    check(fn(h, ptr(q), B, q.shape[1], ptr(k32), ptr(f32), ptr(lam), ptr(m), ptr(slots), ptr(scores), ptr(counts),
             C.byref(ms)))
    return slots, scores, counts, ms.value


def _similar_pairs(fn, h, first: int, size: int, min_score, first_slot, max_pairs):
    """rbk_*_similar_pairs_f64: one page of the pairs (a, b) of live slots a < b with cosine >= min_score (None = -inf)
    for the rows a from first_slot on (None: the first slot, `first`), at most max_pairs of them (None: max(size(),
    2^20)), never part of a row's pairs.  Returns (a int64 [n], b int64 [n], scores float64 [n], next_slot): ascending
    a, then score descending, ties by ascending b; next_slot == first + size() when the pass is complete."""
    first_slot = first if first_slot is None else int(first_slot)
    max_pairs = max(size, 1 << 20) if max_pairs is None else int(max_pairs)
    cap = max(max_pairs, 0)
    a = np.empty(cap, dtype=np.int64)
    b = np.empty(cap, dtype=np.int64)
    scores = np.empty(cap, dtype=np.float64)
    n, nxt, ms = C.c_int64(0), C.c_int64(0), C.c_float(0)
    ms_arg = -np.inf if min_score is None else float(min_score)
    check(fn(h, ms_arg, first_slot, max_pairs, ptr(a), ptr(b), ptr(scores), C.byref(n), C.byref(nxt), C.byref(ms)))
    return a[:n.value].copy(), b[:n.value].copy(), scores[:n.value].copy(), nxt.value


def _search_any_k(ix, queries, k_fetch: int, min_score):
    """Shared by Index and Group: the scan path up to RBK_MAX_K_FETCH hits per query, the two-pass large-k search up
    to RBK_MAX_K_FETCH_LARGE, beyond it the exact scores of every row from the device and the reference's threshold /
    stable sort / slice on the host."""
    if k_fetch <= RBK_MAX_K_FETCH:
        return ix.search(queries, k_fetch, min_score)
    if k_fetch <= RBK_MAX_K_FETCH_LARGE:
        return ix.search_large(queries, k_fetch, min_score)
    sc = ix.exact_scores(queries)
    B = sc.shape[0]
    slots = np.full((B, k_fetch), -1, dtype=np.int64)
    scores = np.full((B, k_fetch), np.nan, dtype=np.float64)
    counts = np.zeros(B, dtype=np.int32)
    for b in range(B):
        with np.errstate(invalid="ignore"):
            keep = np.flatnonzero(sc[b] >= min_score) if min_score is not None else np.flatnonzero(~np.isnan(sc[b]))
        order = keep[np.argsort(-sc[b, keep], kind="stable")][:k_fetch]
        counts[b] = len(order)
        slots[b, :len(order)] = order
        scores[b, :len(order)] = sc[b, order]
    return slots, scores, counts, 0.0


def _search_any_k_on_device(ix, queries, k_fetch: int, min_score):
    """search_any_k of Index and Group: every k_fetch on the GPU.  Above RBK_MAX_K_FETCH_LARGE the unbounded search
    sorts the candidates on the device; up to it, _search_any_k's scan and large-k paths."""
    if k_fetch > RBK_MAX_K_FETCH_LARGE:
        return ix.search_unbounded(queries, k_fetch, min_score)
    return _search_any_k(ix, queries, k_fetch, min_score)


class Index:
    """Thin object wrapper over rbk_index* (one GPU shard)."""

    def __init__(self, dim: int, device: int = 0, capacity_hint: int = 0, keep_f64: bool = False,
                 f64_on_host: bool = False, scan_f16: bool = False, keep_f32: bool = False,
                 keep_f32_split: bool = False):
        """keep_f64: RBK_INDEX_KEEP_F64 — exact for arbitrary float64 rows at 8*dim extra bytes per row.
        keep_f32: RBK_INDEX_KEEP_F32 — the same answers from float32 exact rows at 4*dim bytes per row, for rows whose
        values are all float32-exact; append_f64 / overwrite of any other value raise NotFloat32Error with nothing
        written.  Excludes keep_f64.
        keep_f32_split: RBK_INDEX_KEEP_F32_SPLIT — the answers of keep_f32 at 2*dim bytes per row: the bf16 scan copy
        holds each float32's high half and only the low halves are kept beside it.  Same values accepted, same
        NotFloat32Error.  Excludes keep_f64, keep_f32 and scan_f16.
        f64_on_host: RBK_INDEX_F64_ON_HOST (RBK_INDEX_ROWS_ON_HOST) — those exact rows live in pinned host memory
        instead of on the GPU (same answers; the re-rank reads them over PCIe).  Requires keep_f64 or keep_f32.
        scan_f16: RBK_INDEX_SCAN_F16 — the scan reads per-row scaled fp16 rows instead of bf16 (same bytes, same
        answers, a several times tighter error bound, so fewer wide retries).  Requires keep_f64 or keep_f32."""
        self._h = None
        h = C.c_void_p()
        check(lib.rbk_index_create_ex(dim, device, capacity_hint,
                                      _index_flags(keep_f64, f64_on_host, scan_f16, keep_f32, keep_f32_split),
                                      C.byref(h)))
        self._h = h
        self.dim = dim
        self.device = device
        self.slot_base = 0

    def close(self) -> None:
        if getattr(self, "_h", None):
            lib.rbk_index_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- configuration
    def set_stream(self, cuda_stream: int | None) -> None:
        check(lib.rbk_index_set_stream(self._h, C.c_void_p(cuda_stream or 0)))

    def set_slot_base(self, base: int) -> None:
        check(lib.rbk_index_set_slot_base(self._h, base))
        self.slot_base = int(base)

    @property
    def flags(self) -> int:
        """The creation flags as they are now (RBK_INDEX_KEEP_F64, RBK_INDEX_KEEP_F32 or RBK_INDEX_KEEP_F32_SPLIT |
        RBK_INDEX_F64_ON_HOST | RBK_INDEX_SCAN_F16)."""
        return int(lib.rbk_index_flags(self._h))

    def set_tier(self, *, f64_on_host: bool | None = None, scan_f16: bool | None = None,
                 exact_rows: str | None = None) -> None:
        """Change the storage tier in place (rbk_index_set_tier): move the exact rows between the GPU and pinned host
        memory, switch the scan between bf16 and fp16, keep the exact rows as 'f64', 'f32' or 'f32_split'.  None keeps
        a setting.  Needs exact rows; answers do not change.  Raises RbkError(RBK_ENOMEM) with the index unchanged when
        the new tier cannot be backed, NotFloat32Error when a stored value does not fit exact_rows='f32' or
        'f32_split'."""
        check(lib.rbk_index_set_tier(self._h, _tier_flags(self.flags, f64_on_host, scan_f16, exact_rows)))

    # -- mutation
    def _append(self, fn, rows: np.ndarray) -> int:
        if rows.ndim != 2 or rows.shape[1] != self.dim:
            raise DimensionError(RBK_EDIM, "Vectors must have the same length")
        first = C.c_int64(-1)
        check(fn(self._h, ptr(rows), rows.shape[0], C.byref(first)))
        return first.value

    def append_f64(self, rows) -> int:
        return self._append(lib.rbk_index_append_f64, np.ascontiguousarray(rows, dtype=np.float64))

    def append_f32(self, rows) -> int:
        return self._append(lib.rbk_index_append_f32, np.ascontiguousarray(rows, dtype=np.float32))

    def append_bf16(self, rows_u16) -> int:
        return self._append(lib.rbk_index_append_bf16, np.ascontiguousarray(rows_u16, dtype=np.uint16))

    def append_bf16_device(self, dev_ptr: int, n_rows: int) -> int:
        first = C.c_int64(-1)
        check(lib.rbk_index_append_bf16_device(self._h, C.c_void_p(dev_ptr), n_rows, C.byref(first)))
        return first.value

    def append_f64_device(self, dev_ptr: int, n_rows: int) -> int:
        first = C.c_int64(-1)
        check(lib.rbk_index_append_f64_device(self._h, C.c_void_p(dev_ptr), n_rows, C.byref(first)))
        return first.value

    def overwrite_f64(self, slot: int, row) -> None:
        r = np.ascontiguousarray(row, dtype=np.float64)
        if r.shape != (self.dim,):
            raise DimensionError(RBK_EDIM, "Vectors must have the same length")
        check(lib.rbk_index_overwrite_f64(self._h, slot, ptr(r)))

    def overwrite_f64_batch(self, slots, rows) -> None:
        """rows[i] replaces slots[i]; one call and one host round trip for the whole batch."""
        s = np.ascontiguousarray(slots, dtype=np.int64)
        r = np.ascontiguousarray(rows, dtype=np.float64).reshape(-1, self.dim) if len(s) else np.zeros((0, self.dim))
        if r.shape != (s.shape[0], self.dim):
            raise DimensionError(RBK_EDIM, "Vectors must have the same length")
        check(lib.rbk_index_overwrite_f64_batch(self._h, ptr(s), s.shape[0], ptr(r)))

    def tombstone(self, slots) -> None:
        s = np.ascontiguousarray(slots, dtype=np.int64)
        check(lib.rbk_index_tombstone(self._h, ptr(s), s.shape[0]))

    def compact(self) -> np.ndarray:
        """Reclaim the slots of tombstoned rows: the live rows move down to slots 0 .. count()-1 in their current
        order.  Returns old_to_new, int64 [size() before the call]: each old local slot's new one, -1 if it was
        tombstoned."""
        out = np.empty(self.size(), dtype=np.int64)
        check(lib.rbk_index_compact(self._h, ptr(out), out.shape[0]))
        return out

    def clear(self) -> None:
        check(lib.rbk_index_clear(self._h))

    def trim(self) -> None:
        """Give memory back: capacity down to what size() rows need (unmapping the device storage beyond it), every
        scratch buffer released.  Answers and slots do not change; run it after compact() or clear()."""
        check(lib.rbk_index_trim(self._h))

    def count(self) -> int:
        return lib.rbk_index_count(self._h)

    def size(self) -> int:
        return lib.rbk_index_size(self._h)

    def storage_bytes(self) -> tuple[int, int]:
        """(device bytes, pinned host bytes) of the corpus storage at the current capacity; scratch not counted."""
        dev, host = C.c_int64(0), C.c_int64(0)
        check(lib.rbk_index_storage_bytes(self._h, C.byref(dev), C.byref(host)))
        return dev.value, host.value

    def read_rows_bf16(self, first: int, n: int) -> np.ndarray:
        out = np.empty((n, self.dim), dtype=np.uint16)
        check(lib.rbk_index_read_rows_bf16(self._h, first, n, ptr(out)))
        return out

    def read_rows_f16(self, first: int, n: int) -> np.ndarray:
        """The stored fp16 bits of a scan_f16 index (each row scaled by its own power of two)."""
        out = np.empty((n, self.dim), dtype=np.uint16)
        check(lib.rbk_index_read_rows_f16(self._h, first, n, ptr(out)))
        return out

    # -- search
    def search(self, queries, k_fetch: int, min_score: float | None = 0.5):
        """Returns (slots int64 [B,k], scores float64 [B,k], counts int32 [B], device_ms)."""
        q = np.asarray(queries)
        if q.ndim == 1:
            q = q[None, :]
        if q.dtype == np.float32:
            q = np.ascontiguousarray(q)
            fn = lib.rbk_index_search_f32
        else:
            q = np.ascontiguousarray(q, dtype=np.float64)
            fn = lib.rbk_index_search_f64
        B = q.shape[0]
        slots = np.empty((B, k_fetch), dtype=np.int64)
        scores = np.empty((B, k_fetch), dtype=np.float64)
        counts = np.empty((B,), dtype=np.int32)
        ms = C.c_float(0)
        ms_arg = -np.inf if min_score is None else float(min_score)
        check(fn(self._h, ptr(q), B, q.shape[1], k_fetch, ms_arg, ptr(slots), ptr(scores), ptr(counts), C.byref(ms)))
        return slots, scores, counts, ms.value

    def search_large(self, queries, k_fetch: int, min_score: float | None = 0.5):
        """search() for 1 <= k_fetch <= RBK_MAX_K_FETCH_LARGE (f64 queries): count scan, emit scan, exact re-rank."""
        return _search_large(lib.rbk_index_search_large_f64, self._h, queries, k_fetch, min_score)

    def search_unbounded(self, queries, k_fetch: int, min_score: float | None = 0.5):
        """search() for any k_fetch >= 1 (f64 queries): search_large() up to RBK_MAX_K_FETCH_LARGE; above it the same
        two scans, then the candidates sorted on the device, at most count() hits per query."""
        return _search_large(lib.rbk_index_search_unbounded_f64, self._h, queries, k_fetch, min_score)

    def search_each(self, queries, k_fetch, min_score):
        """Each query at its own k_fetch[b] and min_score[b] (None = -inf) in one call (f64 queries): (slots [B, K],
        scores [B, K], counts [B], device_ms), K = max(k_fetch).  Row b equals search_unbounded(queries[b], k_fetch[b],
        min_score[b]); one scan for the batch when K <= RBK_MAX_K_FETCH, else the two scans of the large-k search."""
        return _search_each(lib.rbk_index_search_each_f64, self._h, queries, k_fetch, min_score)

    def search_slots(self, slots, k_fetch, min_score):
        """search_each() whose queries are the stored rows of global slots [B] (the exact rows widened to float64, or
        the bf16 rows without them), read on the device: (slots [B, K], scores [B, K], counts [B], device_ms).  k_fetch
        and min_score (None = -inf): one per query or one for all.  A query's own slot is among its hits; a slot this
        index does not hold, or a tombstoned one, raises RbkError (RBK_EINVAL)."""
        return _search_slots(lib.rbk_index_search_slots_f64, self._h, slots, k_fetch, min_score)

    def search_mmr(self, queries, k, fetch_k, lambda_mult=0.5, min_score=0.5):
        """Diverse hits by maximal marginal relevance (include/rbk_knn.h): per query, k of the fetch_k hits search_each()
        returns at min_score, picked greedily by lambda_mult * relevance - (1 - lambda_mult) * (largest cosine to a
        pick so far).  Arguments one per query or one for all (min_score None = -inf).  Returns (slots [B, K], scores
        [B, K], counts [B], device_ms), K = max(k): the picks in selection order with their relevance, then -1 / NaN."""
        return _search_mmr(lib.rbk_index_search_mmr_f64, self._h, queries, k, fetch_k, lambda_mult, min_score)

    def similar_pairs(self, min_score, first_slot=None, max_pairs=None):
        """One page of every pair of stored rows at or above min_score (None = -inf), exactly: (a [n], b [n],
        scores [n], next_slot) numpy arrays, slots a < b, first_slot <= a < next_slot (first_slot None: slot_base), at
        most max_pairs entries (None: max(size(), 2^20); at least size()).  Ascending a, then score descending, ties by
        ascending b: a's entries are those of search_slots([a], count(), min_score) above a.  The pass is complete when
        next_slot == slot_base + size(); otherwise call again from next_slot."""
        return _similar_pairs(lib.rbk_index_similar_pairs_f64, self._h, self.slot_base, self.size(), min_score,
                              first_slot, max_pairs)

    def exact_scores(self, queries) -> np.ndarray:
        """float64 [B, size()]: the reference's cosine of every row, NaN for tombstoned / zero rows."""
        q = np.ascontiguousarray(np.atleast_2d(np.asarray(queries, dtype=np.float64)))
        out = np.empty((q.shape[0], self.size()), dtype=np.float64)
        check(lib.rbk_index_exact_scores_f64(self._h, ptr(q), q.shape[0], q.shape[1], ptr(out)))
        return out

    def search_any_k(self, queries, k_fetch: int, min_score: float | None = 0.5):
        """search() for any k_fetch: search_large() above RBK_MAX_K_FETCH, search_unbounded() above
        RBK_MAX_K_FETCH_LARGE."""
        return _search_any_k_on_device(self, queries, k_fetch, min_score)

    def search_device(self, q_ptr: int, B: int, k_fetch: int, min_score: float | None, slots_ptr: int,
                      scores_ptr: int, counts_ptr: int) -> None:
        ms_arg = -np.inf if min_score is None else float(min_score)
        check(lib.rbk_index_search_device(self._h, C.c_void_p(q_ptr), B, k_fetch, ms_arg, C.c_void_p(slots_ptr),
                                          C.c_void_p(scores_ptr), C.c_void_p(counts_ptr)))

    def search_device_async(self, q_ptr: int, B: int, k_fetch: int, min_score: float | None, slots_ptr: int,
                            scores_ptr: int, counts_ptr: int, flags_ptr: int) -> None:
        """Enqueue only (no host sync); flags_ptr: device i32[B], 1 = answer not proven exact."""
        ms_arg = -np.inf if min_score is None else float(min_score)
        check(lib.rbk_index_search_device_async(self._h, C.c_void_p(q_ptr), B, k_fetch, ms_arg,
                                                C.c_void_p(slots_ptr), C.c_void_p(scores_ptr),
                                                C.c_void_p(counts_ptr), C.c_void_p(flags_ptr)))

    def debug_scores(self, queries_f32) -> np.ndarray:
        q = np.ascontiguousarray(queries_f32, dtype=np.float32)
        out = np.empty((q.shape[0], self.size()), dtype=np.float32)
        check(lib.rbk_index_debug_scores_f32(self._h, ptr(q), q.shape[0], ptr(out)))
        return out

    def stats(self) -> dict:
        st = RbkStats()
        check(lib.rbk_index_stats(self._h, C.byref(st)))
        return {f: getattr(st, f) for f, _ in RbkStats._fields_}


class Group:
    """rbk_group*: one corpus sharded over several GPUs behind one handle; the Index surface with GLOBAL slots.
    Every search is one C call: per-GPU scans, one NCCL all-gather, merge on devices[0], one synchronisation."""

    def __init__(self, dim: int, devices, capacity_hint: int = 0, keep_f64: bool = False, f64_on_host: bool = False,
                 scan_f16: bool = False, keep_f32: bool = False, keep_f32_split: bool = False):
        """f64_on_host: every member keeps its exact rows in its own pinned host buffer (see Index).
        scan_f16: every member scans fp16 rows (see Index).  keep_f32 / keep_f32_split: every member keeps float32
        exact rows, whole or split (see Index); a call with any non-float32 value is refused before any member
        writes."""
        self._h = None
        devs = np.ascontiguousarray(list(devices), dtype=np.int32)
        h = C.c_void_p()
        check(lib.rbk_group_create(dim, ptr(devs), devs.shape[0], capacity_hint,
                                   _index_flags(keep_f64, f64_on_host, scan_f16, keep_f32, keep_f32_split),
                                   C.byref(h)))
        self._h = h
        self.dim = dim
        self.devices = [int(d) for d in devs]
        self.device = self.devices[0]

    def close(self) -> None:
        if getattr(self, "_h", None):
            lib.rbk_group_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _append(self, fn, rows: np.ndarray) -> int:
        if rows.ndim != 2 or rows.shape[1] != self.dim:
            raise DimensionError(RBK_EDIM, "Vectors must have the same length")
        first = C.c_int64(-1)
        check(fn(self._h, ptr(rows), rows.shape[0], C.byref(first)))
        return first.value

    def append_f64(self, rows) -> int:
        return self._append(lib.rbk_group_append_f64, np.ascontiguousarray(rows, dtype=np.float64))

    def append_f32(self, rows) -> int:
        return self._append(lib.rbk_group_append_f32, np.ascontiguousarray(rows, dtype=np.float32))

    def append_bf16(self, rows_u16) -> int:
        return self._append(lib.rbk_group_append_bf16, np.ascontiguousarray(rows_u16, dtype=np.uint16))

    def overwrite_f64_batch(self, slots, rows) -> None:
        s = np.ascontiguousarray(slots, dtype=np.int64)
        r = np.ascontiguousarray(rows, dtype=np.float64).reshape(-1, self.dim) if len(s) else np.zeros((0, self.dim))
        if r.shape != (s.shape[0], self.dim):
            raise DimensionError(RBK_EDIM, "Vectors must have the same length")
        check(lib.rbk_group_overwrite_f64_batch(self._h, ptr(s), s.shape[0], ptr(r)))

    def overwrite_f64(self, slot: int, row) -> None:
        self.overwrite_f64_batch([slot], np.asarray(row, dtype=np.float64)[None, :])

    def tombstone(self, slots) -> None:
        s = np.ascontiguousarray(slots, dtype=np.int64)
        check(lib.rbk_group_tombstone(self._h, ptr(s), s.shape[0]))

    def clear(self) -> None:
        check(lib.rbk_group_clear(self._h))

    def compact(self) -> np.ndarray:
        """Index.compact() in global slots: the live rows move down to slots 0 .. count()-1 in their current order,
        between devices where the block-cyclic layout says so.  Returns old_to_new, int64 [size() before the call]."""
        out = np.empty(self.size(), dtype=np.int64)
        check(lib.rbk_group_compact(self._h, ptr(out), out.shape[0]))
        return out

    def trim(self) -> None:
        """Index.trim() on every member; slots do not change."""
        check(lib.rbk_group_trim(self._h))

    @property
    def flags(self) -> int:
        """The members' creation flags as they are now (they share them)."""
        return int(lib.rbk_index_flags(C.c_void_p(lib.rbk_group_member(self._h, 0))))

    def set_tier(self, *, f64_on_host: bool | None = None, scan_f16: bool | None = None,
                 exact_rows: str | None = None) -> None:
        """Index.set_tier() on every member together: every member's allocations come first, so RBK_ENOMEM leaves the
        whole group as it was."""
        check(lib.rbk_group_set_tier(self._h, _tier_flags(self.flags, f64_on_host, scan_f16, exact_rows)))

    def count(self) -> int:
        return lib.rbk_group_count(self._h)

    def size(self) -> int:
        return lib.rbk_group_size(self._h)

    def search(self, queries, k_fetch: int, min_score: float | None = 0.5):
        q = np.asarray(queries)
        if q.ndim == 1:
            q = q[None, :]
        if q.dtype == np.float32:
            q = np.ascontiguousarray(q)
            fn = lib.rbk_group_search_f32
        else:
            q = np.ascontiguousarray(q, dtype=np.float64)
            fn = lib.rbk_group_search_f64
        B = q.shape[0]
        slots = np.empty((B, k_fetch), dtype=np.int64)
        scores = np.empty((B, k_fetch), dtype=np.float64)
        counts = np.empty((B,), dtype=np.int32)
        ms = C.c_float(0)
        ms_arg = -np.inf if min_score is None else float(min_score)
        check(fn(self._h, ptr(q), B, q.shape[1], k_fetch, ms_arg, ptr(slots), ptr(scores), ptr(counts), C.byref(ms)))
        return slots, scores, counts, ms.value

    def search_large(self, queries, k_fetch: int, min_score: float | None = 0.5):
        return _search_large(lib.rbk_group_search_large_f64, self._h, queries, k_fetch, min_score)

    def search_unbounded(self, queries, k_fetch: int, min_score: float | None = 0.5):
        return _search_large(lib.rbk_group_search_unbounded_f64, self._h, queries, k_fetch, min_score)

    def search_each(self, queries, k_fetch, min_score):
        """Index.search_each() over the group: one call, every member on the route of the largest k."""
        return _search_each(lib.rbk_group_search_each_f64, self._h, queries, k_fetch, min_score)

    def search_slots(self, slots, k_fetch, min_score):
        """Index.search_slots() over the group: each slot's member gathers its row, then one search_each."""
        return _search_slots(lib.rbk_group_search_slots_f64, self._h, slots, k_fetch, min_score)

    def search_mmr(self, queries, k, fetch_k, lambda_mult=0.5, min_score=0.5):
        """Index.search_mmr() over the group: the candidates' owners gather their rows, device_ids[0] selects."""
        return _search_mmr(lib.rbk_group_search_mmr_f64, self._h, queries, k, fetch_k, lambda_mult, min_score)

    def similar_pairs(self, min_score, first_slot=None, max_pairs=None):
        """Index.similar_pairs() over the group's global slots [0, size()): the answers of a single index."""
        return _similar_pairs(lib.rbk_group_similar_pairs_f64, self._h, 0, self.size(), min_score, first_slot,
                              max_pairs)

    def exact_scores(self, queries) -> np.ndarray:
        """float64 [B, size()]: every device's exact scores, put back in global slot order (4096-row blocks dealt
        out round-robin)."""
        q = np.ascontiguousarray(np.atleast_2d(np.asarray(queries, dtype=np.float64)))
        n, G, blk = self.size(), len(self.devices), 4096
        out = np.full((q.shape[0], n), np.nan, dtype=np.float64)
        glob = np.arange(n, dtype=np.int64)
        owner = (glob // blk) % G
        for g in range(G):
            member = C.c_void_p(lib.rbk_group_member(self._h, g))
            m = lib.rbk_index_size(member)
            if m == 0:
                continue
            part = np.empty((q.shape[0], m), dtype=np.float64)
            check(lib.rbk_index_exact_scores_f64(member, ptr(q), q.shape[0], q.shape[1], ptr(part)))
            out[:, glob[owner == g]] = part          # local row order == global slot order within a device
        return out

    def search_any_k(self, queries, k_fetch: int, min_score: float | None = 0.5):
        return _search_any_k_on_device(self, queries, k_fetch, min_score)

    def stats(self) -> dict:
        out = {"devices": len(self.devices), "redone_batches": lib.rbk_group_redone_batches(self._h)}
        per = []
        for i in range(len(self.devices)):
            st = RbkStats()
            check(lib.rbk_index_stats(C.c_void_p(lib.rbk_group_member(self._h, i)), C.byref(st)))
            per.append({f: getattr(st, f) for f, _ in RbkStats._fields_})
        for k in ("searches", "queries", "fallback_queries", "scan_launches", "kernel_launches", "retry_batches"):
            out[k] = sum(p[k] for p in per)
        out["per_device"] = per
        return out


def merge_topk_device(device: int, stream: int, G: int, B: int, k_fetch: int, slots_ptr: int, scores_ptr: int,
                      counts_ptr: int, out_slots_ptr: int, out_scores_ptr: int, out_counts_ptr: int) -> None:
    check(lib.rbk_merge_topk_device(device, C.c_void_p(stream), G, B, k_fetch, C.c_void_p(slots_ptr),
                                    C.c_void_p(scores_ptr), C.c_void_p(counts_ptr), C.c_void_p(out_slots_ptr),
                                    C.c_void_p(out_scores_ptr), C.c_void_p(out_counts_ptr)))


def packed_block_bytes(B: int, k_fetch: int) -> int:
    return lib.rbk_packed_block_bytes(B, k_fetch)


def packed_flags_offset(B: int, k_fetch: int) -> int:
    return lib.rbk_packed_flags_offset(B, k_fetch)


def merge_topk_packed_device(device: int, stream: int, G: int, B: int, k_fetch: int, blocks_ptr: int,
                             out_slots_ptr: int, out_scores_ptr: int, out_counts_ptr: int,
                             out_flags_ptr: int | None = None) -> None:
    """out_flags_ptr: device i32[B+1] ([b] = OR of the shards' exactness flags, [B] += dirty queries) or None."""
    check(lib.rbk_merge_topk_packed_device(device, C.c_void_p(stream), G, B, k_fetch, C.c_void_p(blocks_ptr),
                                           C.c_void_p(out_slots_ptr), C.c_void_p(out_scores_ptr),
                                           C.c_void_p(out_counts_ptr), C.c_void_p(out_flags_ptr or 0)))
